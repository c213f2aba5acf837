"""Golden data of Bootstrapped DQN (tests/test_bootstrapped_*.py): the unmodified reference's BootstrappedDQN.update
executed on torch CPU behind oracle/shims, recorded so that the device agent can be checked against it on a machine
without a copy of the reference.

TEST INFRASTRUCTURE ONLY.  Needs the reference (oracle/reference_loader.available()):

    python oracle/make_golden_bootstrapped.py      # -> tests/golden/bootstrapped_dqn_reference.npz

The reference's BootstrappedNet cannot be constructed (a missing comma in its __init__ passes `add_ln ** kwargs`),
so the network under test is the reference's own BootstrappedNet class -- its forward -- with the trunk and heads
built here the way its __init__ would build them: the reference's CNNBase as trunk, and per head an nn.Sequential of
Linear + activation for each append_hidden_shapes entry and a last Linear, initialised with the reference's
basic_init / uniform_init, attached as `head<i>`.  The agent is the reference's BootstrappedDQN with optim.Adam.

Recorded per case (keys "<case>|<what>|<name>"):
  * init|<key>: the initial parameters under the repository's BootstrappedNet names (head<i>.* ->
    bootstrapped_heads.<i>.*);
  * batch<u>|obs, next_obs (uint8 frames; the network sees frames / 255 as float32), acts (B,), rewards (B, 1),
    terminals (B, 1), masks (B, H): the explicit batch of update u;
  * update<u>|pred, next, grad: the reference's all-heads outputs of qf and target_qf as (H, B, A) and the gradient of
    its loss wrt the qf outputs; update<u>|info: [Training/qf_loss, Reward_Mean];
  * final|<key>: the parameters after the last update.
"""
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "bootstrapped_dqn_reference.npz")

A = 6
OBS = (4, 16, 16)
HIDDEN = [[8, [4, 4], [2, 2], [0, 0]], [8, [3, 3], [1, 1], [0, 0]]]
APPEND = [16]
B = 16
# case -> (head_num, updates, agent keyword arguments, seed).  "hard": target copies after updates 2 and 4.
CASES = {
    "hard": (5, 5, dict(use_soft_update=False, target_hard_update_period=2), 0),
    "soft": (3, 3, dict(use_soft_update=True, tau=0.05), 1),
}
QLR, EPS, GAMMA = 1e-3, 1e-4, 0.99


def batches(H, n, seed):
    """n explicit batches: uint8 frames, actions, rewards, terminals (a quarter) and Bernoulli(0.5) masks with one
    all-zero and one all-one row."""
    rs = np.random.RandomState(100 + seed)
    out = []
    for _ in range(n):
        m = (rs.rand(B, H) < 0.5).astype(np.uint8)
        m[0] = 0
        m[1] = 1
        out.append({
            "obs": rs.randint(0, 256, (B,) + OBS).astype(np.uint8),
            "next_obs": rs.randint(0, 256, (B,) + OBS).astype(np.uint8),
            "acts": rs.randint(0, A, B).astype(np.float32),
            "rewards": rs.choice([-1.0, 0.0, 1.0], (B, 1)).astype(np.float32),
            "terminals": (rs.rand(B, 1) < 0.25).astype(np.float32),
            "masks": m,
        })
    return out


def frames_to_float(x):
    return x.astype(np.float32) / np.float32(255.0)


def repo_key(k):
    if k.startswith("head"):
        idx, rest = k[4:].split(".", 1)
        return "bootstrapped_heads.%s.%s" % (idx, rest)
    return k


def _standin_net(trl, H):
    import torch.nn as nn
    from torchrl.networks import base, init, nets

    net = nets.BootstrappedNet.__new__(nets.BootstrappedNet)
    nn.Module.__init__(net)
    net.base = base.CNNBase(input_shape=OBS, hidden_shapes=HIDDEN, activation_func=nn.ReLU, add_ln=False)
    net.add_ln = False
    net.activation_func = nn.ReLU
    net.bootstrapped_heads = []
    for idx in range(H):
        layers, width = [], net.base.output_shape
        for nxt in APPEND:
            fc = nn.Linear(width, nxt)
            init.basic_init(fc)
            layers += [fc, nn.ReLU()]
            width = nxt
        last = nn.Linear(width, A)
        init.uniform_init(last)
        head = nn.Sequential(*layers, last)
        setattr(net, "head{}".format(idx), head)
        net.bootstrapped_heads.append(head)
    return net


def _capture(net, store):
    """Keep every forward's list of head outputs (with their gradients retained) in `store`."""
    fwd = net.forward

    def forward(x, head_idxs):
        out = fwd(x, head_idxs)
        for t in out:
            if t.requires_grad:
                t.retain_grad()
        store.append(out)
        return out

    net.forward = forward


def golden_case(trl, name, H, n, kw, seed, out):
    import gym
    import torch
    from torchrl.algo import BootstrappedDQN
    from torchrl.policies import BootstrappedDQNDiscretePolicy

    torch.manual_seed(seed)
    qf = _standin_net(trl, H)
    for k, v in qf.state_dict().items():
        out["%s|init|%s" % (name, repo_key(k))] = v.numpy().copy()
    pf = BootstrappedDQNDiscretePolicy(qf, H, A)
    env = types.SimpleNamespace(action_space=gym.spaces.Discrete(A))
    collector = types.SimpleNamespace(epoch_frames=B)
    agent = BootstrappedDQN(head_num=H, bernoulli_p=0.5, qf=qf, pf=pf, qlr=QLR, optimizer_info={"eps": EPS},
                            env=env, replay_buffer=None, collector=collector, logger=None, discount=GAMMA,
                            batch_size=B, device="cpu", save_dir=tempfile.mkdtemp(), **kw)
    preds, nexts = [], []
    _capture(agent.qf, preds)
    _capture(agent.target_qf, nexts)
    for u, b in enumerate(batches(H, n, seed)):
        for k, v in b.items():
            out["%s|batch%d|%s" % (name, u, k)] = v
        feed = dict(b, obs=frames_to_float(b["obs"]), next_obs=frames_to_float(b["next_obs"]))
        info = agent.update(feed)
        p, q = preds[-1], nexts[-1]
        out["%s|update%d|pred" % (name, u)] = np.stack([t.detach().numpy() for t in p])
        out["%s|update%d|next" % (name, u)] = np.stack([t.detach().numpy() for t in q])
        out["%s|update%d|grad" % (name, u)] = np.stack([t.grad.numpy() for t in p])
        out["%s|update%d|info" % (name, u)] = np.array([info["Training/qf_loss"], info["Reward_Mean"]], np.float64)
    for k, v in agent.qf.state_dict().items():
        out["%s|final|%s" % (name, repo_key(k))] = v.numpy().copy()


def generate():
    from oracle import reference_loader
    trl = reference_loader.load()
    out = {}
    for name, (H, n, kw, seed) in CASES.items():
        golden_case(trl, name, H, n, kw, seed, out)
    return out


def main():
    out = generate()
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
