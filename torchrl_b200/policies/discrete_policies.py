"""Discrete-action policies (API of /root/reference/torchrl/policies/discrete_policies.py).

Differences from the reference, all documented in SURVEY.md Appendix A: the QR-DQN policy's
`q_to_a` works for any number of envs (the reference calls .item(), A.5) and epsilon-greedy
draws stay on the device unless the noise mode is "reference_cpu" (then np.random is used in
the reference's call order).
"""
import numpy as np
import torch
import torch.nn as nn
from torch.distributions import Categorical

from .. import networks
from .. import ops
from . import distribution as D
from .continuous_policy import _DeviceRng


class UniformPolicyDiscrete(nn.Module):
    def __init__(self, action_num):
        super().__init__()
        self.action_num = action_num
        self.continuous = False

    def forward(self, x):
        return np.random.randint(self.action_num)

    def explore(self, x):
        return {"action": np.random.randint(self.action_num)}


def linear_decay(start, end, frames, count):
    """Exploration rate after `count` decisions: linear from `start` to `end` over `frames`, then flat
    (discrete_policies.py:44-49)."""
    if count >= frames:
        return end
    return start - (start - end) * (count / frames)


def _uniform_and_random_actions(shape, n_actions, device):
    """(u in [0,1), a in {0..n_actions-1}) per decision.  "reference_cpu" mode draws them from the global NumPy
    stream in the reference's order (rand, then randint); otherwise they are generated on the device."""
    if D.get_noise_mode() == "reference_cpu":
        u = torch.Tensor(np.random.rand(*shape)).to(device)
        a = torch.LongTensor(np.random.randint(low=0, high=n_actions, size=shape)).to(device)
        return u, a
    return torch.rand(shape, device=device), torch.randint(0, n_actions, shape, device=device)


class EpsilonGreedyDQNDiscretePolicy:
    """epsilon-greedy decisions on top of a Q network (discrete_policies.py:25-74).  Not an nn.Module, like in the
    reference: `to` / `parameters` forward to the wrapped network."""

    def __init__(self, qf, start_epsilon, end_epsilon, decay_frames, action_shape):
        self.qf = qf
        self.start_epsilon, self.end_epsilon, self.decay_frames = start_epsilon, end_epsilon, decay_frames
        self.action_shape = action_shape
        self.count = 0
        self.epsilon = start_epsilon
        self.continuous = False

    def q_to_a(self, q):
        return q.max(dim=-1, keepdim=True)[1].detach()

    def tick(self):
        """Advance the schedule by one decision (host side).  Collectors that replay a captured step graph call
        this outside the graph and hand the rate over in a device scalar (`explore(x, epsilon=tensor)`)."""
        self.count += 1
        self.epsilon = linear_decay(self.start_epsilon, self.end_epsilon, self.decay_frames, self.count)

    def explore(self, x, epsilon=None):
        if epsilon is None:
            self.tick()
            epsilon = self.epsilon
        x = x.squeeze(0)
        output = self.qf(x)
        greedy = self.q_to_a(output)
        u, random_action = _uniform_and_random_actions(tuple(greedy.shape), self.action_shape, x.device)
        return {"q_value": output, "action": torch.where(u < epsilon, random_action, greedy)}

    def eval_act(self, x):
        with torch.no_grad():
            return self.q_to_a(self.qf(x))

    def to(self, device):
        self.qf.to(device)
        return self

    def parameters(self):
        return self.qf.parameters()


class EpsilonGreedyQRDQNDiscretePolicy(EpsilonGreedyDQNDiscretePolicy):
    """Greedy w.r.t. the mean over quantiles (discrete_policies.py:77-89), batched."""

    def __init__(self, quantile_num, **kwargs):
        super().__init__(**kwargs)
        self.quantile_num = quantile_num
        self.continuous = False

    def q_to_a(self, q):
        q = q.view(q.shape[:-1] + (self.action_shape, self.quantile_num))
        return q.mean(dim=-1).max(dim=-1, keepdim=True)[1].detach()


class BootstrappedDQNDiscretePolicy:
    """Greedy actions of one bootstrapped head per env (discrete_policies.py:92-121), batched over envs.  `head` is the
    (N,) int32 device vector of the envs' current heads (the reference's scalar `idx`, one per env).  The collector's
    captured step calls `act`: all heads in one forward, then one launch (csrc/bootstrapped.cu) that redraws the heads
    of envs starting an episode, picks the greedy actions and writes the transition's Bernoulli(`bernoulli_p`) mask
    row.  Not an nn.Module, like in the reference: `to` / `parameters` forward to the wrapped network."""

    def __init__(self, qf, head_num, action_shape):
        self.qf = qf
        self.head_num = head_num
        self.action_shape = action_shape
        self.bernoulli_p = 0.5                 # BootstrappedDQN hands its own value over
        self.head = None
        self.continuous = False
        self._rng = _DeviceRng()
        self._ticket = None

    def ensure_heads(self, n, device):
        """Allocate the (n,) head vector (all head 0) if it does not exist yet; returns it."""
        if self.head is None or self.head.numel() != n or self.head.device != torch.device(device):
            self.head = torch.zeros(n, dtype=torch.int32, device=device)
        return self.head

    def sample_head(self):
        """A new uniform head for every env (the collector redraws them per env at each episode start)."""
        if self.head is not None:
            self.head.copy_(torch.randint(0, self.head_num, self.head.shape, device=self.head.device))

    def set_head(self, idx):
        """Every env to head `idx` (an int), or per env (an (N,) tensor)."""
        if self.head is None:
            raise RuntimeError("no per-env heads yet: the collector allocates them (ensure_heads)")
        if torch.is_tensor(idx):
            self.head.copy_(idx.to(self.head.device, torch.int32))
        else:
            self.head.fill_(int(idx))

    def explore(self, x):
        """The greedy action of each env's head for x (N, ...)."""
        q = self.qf.all_heads(x)
        head = self.ensure_heads(q.shape[1], q.device).long()
        q_value = q[head, torch.arange(q.shape[1], device=q.device)]
        return {"q_value": q_value, "action": q_value.max(dim=-1)[1].detach()}

    def act(self, x, current_step, action_out, masks_ring, top, u_head=None, u_mask=None):
        """The collector's per-step decision (capturable): see trl_bootstrapped_act.  u_head (N) and u_mask (N, H)
        replace the Philox stream."""
        q = self.qf.all_heads(x)
        q = q if q.is_contiguous() else q.contiguous()
        self.ensure_heads(q.shape[1], q.device)
        rng = None
        if u_head is None:
            rng = self._rng.ensure(q.device)
            if self._ticket is None:
                self._ticket = torch.zeros(1, dtype=torch.int32, device=q.device)
        return ops.bootstrapped_act(q.detach(), current_step, self.head, action_out.reshape(-1), masks_ring, top,
                                    self.bernoulli_p, u_head=u_head, u_mask=u_mask, rng=rng, ticket=self._ticket)

    def eval_act(self, x):
        """argmax of the mean over all heads, per row."""
        with torch.no_grad():
            return self.qf.all_heads(x).mean(dim=0).max(dim=-1)[1].detach()

    def to(self, device):
        self.qf.to(device)
        return self

    def parameters(self):
        return self.qf.parameters()


class CategoricalDisPolicy(networks.Net):
    """softmax over the net's outputs (discrete_policies.py:123-160).  `forward` / `explore` / `update` / `eval_act`
    keep the reference's torch semantics; the collector's `act_only` and the on-policy algorithms' fused minibatch
    loop work on the logits with the categorical kernels (csrc/categorical.cu)."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self.continuous = False
        self._rng = _DeviceRng()

    def logits(self, x):
        return networks.Net.forward(self, x)

    def forward(self, x):
        return torch.softmax(self.logits(x), dim=-1)

    def act_only(self, x, action_out=None, nan_flag=None, u=None, eps=None):
        """Collector fast path: one sampled action index per row (as float) into `action_out`, one launch after the
        net (no softmax launch).  u: optional (M,) uniforms in [0,1) replacing the Philox stream.  In the
        "reference_cpu" noise mode the action is drawn with torch.multinomial on the CPU generator from the device
        probabilities, as the reference's Categorical.sample does on a CPU policy (this syncs; not capturable)."""
        logits = self.logits(x)
        logits = logits if logits.is_contiguous() else logits.contiguous()
        if u is None and D.get_noise_mode() == "reference_cpu":
            probs = torch.softmax(logits.detach(), dim=-1).cpu()
            act = torch.multinomial(probs.reshape(-1, probs.shape[-1]), 1, True).reshape(-1)
            if action_out is None:
                return act.to(logits.device, torch.float32)
            action_out.reshape(-1).copy_(act.to(torch.float32))
            return action_out
        rng = None if u is not None else self._rng.ensure(logits.device)
        out = ops.categorical_sample(logits.detach(), u=u, rng=rng, nan_flag=nan_flag,
                                     action_out=None if action_out is None else action_out.reshape(-1))
        if u is None:
            ops.counter_advance(rng.counter)
        return out

    def explore(self, x, return_log_probs=False):
        output = self.forward(x)
        dis = Categorical(output)
        action = dis.sample()
        out = {"dis": output, "action": action}
        if return_log_probs:
            out["log_prob"] = dis.log_prob(action)
        return out

    def eval_act(self, x):
        return self.forward(x).max(dim=-1)[1].detach()

    def update(self, obs, actions):
        dis = Categorical(self.forward(obs))
        return {"dis": dis, "log_prob": dis.log_prob(actions).unsqueeze(-1), "ent": dis.entropy()}
