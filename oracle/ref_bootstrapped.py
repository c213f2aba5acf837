"""NumPy restatement of Bootstrapped DQN's device pieces (csrc/bootstrapped.cu), in fp64 where the arithmetic is
floating point and exactly in float32 where the kernel's rule is a comparison.

TEST INFRASTRUCTURE ONLY.  The semantics are those of the reference's BootstrappedDQN.update
(/root/reference/torchrl/algo/off_policy/bootstrapped_dqn.py:66-113), which tests/golden/bootstrapped_dqn_reference.npz
records executed, and of its intended vectorised collection (per-env head per episode, Bernoulli mask per transition).
"""
import numpy as np


def bootstrapped_targets(rewards, terminals, next_q, gamma):
    """y[h, b] = r_b + gamma (1 - d_b) max_a next_q[h, b, a]: every head on its own target head."""
    r = np.asarray(rewards, np.float64).reshape(1, -1)
    d = np.asarray(terminals, np.float64).reshape(1, -1)
    return r + gamma * (1.0 - d) * np.asarray(next_q, np.float64).max(axis=-1)


def bootstrapped_dqn_loss(pred, next_q, actions, rewards, terminals, masks, gamma):
    """(loss, grad (H, B, A), info3) of loss = mean_b sum_h m_bh (Q_h(s_b, a_b) - y_hb)^2 / H.
    info3 = [loss, mean over (b, h) of Q_h(s_b, a_b), mean reward], the slot layout of the DQN loss."""
    pred = np.asarray(pred, np.float64)
    H, B, A = pred.shape
    a = np.asarray(actions).reshape(-1).astype(np.int64)
    m = np.asarray(masks, np.float64).reshape(B, H).T                    # (H, B)
    q = pred[:, np.arange(B), a]                                          # (H, B)
    d = q - bootstrapped_targets(rewards, terminals, next_q, gamma)
    loss = float((m * d * d).sum() / (H * B))
    grad = np.zeros_like(pred)
    grad[:, np.arange(B), a] = 2.0 * m * d / (H * B)
    info = np.array([loss, q.mean(), np.asarray(rewards, np.float64).mean()])
    return loss, grad, info


def bootstrapped_act(q_all, current_step, head, u_head, u_mask, p):
    """The collector's per-step rule for N envs: (new head (N,), action (N,), mask row (N, H) uint8).
    head[n] = min(floor(u_head[n] * H), H - 1) in float32 where current_step[n] == 0, else unchanged; the action is the
    first argmax of q_all[head[n], n, :]; mask[n, j] = u_mask[n, j] < p in float32."""
    q_all = np.asarray(q_all, np.float32)
    H, N, _ = q_all.shape
    draw = np.minimum(np.floor(np.asarray(u_head, np.float32) * np.float32(H)).astype(np.int64), H - 1)
    new_head = np.where(np.asarray(current_step) == 0, draw, np.asarray(head, np.int64))
    action = np.argmax(q_all[new_head, np.arange(N)], axis=-1)
    mask = (np.asarray(u_mask, np.float32) < np.float32(p)).astype(np.uint8)
    return new_head.astype(np.int32), action, mask
