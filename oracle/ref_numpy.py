"""NumPy (float64) restatements of the reference's hot-path arithmetic.

TEST INFRASTRUCTURE ONLY -- the checker for the CUDA kernels, never the thing
shipped or measured (bench.py's cpu_baseline leg excepted).  Each function cites
the reference lines it restates (paths relative to /root/reference).  Pinned
against the real reference by oracle/make_golden.py -> tests/golden/*.npz and
tests/test_oracle_vs_reference.py (the latter runs only where /root/reference
exists).
"""
import numpy as np


# --------------------------------------------------------------------------- K6
def gae(rewards, values, terminals, time_limits, last_value, gamma, tau, time_limit_filter):
    """Generalised advantage estimation, backward over time.

    Restates torchrl/replay_buffers/on_policy.py:16-44.  All arrays are
    time-major (T, N, 1) (or (T, N)); last_value is (N, 1) (or (N,)).
        delta_t = r_t + (1-term_t)*gamma*V_{t+1} - V_t
        A_t     = delta_t + (1-term_t)*gamma*tau*A_{t+1};  A_t *= (1-tl_t) if filter
        ret_t   = A_t + V_t
    """
    rewards = np.asarray(rewards, dtype=np.float64)
    values = np.asarray(values, dtype=np.float64)
    nt = 1.0 - np.asarray(terminals, dtype=np.float64)
    keep = 1.0 - np.asarray(time_limits, dtype=np.float64)
    T = rewards.shape[0]
    advs = np.empty_like(rewards)
    rets = np.empty_like(rewards)
    v_next = np.asarray(last_value, dtype=np.float64).reshape(rewards.shape[1:])
    run = np.zeros_like(v_next)
    for t in range(T - 1, -1, -1):
        delta = rewards[t] + nt[t] * gamma * v_next - values[t]
        run = delta + nt[t] * gamma * tau * run
        if time_limit_filter:
            run = run * keep[t]
        advs[t] = run
        rets[t] = run + values[t]
        v_next = values[t]
    return advs, rets


def discount_return(rewards, values, terminals, time_limits, last_value, gamma, time_limit_filter):
    """Discounted-reward returns (the non-GAE branch).

    Restates torchrl/replay_buffers/on_policy.py:46-70:
        R_t = r_t + (1-term_t)*gamma*R_{t+1}*(1-tl_t) + tl_t*V_t      (filter on)
        R_t = r_t + (1-term_t)*gamma*R_{t+1}                           (filter off)
        adv_t = R_t - V_t ; ret_t = R_t
    """
    rewards = np.asarray(rewards, dtype=np.float64)
    values = np.asarray(values, dtype=np.float64)
    nt = 1.0 - np.asarray(terminals, dtype=np.float64)
    tl = np.asarray(time_limits, dtype=np.float64)
    T = rewards.shape[0]
    advs = np.empty_like(rewards)
    rets = np.empty_like(rewards)
    R = np.asarray(last_value, dtype=np.float64).reshape(rewards.shape[1:])
    for t in range(T - 1, -1, -1):
        if time_limit_filter:
            R = rewards[t] + nt[t] * gamma * R * (1.0 - tl[t]) + tl[t] * values[t]
        else:
            R = rewards[t] + nt[t] * gamma * R
        advs[t] = R - values[t]
        rets[t] = R
    return advs, rets


# --------------------------------------------------------------------------- K2
class RunningNorm:
    """Running mean/var observation normaliser.

    Restates torchrl/env/base_wrapper.py:44-60 (Chan parallel-variance merge),
    :63-73 (state: mean 0, var 1, count 1e-4, clip 10), :75-82 (batch moments:
    mean and *population* variance over axis 0) and :91-94 (filter).
    """

    def __init__(self, dim, clip=10.0):
        self.mean = np.zeros((dim,), dtype=np.float64)
        self.var = np.ones((dim,), dtype=np.float64)
        self.count = 1e-4
        self.clip = clip

    def update(self, batch):
        batch = np.asarray(batch, dtype=np.float64)
        b_mean = batch.mean(axis=0)
        b_var = batch.var(axis=0)
        b_n = batch.shape[0]
        delta = b_mean - self.mean
        tot = self.count + b_n
        new_mean = self.mean + delta * b_n / tot
        m2 = self.var * self.count + b_var * b_n + np.square(delta) * self.count * b_n / tot
        self.mean, self.var, self.count = new_mean, m2 / tot, tot

    def filt(self, raw):
        raw = np.asarray(raw, dtype=np.float64)
        return np.clip((raw - self.mean) / (np.sqrt(self.var) + 1e-4), -self.clip, self.clip)


# --------------------------------------------------------------------------- K1 helpers
def norm_act(action, lb, ub):
    """[-1,1] -> [lb,ub] then clip.  torchrl/env/continuous_wrapper.py:18-20."""
    scaled = lb + (np.asarray(action, dtype=np.float64) + 1.0) * 0.5 * (ub - lb)
    return np.clip(scaled, lb, ub)


# --------------------------------------------------------------------------- K7 / K9
def uniform_row_indices(size, batch_size, env_nums):
    """Row indices of BaseReplayBuffer.random_batch (torchrl/replay_buffers/base.py:39-44):
    batch_size//env_nums draws of np.random.randint(0, size) from the GLOBAL legacy RNG."""
    assert batch_size % env_nums == 0
    return np.random.randint(0, size, batch_size // env_nums)


def epoch_row_order(rows, shuffle):
    """Row visiting order of one_iteration (torchrl/replay_buffers/on_policy.py:76-78)."""
    if shuffle:
        return np.random.permutation(rows)
    return np.arange(rows)


def gather_rows(arr, idx):
    """(T,N,D)[idx] -> (len(idx)*N, D).  base.py:46-50 / on_policy.py:83-88."""
    out = np.asarray(arr)[idx]
    return out.reshape((out.shape[0] * out.shape[1],) + out.shape[2:])


def normalize_advantages(advs):
    """(adv-mean)/(std_unbiased+1e-5) over the minibatch.  torchrl/algo/on_policy/ppo.py:147
    (torch.std defaults to the unbiased estimator)."""
    advs = np.asarray(advs, dtype=np.float64)
    return (advs - advs.mean()) / (advs.std(ddof=1) + 1e-5)


# --------------------------------------------------------------------------- K3 / K8
_LOG_2PI = np.log(2.0 * np.pi)


def normal_log_prob(x, mean, std):
    return -((x - mean) ** 2) / (2.0 * std * std) - np.log(std) - 0.5 * _LOG_2PI


def normal_entropy(std):
    return 0.5 + 0.5 * _LOG_2PI + np.log(std)


def tanh_normal_log_prob(action, mean, std, pre_tanh=None, eps=1e-6):
    """Per-dimension log-prob of a tanh-squashed Gaussian.

    torchrl/policies/distribution.py:33-45: when the pre-tanh value is not given it
    is recovered as log((1+a)/(1-a))/2 (a = +-1 gives +-inf -- kept on purpose)."""
    action = np.asarray(action, dtype=np.float64)
    if pre_tanh is None:
        with np.errstate(divide="ignore", invalid="ignore"):
            pre_tanh = np.log((1.0 + action) / (1.0 - action)) / 2.0
    return normal_log_prob(pre_tanh, mean, std) - np.log(1.0 - action * action + eps)


def ppo_actor_loss(mean, log_std, actions, old_log_prob, advs, clip_para, entropy_coeff, tanh_action=True):
    """PPO clipped surrogate + entropy bonus (scalar) and the per-sample pieces.

    torchrl/algo/on_policy/ppo.py:48-67 with log-probs from
    torchrl/policies/continuous_policy.py:134-153 (sum over action dims, keepdim)
    and Normal entropy (distribution.py:78-79)."""
    std = np.exp(log_std)
    std_b = np.broadcast_to(std, mean.shape)
    if tanh_action:
        lp = tanh_normal_log_prob(actions, mean, std_b)
    else:
        lp = normal_log_prob(actions, mean, std_b)
    log_prob = lp.sum(-1, keepdims=True)
    ent = normal_entropy(std_b).sum(-1, keepdims=True)
    ratio = np.exp(log_prob - old_log_prob)
    s1 = ratio * advs
    s2 = np.clip(ratio, 1.0 - clip_para, 1.0 + clip_para) * advs
    loss = -np.mean(np.minimum(s2, s1)) - entropy_coeff * ent.mean()
    return loss, log_prob, ratio, ent


def ppo_critic_loss(values, old_values, returns, clip_para, clipped):
    """torchrl/algo/on_policy/ppo.py:100-111."""
    if clipped:
        v_clip = old_values + np.clip(values - old_values, -clip_para, clip_para)
        return 0.5 * np.mean(np.maximum((values - returns) ** 2, (v_clip - returns) ** 2))
    return np.mean((values - returns) ** 2)


# --------------------------------------------------------------------------- K10
def sac_q_target(rewards, terminals, q1_next, q2_next, next_log_prob, alpha, gamma):
    """r + (1-d)*gamma*(min(Q1',Q2') - alpha*logpi').  torchrl/algo/off_policy/twin_sac_q.py:133-139."""
    v = np.minimum(q1_next, q2_next) - alpha * next_log_prob
    return rewards + (1.0 - terminals) * gamma * v


def td3_q_target(rewards, terminals, q1_next, q2_next, gamma):
    """r + (1-d)*gamma*min(Q1',Q2').  torchrl/algo/off_policy/td3.py:86-90."""
    return rewards + (1.0 - terminals) * gamma * np.minimum(q1_next, q2_next)


def td3_smooth_action(target_action, noise, noise_clip):
    """clamp(a' + clamp(noise, +-c), -1, 1).  torchrl/algo/off_policy/td3.py:82-84."""
    return np.clip(target_action + np.clip(noise, -noise_clip, noise_clip), -1.0, 1.0)


def huber(x, k=1.0):
    """torchrl/algo/utils.py:12-13."""
    ax = np.abs(x)
    return np.where(ax < k, 0.5 * x * x, k * (ax - 0.5 * k))


def quantile_regression_loss(tau, source, target):
    """mean over (B, Q_target, Q_source) of huber(diff)*|tau - 1[diff<0]|.

    torchrl/algo/utils.py:5-9: diff[b,j,i] = target[b,j] - source[b,i]; the
    coefficient tau (1,Q) broadcasts along the LAST axis (source index i)."""
    diff = target[:, :, None] - source[:, None, :]
    w = np.abs(tau.reshape(1, 1, -1) - (diff < 0).astype(np.float64))
    return np.mean(huber(diff) * w)


def qrdqn_targets(rewards, terminals, next_quantiles, gamma):
    """Greedy-by-mean target quantiles.  torchrl/algo/off_policy/qrdqn.py:46-55.
    next_quantiles (B, A, Q); rewards/terminals (B, 1) -> (B, Q)."""
    a_star = next_quantiles.mean(axis=2).argmax(axis=1)
    picked = next_quantiles[np.arange(next_quantiles.shape[0]), a_star]
    return rewards + gamma * (1.0 - terminals) * picked, a_star


def dqn_target(rewards, terminals, next_q, gamma):
    """r + gamma*(1-d)*max_a Q'(s',a).  torchrl/algo/off_policy/dqn.py:57-58."""
    return rewards + gamma * (1.0 - terminals) * next_q.max(axis=-1, keepdims=True)


# --------------------------------------------------------------------------- K11
def polyak(target, source, tau):
    """theta' <- (1-tau)*theta' + tau*theta.  torchrl/algo/utils.py:16-20."""
    return target * (1.0 - tau) + source * tau


def clip_coef(total_norm, max_norm):
    """torch.nn.utils.clip_grad_norm_: min(1, max_norm/(norm+1e-6))."""
    return min(1.0, max_norm / (total_norm + 1e-6))


def adam_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """torch.optim.Adam (no weight decay / amsgrad), `step` is the 1-based count."""
    m = beta1 * m + (1 - beta1) * g
    v = beta2 * v + (1 - beta2) * g * g
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = np.sqrt(v) / np.sqrt(bc2) + eps
    return p - (lr / bc1) * m / denom, m, v


# --------------------------------------------------------------------------- prioritised replay (unpinned)
def per_sample(prio, size, u, beta):
    """Stratified proportional sampling of time rows + importance weights.

    PARITY UNPINNED against the reference (it has no prioritised replay, SURVEY.md fact 7).  What is restated here
    is the PUBLISHED algorithm -- Schaul, Quan, Antonoglou, Silver, "Prioritized Experience Replay", ICLR 2016
    (arXiv:1511.05952), proportional variant -- at this buffer's sampling granularity (one priority per time row):
      * eq. (1): P(i) = p_i^alpha / sum_k p_k^alpha            (`prio` already holds p_i^alpha, see per_update)
      * sec. 3.4: w_i = (N * P(i))^-beta, normalised by max_i w_i = (N * min_k P(k))^-beta (over the rows with
        P(k) > 0, the only ones that can be drawn)
      * appendix B.2.1: "to sample a minibatch of size k, the range [0, p_total] is divided equally into k ranges;
        next, a value is uniformly sampled from each range": target_k = (k + u_k) / b * p_total, and the row whose
        cumulative priority interval contains the target is retrieved (their sum-tree walk == searchsorted on the
        inclusive prefix sum).
    tests/test_per_oracle.py holds this function to those three statements (sampling frequencies, weight formula,
    one draw per stratum).  prio: (rows,) float32; u: (b,) uniforms in [0,1).  Returns (idx int64 (b,), weights
    float64 (b,))."""
    p = np.asarray(prio[:size], dtype=np.float64)
    pre = np.cumsum(p)
    total = pre[-1]
    b = len(u)
    target = (np.arange(b, dtype=np.float64) + np.asarray(u, dtype=np.float64)) / b * total
    idx = np.searchsorted(pre, target, side="right")
    # a target that rounds up to the total ((b-1+u)/b == 1 for u within 2^-53 of 1) finds no row: it draws the last
    # row with a positive priority (a zero-priority row has probability 0 and is never drawn)
    positive = np.flatnonzero(p > 0)
    assert positive.size, "per_sample needs at least one row with a positive priority (all %d are zero)" % size
    idx = np.minimum(idx, positive[-1])
    max_w = (size * p[positive].min() / total) ** (-beta)
    w = (size * p[idx] / total) ** (-beta) / max_w
    return idx.astype(np.int64), w


def per_update(prio, idx, td, alpha, eps, max_prio):
    """Schaul et al. 2016, Algorithm 1 line 12 with the proportional priority of sec. 3.3: p_i = |delta_i| + eps,
    stored as p_i^alpha.  A sampled index is a time row of N transitions: its |delta| is the mean over the row's N
    TD errors.  Returns the new running maximum priority (Algorithm 1 line 6: new transitions enter with max p)."""
    new = (np.abs(np.asarray(td, dtype=np.float64)).mean(axis=1).astype(np.float32) + np.float32(eps)) ** np.float32(alpha)
    prio[idx] = new
    return max(float(max_prio), float(new.max()))
