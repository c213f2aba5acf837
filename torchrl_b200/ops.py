"""Tensor-level wrappers over the C ABI (include/torchrl_b200.h).

Each function takes torch CUDA tensors and launches the sm_90a kernel on torch's *current*
stream (so every call is CUDA-graph capturable); _lib.call checks every tensor's dtype,
contiguity and device against the header's declaration before the launch.  Memory is owned
by PyTorch's caching allocator; the library never allocates.  There is no CPU
implementation: CPU tensors raise.
"""
import ctypes

import torch

from . import _lib

F32, F64, I32, I64 = torch.float32, torch.float64, torch.int32, torch.int64


def _stream():
    """torch's current stream.  Until torch has initialised CUDA that is the null stream (0) and no tensor is on the
    device, so a wrapper handed CPU tensors reaches _lib.call's operand check instead of failing here first."""
    return torch.cuda.current_stream().cuda_stream if torch.cuda.is_initialized() else 0


class CapturedGraph:
    """torch.cuda.CUDAGraph capture of `fn` that also remembers how many library kernels it holds,
    so that replays keep `_lib.launch_count()` truthful."""

    def __init__(self, fn):
        self.graph = torch.cuda.CUDAGraph()
        before = _lib.launch_count()
        with torch.cuda.graph(self.graph):
            fn()
        self.launches = _lib.launch_count() - before
        _lib.add_launches(-self.launches)          # capture records, it does not execute

    def replay(self):
        self.graph.replay()
        _lib.add_launches(self.launches)


def _tn(t):
    """(T, N) sizes of a (T,N) or (T,N,1) tensor."""
    if t.dim() == 3 and t.shape[2] == 1:
        return t.shape[0], t.shape[1]
    if t.dim() == 2:
        return t.shape[0], t.shape[1]
    raise ValueError("expected a (T,N) or (T,N,1) tensor, got %s" % (tuple(t.shape),))


# ------------------------------------------------------------------------------------------ K6
def gae_scan(rewards, values, terminals, time_limits, last_value, gamma, tau, time_limit_filter,
             advs=None, returns=None, variant=1):
    """GAE backward scan.  Mirrors OnPolicyReplayBufferBase.generalized_advantage_estimation
    (/root/reference/torchrl/replay_buffers/on_policy.py:16-44) on (T,N[,1]) device tensors."""
    T, N = _tn(rewards)
    if advs is None:
        advs = torch.empty_like(rewards)
    if returns is None:
        returns = torch.empty_like(rewards)
    assert values.shape == rewards.shape and terminals.shape == rewards.shape and \
        time_limits.shape == rewards.shape and last_value.numel() == N
    _lib.call("trl_gae_scan", rewards, values, terminals, time_limits, last_value, advs, returns, T, N, float(gamma),
              float(tau), int(bool(time_limit_filter)), int(variant), _stream())
    return advs, returns


def discount_return(rewards, values, terminals, time_limits, last_value, gamma, time_limit_filter,
                    advs=None, returns=None, variant=1):
    """Discounted-reward returns.  Mirrors OnPolicyReplayBufferBase.discount_reward
    (/root/reference/torchrl/replay_buffers/on_policy.py:46-70)."""
    T, N = _tn(rewards)
    if advs is None:
        advs = torch.empty_like(rewards)
    if returns is None:
        returns = torch.empty_like(rewards)
    assert values.shape == rewards.shape and last_value.numel() == N
    _lib.call("trl_discount_return", rewards, values, terminals, time_limits, last_value, advs, returns, T, N,
              float(gamma), int(bool(time_limit_filter)), int(variant), _stream())
    return advs, returns


# ------------------------------------------------------------------------------------------ K2
def obs_norm_moments(x, sums=None):
    N, o = x.shape
    if sums is None:
        sums = torch.empty(2 * o, dtype=F64, device=x.device)
    _lib.call("trl_obs_norm_moments", x, N, o, sums, _stream())
    return sums


def obs_norm_merge(sums, batch_n, mean, var, count):
    o = mean.numel()
    _lib.call("trl_obs_norm_merge", sums, float(batch_n), o, mean, var, count, _stream())


def obs_norm_filt(raw, mean, var, clip=10.0, out=None):
    N, o = raw.shape
    if out is None:
        out = torch.empty_like(raw)
    _lib.call("trl_obs_norm_filt", raw, mean, var, N, o, float(clip), out, _stream())
    return out


# ------------------------------------------------------------------------------------------ K3
def tanh_gaussian_sample(mean, log_std, eps=None, tanh_action=True, want_log_prob=False, want_pre_tanh=False,
                         want_eps=False, noise_scale=1.0, rng=None, nan_flag=None, action_out=None):
    """action = tanh(mean + exp(log_std)*eps) (+ log-prob, pre-tanh).  eps None -> Philox noise keyed by
    (rng.seed, rng.counter).  Mirrors TanhNormal.rsample / log_prob
    (/root/reference/torchrl/policies/distribution.py:60-76, 33-45)."""
    a = mean.shape[-1]
    M = mean.numel() // a
    action = action_out if action_out is not None else torch.empty_like(mean)
    pre = torch.empty_like(mean) if want_pre_tanh else None
    logp = torch.empty(mean.shape[:-1] + (1,), dtype=F32, device=mean.device) if want_log_prob else None
    eps_out = torch.empty_like(mean) if want_eps else None
    ls_stride = 0 if log_std.dim() == 1 else a
    if ls_stride:
        assert log_std.shape == mean.shape
    seed, ctr = (0, None)
    if eps is None:
        if rng is None or rng.counter is None:
            raise ValueError("tanh_gaussian_sample needs either eps or an rng state")
        seed, ctr = rng.seed, rng.counter
    _lib.call("trl_tanh_gaussian_sample", mean, log_std, ls_stride, eps, float(noise_scale), ctypes.c_uint64(seed), ctr,
              M, a, int(bool(tanh_action)), action, pre, logp, eps_out, nan_flag, _stream())
    out = {"action": action}
    if pre is not None:
        out["pre_tanh"] = pre
    if logp is not None:
        out["log_prob"] = logp
    if eps_out is not None:
        out["eps"] = eps_out
    return out


def tanh_gaussian_sample_bwd(action, eps, log_std, g_action, g_logp, tanh_action):
    a = action.shape[-1]
    M = action.numel() // a
    g_mean = torch.empty_like(action)
    g_ls = torch.empty_like(action)
    ls_stride = 0 if log_std.dim() == 1 else a
    ga = g_action.contiguous() if g_action is not None else None
    gl = g_logp.contiguous() if g_logp is not None else None
    _lib.call("trl_tanh_gaussian_sample_bwd", action, eps, log_std, ls_stride, ga, gl, M, a, int(bool(tanh_action)),
              g_mean, g_ls, _stream())
    return g_mean, g_ls


def counter_advance(counter, t_ptr=None, T=1, size_ptr=None):
    """Device-side `counter += 1` (and optionally t = (t+1) % T, size = min(size+1, T))."""
    _lib.call("trl_step_advance", t_ptr, int(T), size_ptr, counter, _stream())


def collect_finalize(cur_ob_in, next_norm, state, act, value, v_next, reward, done, tl, elapsed, episode, seeds,
                     step_count, ep_return, epoch_reward, ret_log, n_done, any_reset, norm_mean, norm_var, cur_ob_out,
                     b_obs, b_next_obs, b_acts, b_values, b_rewards, b_terminals, b_time_limits, t_ptr,
                     max_episode_frames, discount, init_scale, clip, terminal_includes_surpass, raw_obs_after_reset):
    """The end of one collector step (csrc/collect.cu): row `*t_ptr` of the replay ring, episode returns, the timeout
    bootstrap and the partial reset of the finished envs.  cur_ob_in (N, o), act (N, a).  state / elapsed / episode /
    seeds / any_reset None: host envs (the host resets them afterwards)."""
    N, o = cur_ob_in.shape
    _lib.call("trl_collect_finalize", cur_ob_in, next_norm, state, act, value, v_next, reward, done, tl, elapsed,
              episode, seeds, step_count, ep_return, epoch_reward, ret_log, n_done, any_reset, norm_mean, norm_var,
              cur_ob_out, b_obs, b_next_obs, b_acts, b_values, b_rewards, b_terminals, b_time_limits, t_ptr, N, o,
              act.numel() // N, int(max_episode_frames), float(discount), float(init_scale), float(clip),
              int(bool(terminal_includes_surpass)), int(bool(raw_obs_after_reset)), _stream())


# ------------------------------------------------------------------------------------------ K7/K9/K4
class RowCopyPlan:
    """Pre-built key table for trl_row_gather / trl_ring_write (host arrays of device pointers)."""

    def __init__(self, srcs, dsts, row_bytes):
        n = len(srcs)
        assert n == len(dsts) == len(row_bytes) and 1 <= n <= 8
        self.n = n
        self.src = (ctypes.c_void_p * n)(*[s.data_ptr() for s in srcs])
        self.dst = (ctypes.c_void_p * n)(*[d.data_ptr() for d in dsts])
        self.rb = (ctypes.c_int64 * n)(*[int(b) for b in row_bytes])
        self._keep = (list(srcs), list(dsts))


def row_bytes_of(t):
    """bytes of one time-row of a (T, N, ...) tensor"""
    return t[0].numel() * t.element_size()


def row_gather(plan, idx, rows, pos_ptr=None):
    """dst[k] = src[idx[pos*rows + k]] for every key of the plan; idx is an int64 device tensor."""
    _lib.call("trl_row_gather", plan.n, plan.src, plan.dst, plan.rb, idx, pos_ptr, int(rows), _stream())


def ring_write(plan, row_ptr):
    """dst[*row_ptr] = src[0] for every key of the plan (one time-row)."""
    _lib.call("trl_ring_write", plan.n, plan.src, plan.dst, plan.rb, row_ptr, _stream())


def ring_write_advance(plan, row_ptr, T, ticket, size_ptr=None):
    """ring_write(plan, row_ptr) then row_ptr = (row_ptr + 1) % T [, size = min(size + 1, T)] in one launch.
    ticket: a zero-initialised int32[1] owned by the caller."""
    _lib.call("trl_ring_write_advance", plan.n, plan.src, plan.dst, plan.rb, row_ptr, int(T), size_ptr, ticket,
              _stream())


def vec_stats(x, out=None):
    """[mean, unbiased std, max, min] of a float vector, on the device."""
    if out is None:
        out = torch.empty(4, dtype=F32, device=x.device)
    _lib.call("trl_vec_stats", x, x.numel(), out, _stream())
    return out


def vec_moments(x, out):
    """out (4) f64 = sum, sum of squares, max, -min of a float vector: one rank's share of vec_stats."""
    _lib.call("trl_vec_moments", x, x.numel(), out, _stream())
    return out


def vec_stats_from_moments(gathered, world, n_total, out):
    """out (4) f32 = mean, unbiased std, max, min from `world` ranks' vec_moments, (world, 4) f64."""
    _lib.call("trl_vec_stats_from_moments", gathered, int(world), float(n_total), out, _stream())
    return out


# ------------------------------------------------------------------------------------------ K8
class LossScratch:
    """Scratch + ticket for the two-level reductions of the loss kernels (allocated once)."""

    def __init__(self, B, act_dim, device, categorical=False):
        lib = _lib.load()
        n = int(lib.trl_ppo_categorical_actor_scratch_doubles(int(B)) if categorical
                else lib.trl_ppo_actor_scratch_doubles(int(B), int(act_dim)))
        self.actor = torch.zeros(max(n, 1), dtype=F64, device=device)
        self.critic = torch.zeros(max((int(B) + 255) // 256, 1), dtype=F64, device=device)
        self.tickets = torch.zeros(4, dtype=I32, device=device)
        self.B, self.a = int(B), int(act_dim)


def ppo_actor_loss(mean, log_std, actions, old_logp, advs, adv_stats, clip_para, entropy_coeff, tanh_action,
                   scratch, g_mean=None, g_log_std=None, info=None, logp_out=None, stats_pos=None, ls_clamp=None):
    """PPO clipped-surrogate loss value, dL/dmean, dL/dlog_std and logged stats in one launch
    (/root/reference/torchrl/algo/on_policy/ppo.py:41-91).  ls_clamp=(lo, hi): `log_std` is the raw parameter, the
    policy's torch.clamp is applied inside the kernel and g_log_std is the gradient of the raw parameter."""
    ls_lo, ls_hi = (1.0, -1.0) if ls_clamp is None else (float(ls_clamp[0]), float(ls_clamp[1]))
    B, a = mean.shape
    assert scratch.B >= B and scratch.a == a
    ls_stride = 0 if log_std.dim() == 1 else a
    if g_mean is None:
        g_mean = torch.empty_like(mean)
    if g_log_std is None:
        g_log_std = torch.empty_like(log_std)
    if info is None:
        info = torch.zeros(16, dtype=F32, device=mean.device)
    _lib.call("trl_ppo_actor_loss", mean, log_std, ls_stride, actions, old_logp, advs, adv_stats, stats_pos, B, a,
              int(bool(tanh_action)), float(clip_para), float(entropy_coeff), ls_lo, ls_hi, g_mean, g_log_std, logp_out,
              info, scratch.actor, scratch.tickets[0:1], _stream())
    return g_mean, g_log_std, info


def ppo_critic_loss(values, returns, old_values, clipped, clip_para, scratch, g_values=None, info=None):
    """Critic loss value and dL/dV (/root/reference/torchrl/algo/on_policy/ppo.py:93-122)."""
    B = values.numel()
    if g_values is None:
        g_values = torch.empty_like(values)
    if info is None:
        info = torch.zeros(1, dtype=F32, device=values.device)
    _lib.call("trl_ppo_critic_loss", values, returns, old_values, B, int(bool(clipped)), float(clip_para), g_values,
              info, scratch.critic, scratch.tickets[1:2], _stream())
    return g_values, info


def gaussian_log_prob(mean, log_std, actions, tanh_action, out=None):
    B, a = mean.shape
    if out is None:
        out = torch.empty(B, dtype=F32, device=mean.device)
    ls_stride = 0 if log_std.dim() == 1 else a
    _lib.call("trl_gaussian_log_prob", mean, log_std, ls_stride, actions, B, a, int(bool(tanh_action)), out, _stream())
    return out


# ------------------------------------------------------------------------------------------ K13 categorical
def categorical_sample(logits, u=None, rng=None, action_out=None, want_log_prob=False, nan_flag=None):
    """Action index (as float) ~ Categorical(softmax(logits)) by inverse CDF: u (M,) supplied uniforms in [0,1), or
    Philox keyed by (rng.seed, rng.counter, row).  Mirrors CategoricalDisPolicy.explore
    (/root/reference/torchrl/policies/discrete_policies.py:131-144)."""
    A = logits.shape[-1]
    M = logits.numel() // A
    action = action_out if action_out is not None else torch.empty(M, dtype=F32, device=logits.device)
    assert action.numel() == M
    logp = torch.empty(M, dtype=F32, device=logits.device) if want_log_prob else None
    seed, ctr = (0, None)
    if u is None:
        if rng is None or rng.counter is None:
            raise ValueError("categorical_sample needs either u or an rng state")
        seed, ctr = rng.seed, rng.counter
    _lib.call("trl_categorical_sample", logits, u, ctypes.c_uint64(seed), ctr, M, A, action, logp, nan_flag, _stream())
    return (action, logp) if want_log_prob else action


def categorical_log_prob(logits, actions, out=None):
    """log(clamp(softmax(logits)[a], eps, 1-eps)) per row: Categorical.log_prob of stored actions."""
    A = logits.shape[-1]
    M = logits.numel() // A
    if out is None:
        out = torch.empty(M, dtype=F32, device=logits.device)
    assert actions.numel() == M and out.numel() == M
    _lib.call("trl_categorical_log_prob", logits, actions, M, A, out, _stream())
    return out


def ppo_categorical_actor_loss(logits, actions, old_logp, advs, adv_stats, clip_para, entropy_coeff, scratch,
                               g_logits=None, info=None, logp_out=None, stats_pos=None):
    """The actor loss of PPO (old_logp given, clipped surrogate) or A2C (old_logp None) for a categorical policy:
    value, dL/dlogits and the logged statistics in one launch (ppo.py:41-91, a2c.py:66-70).  `scratch` is a
    LossScratch(..., categorical=True)."""
    B, A = logits.shape
    assert scratch.B >= B
    if g_logits is None:
        g_logits = torch.empty_like(logits)
    if info is None:
        info = torch.zeros(16, dtype=F32, device=logits.device)
    _lib.call("trl_ppo_categorical_actor_loss", logits, actions, old_logp, advs, adv_stats, stats_pos, B, A,
              float(clip_para), float(entropy_coeff), g_logits, logp_out, info, scratch.actor, scratch.tickets[0:1],
              _stream())
    return g_logits, info


def vmpo_select(advs, stats, groups, b, perm=None, out=None):
    """V-MPO's top half of every minibatch (v_mpo.py:65-71) in one launch: out (groups, k) int64, k = B - B // 2, the
    ascending positions of the k largest normalised advantages of minibatch u (ties: lower position first), where
    minibatch u is the time rows perm[u*b:(u+1)*b] of advs (rows, n) in gather_rows order, B = b * n, normalised with
    stats row u.  perm None: advs holds one minibatch of B = b * n values in order (groups must be 1)."""
    n = advs.numel() // advs.shape[0] if perm is not None else advs.numel() // b
    B = b * n
    if perm is None and groups != 1:
        raise ValueError("vmpo_select without a permutation selects from one minibatch")
    if stats.numel() < 4 * groups:
        raise ValueError("vmpo_select needs a (groups, 4) statistics table")
    if out is None:
        out = torch.empty(groups, B - B // 2, dtype=I64, device=advs.device)
    if out.numel() != groups * (B - B // 2):
        raise ValueError("vmpo_select: out must hold (groups, B - B // 2) positions")
    _lib.call("trl_vmpo_select", advs, perm, int(groups), int(b), int(n), stats, out, _stream())
    return out


class VMPOScratch:
    """Scratch + ticket of trl_vmpo_categorical_loss for up to k selected rows (allocated once)."""

    def __init__(self, k, device):
        n = int(_lib.load().trl_vmpo_categorical_scratch_doubles(int(k)))
        self.partial = torch.zeros(max(n, 1), dtype=F64, device=device)
        self.ticket = torch.zeros(1, dtype=I32, device=device)
        self.k = int(k)


def vmpo_categorical_loss(logits, target_logits, actions, advs, adv_stats, dual, eta_eps, alpha_eps, per_row_kl,
                          scratch, g_dual, info, stats_pos=None, g_logits=None):
    """The categorical V-MPO actor loss on the k selected rows (v_mpo.py:73-99): dL/dlogits (returned), dL/d[eta,
    alpha] written into g_dual (2) -- the duals' slice of the flat gradient -- and info (12) = policy_loss,
    alpha_loss, -, -, logprob/{mean,std,max,min}, KL/{mean,std,max,min}.  per_row_kl False: the reference's summed KL
    (reference_quirks); True: the per-row KL."""
    k, A = logits.shape
    if target_logits.shape != logits.shape:
        raise ValueError("target_logits must have the shape of logits")
    if actions.numel() != k or advs.numel() != k or dual.numel() != 2 or g_dual.numel() != 2 or info.numel() < 12:
        raise ValueError("vmpo_categorical_loss: (k) actions and advs, (2) dual and g_dual, (12) info")
    if scratch.k < k:
        raise ValueError("vmpo_categorical_loss: scratch sized for %d rows, got %d" % (scratch.k, k))
    if g_logits is None:
        g_logits = torch.empty_like(logits)
    _lib.call("trl_vmpo_categorical_loss", logits, target_logits, actions, advs, adv_stats, stats_pos, dual, int(k),
              int(A), float(eta_eps), float(alpha_eps), int(bool(per_row_kl)), g_logits, g_dual, info, scratch.partial,
              scratch.ticket, _stream())
    return g_logits


def categorical_fisher_vp(logits, tangent, scale, out=None):
    """TRPO's Fisher-vector product in logit space (trpo.py:29-86): scale * (p * t - p <p, t>) per row of (M, A)
    logits and their tangent t = J v, p = softmax(logits).  Back-propagating the result through the logits gives
    J^T (diag p - p p^T) J v * scale."""
    A = logits.shape[-1]
    M = logits.numel() // A
    if tangent.shape != logits.shape:
        raise ValueError("categorical_fisher_vp: tangent must have the shape of logits")
    if out is None:
        out = torch.empty_like(logits)
    if out.shape != logits.shape:
        raise ValueError("categorical_fisher_vp: out must have the shape of logits")
    _lib.call("trl_categorical_fisher_vp", logits, tangent, M, A, float(scale), out, _stream())
    return out


def tangent_bias_act(t, bias_tangent, y, act):
    """In place t <- (t + bias_tangent[c]) * act'(y) (act 0 none, 1 tanh, 2 ReLU; act'(y) from the layer's cached
    output y) on (M, C, H, W) conv outputs or (M, C) linear outputs: the bias and activation step of TRPO's tangent
    forward pass.  Returns t."""
    if t.dim() < 2:
        raise ValueError("tangent_bias_act: t must be (M, C) or (M, C, H, W)")
    M, C = t.shape[0], t.shape[1]
    S = t.numel() // max(M * C, 1) if M * C else 1
    if bias_tangent.numel() != C:
        raise ValueError("tangent_bias_act: bias_tangent must hold one value per channel (%d)" % C)
    if act != 0 and (y is None or y.shape != t.shape):
        raise ValueError("tangent_bias_act: y must have the shape of t")
    _lib.call("trl_tangent_bias_act", t, bias_tangent, y if act != 0 else None, M, C, S, int(act), _stream())
    return t


class SurrogateScratch:
    """Scratch + ticket of trl_categorical_surrogate for up to M rows (allocated once)."""

    def __init__(self, M, device):
        self.partial = torch.zeros(max((int(M) + 255) // 256, 1), dtype=F64, device=device)
        self.ticket = torch.zeros(1, dtype=I32, device=device)
        self.M = int(M)


def categorical_surrogate(logits, actions, logp_old, advn, scratch, out=None):
    """TRPO's line-search score of one candidate (trpo.py:113-129): -mean(exp(logp - logp_old) * advn) as a (1,)
    device tensor, logp the clamped log-probability of categorical_log_prob.  Deterministic, one launch."""
    A = logits.shape[-1]
    M = logits.numel() // A
    if actions.numel() != M or logp_old.numel() != M or advn.numel() != M:
        raise ValueError("categorical_surrogate: (M) actions, logp_old and advn")
    if scratch.M < M:
        raise ValueError("categorical_surrogate: scratch sized for %d rows, got %d" % (scratch.M, M))
    if out is None:
        out = torch.empty(1, dtype=F32, device=logits.device)
    _lib.call("trl_categorical_surrogate", logits, actions, logp_old, advn, M, A, out, scratch.partial, scratch.ticket,
              _stream())
    return out


def row_group_moments(x, idx, groups, b, out=None):
    """out (groups,4) f64 = sum, sum of squares, max, -min over the rows idx[u*b:(u+1)*b] of x (rows, n)."""
    n = x.numel() // x.shape[0]
    if out is None:
        out = torch.empty(groups, 4, dtype=F64, device=x.device)
    _lib.call("trl_row_group_moments", x, idx, int(groups), int(b), n, out, _stream())
    return out


def group_stats_from_moments(gathered, world, groups, n_total, out=None):
    """out (groups,4) f32 = mean, unbiased std, max, min per group from (world, groups, 4) raw moments."""
    if out is None:
        out = torch.empty(groups, 4, dtype=F32, device=gathered.device)
    _lib.call("trl_group_stats_from_moments", gathered, int(world), int(groups), float(n_total), out, _stream())
    return out


# ------------------------------------------------------------------------------------------ K11
def polyak_update(target_flat, source_flat, tau, planes=None):
    """target <- (1 - tau) target + tau source on flat buffers; planes = (hi, lo) flat TF32 planes of the target
    kept current in the same pass (flat.FlatParams.hi / .lo)."""
    hi, lo = planes if planes is not None else (None, None)
    _lib.call("trl_polyak_update", target_flat, source_flat, target_flat.numel(), float(tau), hi, lo, _stream())


def grad_sumsq_blocks(nseg):
    """float64 scratch elements of grad_sumsq for `nseg` segments."""
    return int(_lib.load().trl_grad_sumsq_blocks(int(nseg)))


def grad_sumsq(grad, seg_begin, nseg, mask, sumsq3, step_counts, betas, scratch, ticket):
    """Per-segment sum of squares of the flat gradient, Adam step counts and bias corrections into sumsq3 (3 nseg f64)
    for the active segments of `mask`.  seg_begin: host int64 array of the nseg + 1 segment offsets."""
    _lib.call("trl_grad_sumsq", grad, seg_begin, int(nseg), int(mask), sumsq3, step_counts, float(betas[0]),
              float(betas[1]), scratch, ticket, _stream())


def adam_step(param, grad, exp_avg, exp_avg_sq, seg_begin, nseg, mask, sumsq3, lr, max_norm, eps, betas, grad_scale,
              zero_grad, hi, lo):
    """Clip (per segment, by the norms in sumsq3) + Adam on the flat buffers, optionally zeroing `grad`; hi / lo: the
    TF32 planes of `param` kept current.  seg_begin / max_norm / eps: host arrays (int64, float, float)."""
    _lib.call("trl_adam_step", param, grad, exp_avg, exp_avg_sq, seg_begin, int(nseg), int(mask), sumsq3, lr, max_norm,
              eps, float(betas[0]), float(betas[1]), float(grad_scale), int(bool(zero_grad)), hi, lo, _stream())


# ------------------------------------------------------------------------------------------ K10
class OffPolicyScratch:
    """Scratch + tickets for the off-policy loss kernels (allocated once per batch size)."""

    def __init__(self, B, device):
        n = int(_lib.load().trl_offpolicy_scratch_doubles(int(B)))
        self.buf = [torch.zeros(max(n, 1), dtype=F64, device=device) for _ in range(5)]
        self.tickets = torch.zeros(8, dtype=I32, device=device)
        self.B = int(B)

    def t(self, i):
        return self.tickets[i:i + 1]

    def b(self, i):
        return self.buf[i]


def td_target(rewards, terminals, q1_next, q2_next, logp_next, log_alpha, gamma, scratch, y=None, info=None,
              fixed_alpha=1.0):
    """y = r + (1-d)*gamma*(min(Q1',Q2') - alpha*logpi')  (SAC, twin_sac_q.py:133-139) or the TD3 form
    (td3.py:86-90) when logp_next is None.  info[0] = mean reward."""
    B = rewards.numel()
    if y is None:
        y = torch.empty(B, dtype=F32, device=rewards.device)
    if info is None:
        info = torch.zeros(1, dtype=F32, device=rewards.device)
    _lib.call("trl_td_target", rewards, terminals, q1_next, q2_next, logp_next, log_alpha, float(fixed_alpha),
              float(gamma), B, y, info, scratch.b(0), scratch.t(0), _stream())
    return y, info


def td3_smooth_action(action, sigma, noise_clip, eps=None, rng=None, out=None):
    """clamp(a + clamp(sigma*eps, +-c), +-1)  (td3.py:75-84)."""
    if out is None:
        out = torch.empty_like(action)
    seed, ctr = (0, None)
    if eps is None:
        seed, ctr = rng.seed, rng.counter
    _lib.call("trl_td3_smooth_action", action, eps, float(sigma), float(noise_clip), ctypes.c_uint64(seed), ctr,
              action.numel(), out, _stream())
    return out


def sac_alpha_step(logp, target_entropy, log_alpha, adam_state, lr, scratch, info=None, betas=(0.9, 0.999), eps=1e-8):
    """Temperature loss and its Adam step in one launch (twin_sac_q.py:111-123); info = [alpha, alpha_loss]."""
    if info is None:
        info = torch.zeros(2, dtype=F32, device=logp.device)
    _lib.call("trl_sac_alpha_step", logp, float(target_entropy), log_alpha, adam_state, float(lr), float(betas[0]),
              float(betas[1]), float(eps), logp.numel(), info, scratch.b(1), scratch.t(1), _stream())
    return info


def sac_policy_loss(logp, q1, q2, log_alpha, scratch, info=None, fixed_alpha=1.0):
    """mean(alpha*logpi - min(q1,q2)) with gradients wrt its three inputs (twin_sac_q.py:145-153)."""
    B = logp.numel()
    g_lp, g1, g2 = torch.empty_like(logp), torch.empty_like(q1), torch.empty_like(q2)
    if info is None:
        info = torch.zeros(5, dtype=F32, device=logp.device)
    _lib.call("trl_sac_policy_loss", logp, q1, q2, log_alpha, float(fixed_alpha), B, g_lp, g1, g2, info, scratch.b(2),
              scratch.t(2), _stream())
    return g_lp, g1, g2, info


def sac_v_loss(logp, qn1, qn2, v_pred, log_alpha, scratch, reparameterization=True, info=None, fixed_alpha=1.0):
    """SAC / TwinSAC with a V network (sac.py:128-144, twin_sac.py:138-156) in one launch: value target
    min(qn1, qn2) - alpha*logpi (qn2 None: one critic), mean squared value error and the policy loss, with the
    gradients wrt logp, qn1, qn2 and v_pred.  info = [policy_loss, vf_loss, logp mean/std/max/min]."""
    B = logp.numel()
    g_lp, g1, g_v = torch.empty_like(logp), torch.empty_like(qn1), torch.empty_like(v_pred)
    g2 = torch.empty_like(qn2) if qn2 is not None else None
    if info is None:
        info = torch.zeros(6, dtype=F32, device=logp.device)
    _lib.call("trl_sac_v_loss", logp, qn1, qn2, v_pred, log_alpha, float(fixed_alpha), int(bool(reparameterization)), B,
              g_lp, g1, g2, g_v, info, scratch.b(2), scratch.t(5), _stream())
    return g_lp, g1, g2, g_v, info


def twin_mse_loss(q1, q2, y, scratch, info=None):
    """MSE of one or two critics against y: losses in info[0:2], gradients returned (twin_sac_q.py:142-143)."""
    B = q1.numel()
    g1 = torch.empty_like(q1)
    g2 = torch.empty_like(q2) if q2 is not None else None
    if info is None:
        info = torch.zeros(2, dtype=F32, device=q1.device)
    _lib.call("trl_twin_mse_loss", q1, q2, y, B, g1, g2, info, scratch.b(3), scratch.t(3), _stream())
    return g1, g2, info


def twin_mse_loss_weighted(q1, q2, y, weights, scratch, info=None, td_out=None):
    """Importance-weighted MSE of one or two critics against y (prioritised replay): mean(w (q - y)^2) in info[0:2],
    gradients returned, the unweighted |q - y| in td_out (B, critics) when given.  weights None: twin_mse_loss's bits."""
    B = q1.numel()
    g1 = torch.empty_like(q1)
    g2 = torch.empty_like(q2) if q2 is not None else None
    if info is None:
        info = torch.zeros(2, dtype=F32, device=q1.device)
    if weights is not None and weights.numel() != B:
        raise ValueError("weights has %d elements for a batch of %d" % (weights.numel(), B))
    if td_out is not None and td_out.numel() != B * (1 if q2 is None else 2):
        raise ValueError("td_out has %d elements, want %d" % (td_out.numel(), B * (1 if q2 is None else 2)))
    _lib.call("trl_twin_mse_loss_weighted", q1, q2, y, weights, B, g1, g2, td_out, info, scratch.b(3), scratch.t(3),
              _stream())
    return g1, g2, info


def qr_dqn_loss(pred, nxt, actions, rewards, terminals, gamma, scratch, n_actions, n_quantiles, mse=False, kappa=1.0,
                info=None, weights=None, td_out=None):
    """Fused (QR-)DQN loss: quantile-Huber (qrdqn.py:36-60, utils.py:5-13) or squared TD error (dqn.py:53-60);
    returns d loss / d pred with the shape of pred and info = [loss, mean q_s_a, mean reward]."""
    B = rewards.numel()
    grad = torch.empty_like(pred)
    if info is None:
        info = torch.zeros(3, dtype=F32, device=pred.device)
    _lib.call("trl_qr_dqn_loss", pred, nxt, actions, rewards, terminals, weights, B, int(n_actions), int(n_quantiles),
              float(gamma), float(kappa), int(bool(mse)), grad, td_out, info, scratch.b(4), scratch.t(4), _stream())
    return grad, info


def bootstrapped_dqn_loss(pred, nxt, actions, rewards, terminals, masks, gamma, scratch, info=None, grad=None):
    """Masked multi-head TD loss of Bootstrapped DQN (bootstrapped_dqn.py:66-113) in one launch: pred / nxt (H, B, A),
    masks (B, H) uint8.  Returns d loss / d pred (H, B, A) and info = [loss, mean q_s_a over (b, h), mean reward]."""
    H, B, A = pred.shape
    assert nxt.shape == pred.shape and masks.shape == (B, H) and rewards.numel() == B and scratch.B >= B
    if grad is None:
        grad = torch.empty_like(pred)
    if info is None:
        info = torch.zeros(3, dtype=F32, device=pred.device)
    _lib.call("trl_bootstrapped_dqn_loss", pred, nxt, actions, rewards, terminals, masks, B, H, A, float(gamma), grad,
              info, scratch.b(4), scratch.t(4), _stream())
    return grad, info


def bootstrapped_act(q_all, current_step, head, action, masks_ring, top, bernoulli_p, u_head=None, u_mask=None,
                     rng=None, ticket=None):
    """Per-env head / greedy action / bootstrap mask row of one collector step (csrc/bootstrapped.cu): q_all (H, N, A);
    new heads where current_step == 0; masks_ring (T, N, H) row *top written.  Uniforms u_head (N) and u_mask (N, H),
    or Philox keyed by (rng.seed, rng.counter), which the launch advances (ticket: zeroed int32[1])."""
    H, N, A = q_all.shape
    assert masks_ring.shape[1:] == (N, H)
    seed, ctr = 0, None
    if u_head is None:
        if rng is None or rng.counter is None or ticket is None:
            raise ValueError("bootstrapped_act needs u_head / u_mask or an rng state and a ticket")
        seed, ctr = rng.seed, rng.counter
    _lib.call("trl_bootstrapped_act", q_all, current_step, head, action, masks_ring, top, u_head, u_mask,
              ctypes.c_uint64(seed), ctr, ticket, N, H, A, float(bernoulli_p), _stream())
    return action


# ------------------------------------------------------------------------------------------ K9 prioritised
def per_sample(prio, size, u, beta, idx=None, weights=None):
    """Stratified proportional row sampling + importance weights (csrc/prioritized.cu; parity unpinned)."""
    b = u.numel()
    if idx is None:
        idx = torch.empty(b, dtype=I64, device=prio.device)
    if weights is None:
        weights = torch.empty(b, dtype=F32, device=prio.device)
    _lib.call("trl_per_sample", prio, int(size), u, b, float(beta), idx, weights, _stream())
    return idx, weights


PER_MAX_ROWS = 1 << 24


def per_scratch_doubles(capacity):
    """Scratch doubles per_sample_rows needs for a ring of `capacity` rows."""
    n = int(_lib.load().trl_per_scratch_doubles(int(capacity)))
    if n < 0:
        raise ValueError("a prioritised ring holds 1..%d rows, not %d" % (PER_MAX_ROWS, capacity))
    return n


def per_sample_rows(prio, size_ptr, u, pos_ptr, b, beta, scratch, idx, weights):
    """per_sample's draw over a ring of prio.numel() <= 2^24 rows with the live size (*size_ptr) and the draw position
    (uniforms u[*pos_ptr * b:][:b]) on the device, so one captured graph serves every update (two kernels)."""
    capacity = prio.numel()
    if scratch.numel() < per_scratch_doubles(capacity):
        raise ValueError("per_sample_rows: scratch holds %d doubles, want %d" % (scratch.numel(),
                                                                                 per_scratch_doubles(capacity)))
    if idx.numel() != b or weights.numel() != b:
        raise ValueError("per_sample_rows: idx / weights must hold b = %d elements" % b)
    _lib.call("trl_per_sample_rows", prio, capacity, size_ptr, u, pos_ptr, int(b), float(beta), idx, weights, scratch,
              _stream(), kernels=2)
    return idx, weights


def per_update(prio, idx, td, alpha, eps, max_prio):
    """prio[idx_k] = (mean_n |td[k,n]| + eps)^alpha (a row drawn twice: its last draw's value) and running max
    priority."""
    b = idx.numel()
    n = td.numel() // b
    _lib.call("trl_per_update", prio, idx, td, b, n, float(alpha), float(eps), max_prio, _stream())


def per_insert(prio, row_ptr, max_prio):
    _lib.call("trl_per_insert", prio, row_ptr, max_prio, _stream())


# ------------------------------------------------------------------------------------------ tensor-core GEMM
def gemm_tf32x3_nt(a, b, out=None, splits=1, workspace=None, bias=None, act=0):
    """out (M,256) = a (M,K) @ b (256,K)^T on the tensor cores (wgmma) with 3xTF32 error compensation
    (csrc/gemm_tf32x3.cu).  a, b contiguous fp32, K % (32*splits) == 0."""
    M, K = a.shape
    assert b.shape == (256, K), "B must be (256, K)"
    if out is None:
        out = torch.empty(M, 256, dtype=F32, device=a.device)
    if splits > 1 and workspace is None:
        workspace = torch.empty(splits * M * 256, dtype=F32, device=a.device)
    _lib.call("trl_gemm_tf32x3_nt", a, b, out, M, K, int(splits), workspace, bias, int(act), _stream(),
              kernels=2 if splits > 1 else 1)       # + the split-K reduction
    return out


def gemm_tf32x3_tn(a, b, out=None, splits=1, workspace=None):
    """out (M,256) = a (K,M)^T @ b (K,256): the weight-gradient shape dW = g^T x on the tensor cores (wgmma)
    (3xTF32), operands consumed M/N-major straight from their row-major storage (no transposes)."""
    K, M = a.shape
    assert b.shape == (K, 256), "B must be (K, 256)"
    if out is None:
        out = torch.empty(M, 256, dtype=F32, device=a.device)
    if splits > 1 and workspace is None:
        workspace = torch.empty(splits * M * 256, dtype=F32, device=a.device)
    _lib.call("trl_gemm_tf32x3_tn", a, b, out, M, K, int(splits), workspace, _stream(), kernels=2 if splits > 1 else 1)
    return out


def gemm3_pair(a, b, out=None, planes=None, b_nmajor=False, bias=None, act=0):
    """out (M,256) = act(a (M,K) @ B + bias) on the tensor cores (csrc/gemm_pair.cu, wgmma, 3xTF32).
    b_nmajor False: b is (256,K) and B = b^T (Linear forward); True: b is (K,256) and B = b (dgrad).
    planes = (hi, lo): pre-split TF32 planes of b (same shape), else b is split in shared memory."""
    M, K = a.shape
    assert tuple(b.shape) == ((K, 256) if b_nmajor else (256, K)), "B must be (K,256) if b_nmajor else (256,K)"
    if out is None:
        out = torch.empty(M, 256, dtype=F32, device=a.device)
    bh, bl = planes if planes is not None else (b, None)
    assert bh.shape == b.shape and (bl is None or bl.shape == b.shape)
    _lib.call("trl_gemm3_pair", a, bh, bl, out, M, K, int(bool(b_nmajor)), bias, int(act), _stream())
    return out


def gemm3_pair_tn(a, b, out=None, splits=1, workspace=None):
    """out (M,256) = a (K,M)^T @ b (K,256) on the tensor cores: the weight-gradient shape, deterministic split-K."""
    K, M = a.shape
    assert b.shape == (K, 256), "B must be (K, 256)"
    if out is None:
        out = torch.empty(M, 256, dtype=F32, device=a.device)
    if splits > 1 and workspace is None:
        workspace = torch.empty(splits * M * 256, dtype=F32, device=a.device)
    _lib.call("trl_gemm3_pair_tn", a, b, out, M, K, int(splits), workspace, _stream(), kernels=2 if splits > 1 else 1)
    return out


def gemm3_pair_tn_cluster(a, b, workspace, tickets, out=None, splits=64):
    """gemm3_pair_tn's result bit for bit in one launch: the split-K sum runs through thread-block clusters.
    workspace: 8*M*256 floats; tickets: M // 8 zeroed int32 (left zero), one set per stream."""
    K, M = a.shape
    assert b.shape == (K, 256), "B must be (K, 256)"
    assert workspace.numel() >= 8 * M * 256 and tickets.numel() >= M // 8, "workspace / tickets too small"
    if out is None:
        out = torch.empty(M, 256, dtype=F32, device=a.device)
    _lib.call("trl_gemm3_pair_tn_cluster", a, b, out, M, K, int(splits), workspace, tickets, _stream())
    return out


def gemm3_pair_dgrad_act_wgrad(g, planes_t, h1, x, act, scratch):
    """The first layer's weight / bias gradient slab partials of dH1 = g (M,256) @ W2, dH1 never stored: the
    partials trl_skinny_act_wgrad_partial(dH1, h1, x) writes, bit for bit, into `scratch`
    (trl_skinny_tn_scratch_floats(M, 256, K) floats; summed by trl_skinny_reduce_jobs, kind 1).
    planes_t = (hi^T, lo^T): the transposed pre-split planes of W2.  M <= 16896, x (M,K) with K <= 24."""
    M, K = x.shape
    hi, lo = planes_t
    assert g.shape == (M, 256) and h1.shape == (M, 256) and hi.shape == (256, 256) and lo.shape == (256, 256)
    _lib.call("trl_gemm3_pair_dgrad_act_wgrad", g, hi, lo, h1, x, M, K, int(act), scratch, _stream())
    return scratch


def skinny_n_dgrad_act_wgrad_partial(g, w, y, act, gz, db_scratch, w_scratch):
    """The output layer's backward in one pass over y (M,256): gz = (g (M,N) @ w (N,256)) * act'(y) into `gz`, and
    the slab partials of db = colsum(gz) into `db_scratch` (trl_skinny_dgrad_act_scratch_floats(M, 256) floats;
    reduce kind 2) and of dW = g^T y, dbias = colsum(g) into `w_scratch` (trl_skinny_tn_scratch_floats(M, 256, N)
    floats; kind 0, out_transposed = 1): trl_skinny_n_dgrad_act_partial's and trl_skinny_tn_partial's bits."""
    M, H = y.shape
    N = w.shape[0]
    assert g.shape == (M, N) and w.shape == (N, H) and gz.shape == (M, H)
    _lib.call("trl_skinny_n_dgrad_act_wgrad_partial", g, w, y, gz, M, H, N, int(act), db_scratch, w_scratch, _stream())


def skinny_n_dgrad_act_wgrad(g, w, y, act, gz, db, dw, dbias, db_scratch, w_scratch):
    """skinny_n_dgrad_act_wgrad_partial, then both slab sums in one launch: db (256), dw (N,256), dbias (N)."""
    M, H = y.shape
    N = w.shape[0]
    assert g.shape == (M, N) and w.shape == (N, H) and gz.shape == (M, H)
    assert db.shape == (H,) and dw.shape == (N, H) and dbias.shape == (N,)
    _lib.call("trl_skinny_n_dgrad_act_wgrad", g, w, y, gz, db, dw, dbias, M, H, N, int(act), db_scratch, w_scratch,
              _stream(), kernels=2)


def transpose_f32(x, out=None):
    """out (C,R) = x (R,C)^T (contiguous)."""
    R, C = x.shape
    if out is None:
        out = torch.empty(C, R, dtype=F32, device=x.device)
    _lib.call("trl_transpose_f32", x, out, R, C, _stream())
    return out


def split_tf32(x, hi=None, lo=None):
    """(hi, lo) TF32 planes of a contiguous fp32 tensor: hi = tf32(x), lo = x - hi (csrc/mlp_epilogue.cu)."""
    hi = torch.empty_like(x) if hi is None else hi
    lo = torch.empty_like(x) if lo is None else lo
    assert hi.numel() == x.numel() and lo.numel() == x.numel()
    _lib.call("trl_split_tf32", x, x.numel(), hi, lo, _stream(), kernels=int(x.numel() > 0))
    return hi, lo


# ------------------------------------------------------------------------------------------ MLP layer epilogues
def bias_act_bwd_scratch_floats(M, H):
    return int(_lib.load().trl_bias_act_bwd_scratch_floats(int(M), int(H)))


def bias_act_fwd(z, bias, act):
    """z (M,H) <- act(z + bias) in place."""
    M, H = z.shape
    _lib.call("trl_bias_act_fwd", z, bias, M, H, int(act), _stream(), kernels=int(M > 0))
    return z


def bias_act_bwd(g, y, gz, db, act, scratch, tickets):
    """gz = g * act'(y) and db = colsum(gz) for y (M,H); scratch: bias_act_bwd_scratch_floats(M, H) floats, tickets:
    (H + 127) // 128 zeroed int32 (left zero)."""
    M, H = y.shape
    _lib.call("trl_bias_act_bwd", g, y, gz, db, M, H, int(act), scratch, tickets, _stream())


# ------------------------------------------------------------------------------------------ skinny layers
# First layer (K = obs_dim <= 24) and output layer (N <= 8) of the MLPs (csrc/skinny.cu).  The weight / bias gradients
# are per-CTA slabs in a scratch buffer, then a slab sum: the plain entry points launch both kernels, the *_partial
# ones only the first and skinny_reduce_jobs sums the slabs of up to 8 jobs in one launch.
def skinny_tn_scratch_floats(M, H, K):
    return int(_lib.load().trl_skinny_tn_scratch_floats(int(M), int(H), int(K)))


def skinny_dgrad_act_scratch_floats(M, H):
    return int(_lib.load().trl_skinny_dgrad_act_scratch_floats(int(M), int(H)))


def skinny_k_fwd(x, w, bias, act, out=None):
    """out (M,H) = act(x (M,K) @ w (H,K)^T + bias)."""
    M, K = x.shape
    H = w.shape[0]
    if out is None:
        out = torch.empty(M, H, dtype=F32, device=x.device)
    _lib.call("trl_skinny_k_fwd", x, w, bias, out, M, K, H, int(act), _stream())
    return out


def skinny_n_fwd(x, w, bias, out=None):
    """out (M,N) = x (M,H) @ w (N,H)^T + bias."""
    M, H = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty(M, N, dtype=F32, device=x.device)
    _lib.call("trl_skinny_n_fwd", x, w, bias, out, M, H, N, _stream())
    return out


def skinny_n_dgrad(g, w, out=None):
    """out (M,H) = g (M,N) @ w (N,H)."""
    M = g.shape[0]
    N, H = w.shape
    if out is None:
        out = torch.empty(M, H, dtype=F32, device=g.device)
    _lib.call("trl_skinny_n_dgrad", g, w, out, M, H, N, _stream())
    return out


def skinny_tn(a, b, out, colsum, out_transposed, scratch):
    """out = a^T @ b for a (M,H), b (M,K) ((H,K), or (K,H) when out_transposed) [+ colsum (K) = colsum(b)];
    scratch: skinny_tn_scratch_floats(M, H, K) floats."""
    M, H = a.shape
    K = b.shape[1]
    _lib.call("trl_skinny_tn", a, b, out, colsum, M, H, K, int(bool(out_transposed)), scratch, _stream(), kernels=2)
    return out


def skinny_act_wgrad(g, y, x, dw, db, act, scratch):
    """The first layer's dW (H,K) = (g * act'(y))^T x and db = colsum(g * act'(y)) in one pass over g and y (M,H);
    scratch: skinny_tn_scratch_floats(M, H, K) floats."""
    M, H = y.shape
    K = x.shape[1]
    _lib.call("trl_skinny_act_wgrad", g, y, x, dw, db, M, H, K, int(act), scratch, _stream(), kernels=2)


def skinny_act_wgrad_partial(g, y, x, act, scratch):
    """The slabs of skinny_act_wgrad (reduce job kind 1)."""
    M, H = y.shape
    K = x.shape[1]
    _lib.call("trl_skinny_act_wgrad_partial", g, y, x, M, H, K, int(act), scratch, _stream())


def skinny_reduce_jobs(jobs):
    """The slab sums of up to 8 jobs (kind, scratch, out, colsum, M, H, K, out_transposed) in one launch: kind 0 =
    skinny_tn's slabs (colsum None or (K); skinny_n_dgrad_act_wgrad_partial's w_scratch), 1 = skinny_act_wgrad_partial
    (colsum = db (H)), 2 = skinny_n_dgrad_act_wgrad_partial's db_scratch (colsum = db (H), out None)."""
    n = len(jobs)
    assert n <= 8
    ci = ctypes.c_int
    _lib.call("trl_skinny_reduce_jobs", n, (ci * n)(*[j[0] for j in jobs]), [j[1] for j in jobs],
              [j[2] for j in jobs], [j[3] for j in jobs], (ctypes.c_int64 * n)(*[j[4] for j in jobs]),
              (ci * n)(*[j[5] for j in jobs]), (ci * n)(*[j[6] for j in jobs]), (ci * n)(*[j[7] for j in jobs]),
              _stream(), kernels=int(n > 0))


# ------------------------------------------------------------------------------------------ K1 synthetic envs
def synth_env_num_ctas(N):
    return int(_lib.load().trl_synth_env_num_ctas(int(N)))


def synth_env_seed(seeds, episode, seed, n_total, first_env):
    """VecEnv.seed: env i of this shard gets seed * n_total + first_env + i; episode counters restart."""
    _lib.call("trl_synth_env_seed", seeds, episode, seeds.numel(), int(seed) & 0xFFFFFFFF, int(n_total) & 0xFFFFFFFF,
              int(first_env) & 0xFFFFFFFF, _stream())


def synth_env_reset(state, elapsed, episode, seeds, mask, init_scale):
    """New episodes for every env (mask None) or the envs whose uint8 mask is set; state (N, o)."""
    N, o = state.shape
    _lib.call("trl_synth_env_reset", state, elapsed, episode, seeds, mask, N, o, float(init_scale), _stream())


def synth_env_step(state, actions, A, B, c, lb, ub, elapsed, step_count, reward, done, time_limit, partial, batch_sums,
                   norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, rho, eta, ctrl_cost, term_thr,
                   reward_scale, max_episode_steps, max_episode_frames, merge_stats):
    """One step of all N envs (csrc/env_step.cu): state (N, o) in place, actions (N, a).  partial / batch_sums /
    norm_*: the observation-normaliser moments (all None: not estimated); step_count / t_ptr: the collector's step
    counters and ring row (None outside a collector)."""
    N, o = state.shape
    _lib.call("trl_synth_env_step", state, actions, A, B, c, lb, ub, elapsed, step_count, reward, done, time_limit,
              partial, batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, N, o,
              actions.numel() // N, float(rho), float(eta), float(ctrl_cost), float(term_thr), float(reward_scale),
              int(max_episode_steps), int(max_episode_frames), int(bool(merge_stats)), _stream())


def cartpole_num_ctas(N):
    return int(_lib.load().trl_cartpole_num_ctas(int(N)))


def cartpole_step(state, actions, elapsed, step_count, reward, done, time_limit, action_error, partial, batch_sums,
                  norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, reward_scale, max_episode_steps,
                  max_episode_frames, merge_stats):
    """One CartPole step of all N envs (csrc/cartpole.cu): state (N, 4) in place, actions (N) 0.0 / 1.0 (anything else
    sets action_error (1) int32).  partial / batch_sums / norm_*: the observation-normaliser moments (all None: not
    estimated); step_count / t_ptr: the collector's step counters and ring row (None outside a collector)."""
    N = state.shape[0]
    if state.dim() != 2 or state.shape[1] != 4:
        raise ValueError("cartpole_step: state must be (N, 4), got %s" % (tuple(state.shape),))
    if actions.numel() != N:
        raise ValueError("cartpole_step: one action per env expected, got %d for %d envs" % (actions.numel(), N))
    _lib.call("trl_cartpole_step", state, actions, elapsed, step_count, reward, done, time_limit, action_error, partial,
              batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, N, float(reward_scale),
              int(max_episode_steps), int(max_episode_frames), int(bool(merge_stats)), _stream(), kernels=int(N > 0))


def pendulum_num_ctas(N):
    return int(_lib.load().trl_pendulum_num_ctas(int(N)))


def pendulum_step(phys, obs, actions, elapsed, step_count, reward, done, time_limit, action_error, partial, batch_sums,
                  norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, reward_scale, max_episode_steps,
                  max_episode_frames, merge_stats):
    """One Pendulum-v1 step of all N envs (csrc/pendulum.cu): phys (N, 2) fp64 and obs (N, 3) in place, actions (N) in
    [-1, 1] (a non-finite one sets action_error (1) int32).  partial / batch_sums / norm_*: the observation-normaliser
    moments (all None: not estimated); step_count / t_ptr: the collector's step counters and ring row (None outside a
    collector)."""
    _env_step("pendulum_step", 2, 3, phys, obs, actions, elapsed, step_count, reward, done, time_limit, action_error,
              partial, batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, reward_scale,
              max_episode_steps, max_episode_frames, merge_stats)


def pendulum_reset(phys, obs, elapsed, episode, seeds, mask=None, step_count=None, next_norm=None, cur_ob=None,
                   any_reset=None, t_ptr=None, norm_mean=None, norm_var=None, clip=10.0, raw_obs_after_reset=True):
    """New Pendulum episodes for every env (mask and step_count None), the envs of the uint8 `mask`, or those whose
    int32 `step_count` is 0 (the collector's path).  With `cur_ob` the next observation of every env is written there
    as collect_finalize writes it (next_norm / any_reset / t_ptr / norm_* / clip / raw_obs_after_reset)."""
    _env_reset("pendulum_reset", 2, 3, phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob,
               any_reset, t_ptr, norm_mean, norm_var, clip, raw_obs_after_reset)


def _check_phys_obs(fn, phys, obs, P, D):
    N = phys.shape[0]
    if phys.dim() != 2 or phys.shape[1] != P or tuple(obs.shape) != (N, D):
        raise ValueError("%s: phys must be (N, %d) and obs (N, %d), got %s and %s"
                         % (fn, P, D, tuple(phys.shape), tuple(obs.shape)))
    return N


def _env_step(fn, P, D, phys, obs, actions, elapsed, step_count, reward, done, time_limit, action_error, partial,
              batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, reward_scale, max_episode_steps,
              max_episode_frames, merge_stats, *extra):
    """The step of an env with an fp64 state (N, P), an fp32 observation (N, D) and one action per env."""
    N = _check_phys_obs(fn, phys, obs, P, D)
    if actions.numel() != N:
        raise ValueError("%s: one action per env expected, got %d for %d envs" % (fn, actions.numel(), N))
    _lib.call("trl_" + fn, phys, obs, actions, elapsed, step_count, reward, done, time_limit, action_error, partial,
              batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, N, float(reward_scale),
              int(max_episode_steps), int(max_episode_frames), int(bool(merge_stats)), *extra, _stream(),
              kernels=int(N > 0))


def _env_reset(fn, P, D, phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob, any_reset, t_ptr,
               norm_mean, norm_var, clip, raw_obs_after_reset):
    """The own reset of an env with an fp64 state (N, P) and an fp32 observation (N, D), as pendulum_reset."""
    N = _check_phys_obs(fn, phys, obs, P, D)
    if mask is not None and step_count is not None:
        raise ValueError("%s: select envs by mask or by step_count, not both" % fn)
    if cur_ob is not None and (step_count is None or next_norm is None or any_reset is None or t_ptr is None):
        raise ValueError("%s: cur_ob needs step_count, next_norm, any_reset and t_ptr" % fn)
    _lib.call("trl_" + fn, phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob, any_reset, t_ptr,
              norm_mean, norm_var, N, float(clip), int(bool(raw_obs_after_reset)), _stream(), kernels=int(N > 0))


def acrobot_num_ctas(N):
    return int(_lib.load().trl_acrobot_num_ctas(int(N)))


def acrobot_step(phys, obs, actions, elapsed, step_count, reward, done, time_limit, action_error, partial, batch_sums,
                 norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, reward_scale, max_episode_steps,
                 max_episode_frames, merge_stats):
    """One Acrobot-v1 step of all N envs (csrc/acrobot.cu): phys (N, 4) fp64 and obs (N, 6) in place, actions (N) 0.0 /
    1.0 / 2.0 (anything else sets action_error (1) int32).  partial / batch_sums / norm_*: the observation-normaliser
    moments (all None: not estimated); step_count / t_ptr: the collector's step counters and ring row (None outside a
    collector)."""
    _env_step("acrobot_step", 4, 6, phys, obs, actions, elapsed, step_count, reward, done, time_limit, action_error,
              partial, batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, reward_scale,
              max_episode_steps, max_episode_frames, merge_stats)


def acrobot_reset(phys, obs, elapsed, episode, seeds, mask=None, step_count=None, next_norm=None, cur_ob=None,
                  any_reset=None, t_ptr=None, norm_mean=None, norm_var=None, clip=10.0, raw_obs_after_reset=True):
    """New Acrobot episodes, selected and written as pendulum_reset does."""
    _env_reset("acrobot_reset", 4, 6, phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob,
               any_reset, t_ptr, norm_mean, norm_var, clip, raw_obs_after_reset)


def mountain_car_num_ctas(N):
    return int(_lib.load().trl_mountain_car_num_ctas(int(N)))


def mountain_car_step(phys, obs, actions, elapsed, step_count, reward, done, time_limit, action_error, partial,
                      batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr, reward_scale,
                      max_episode_steps, max_episode_frames, merge_stats, continuous):
    """One Mountain Car step of all N envs (csrc/mountain_car.cu): phys (N, 2) fp64 and obs (N, 2) in place.
    MountainCar-v0 (continuous False): actions (N) 0.0 / 1.0 / 2.0; MountainCarContinuous-v0: actions (N) in [-1, 1]; a
    refused action sets action_error (1) int32.  Other arguments as acrobot_step."""
    _env_step("mountain_car_step", 2, 2, phys, obs, actions, elapsed, step_count, reward, done, time_limit,
              action_error, partial, batch_sums, norm_mean, norm_var, norm_count, ticket, any_reset, t_ptr,
              reward_scale, max_episode_steps, max_episode_frames, merge_stats, int(bool(continuous)))


def mountain_car_reset(phys, obs, elapsed, episode, seeds, mask=None, step_count=None, next_norm=None, cur_ob=None,
                       any_reset=None, t_ptr=None, norm_mean=None, norm_var=None, clip=10.0, raw_obs_after_reset=True):
    """New Mountain Car episodes (both ids), selected and written as pendulum_reset does."""
    _env_reset("mountain_car_reset", 2, 2, phys, obs, elapsed, episode, seeds, mask, step_count, next_norm, cur_ob,
               any_reset, t_ptr, norm_mean, norm_var, clip, raw_obs_after_reset)


def synth_atari_reset(obs, latent, elapsed, episode, seeds, mask=None, zero_is_mask=None, episode_bias=0, bump=1):
    """New episodes for every env, the envs of the uint8 `mask`, or those whose int32 `zero_is_mask` entry is 0."""
    _lib.call("trl_synth_atari_reset", obs, latent, elapsed, episode, seeds, mask, zero_is_mask, int(episode_bias),
              int(bump), obs.shape[0], _stream())


def synth_atari_step(obs, latent, actions, elapsed, reward, done, time_limit, max_steps):
    """One step of all envs: obs (N, 4, 84, 84) uint8 in place, actions (N) float action indices."""
    _lib.call("trl_synth_atari_step", obs, latent, actions, elapsed, reward, done, time_limit, obs.shape[0],
              int(max_steps), _stream())


def u8_to_f32(x, scale, out=None):
    """out = x * scale as float32."""
    if out is None:
        out = torch.empty(x.shape, dtype=F32, device=x.device)
    assert out.numel() == x.numel()
    _lib.call("trl_u8_to_f32", x, out, x.numel(), float(scale), _stream())
    return out


def atari_warp_stack(frames, stack, tab_i, tab_w, env_idx=None, fresh=None):
    """WarpFrame + FrameStack in one launch (csrc/atari_frames.cu): frames (M, H, W, 3) uint8 RGB -> gray, 84x84
    INTER_AREA -> the (N, C, 84, 84) uint8 stack of env env_idx[m] (None: env m), filling every slot of a fresh env
    (fresh None: all envs fresh) and shifting in the new frame for the others.  tab_i / tab_w: area_tables(H, W) of
    env/atari_host.py on the device.  One launch, none when M == 0."""
    M, H, W, three = frames.shape
    N, C = stack.shape[:2]
    if three != 3 or tuple(stack.shape[2:]) != (84, 84):
        raise ValueError("atari_warp_stack: frames (M, H, W, 3) and stack (N, C, 84, 84), got %s and %s"
                         % (tuple(frames.shape), tuple(stack.shape)))
    _lib.call("trl_atari_warp_stack", frames, env_idx, fresh, stack, tab_i, tab_w, M, N, H, W, C, _stream(),
              kernels=int(M > 0))


def u8_lut_f32(x, lut, out=None):
    """out = lut[x] as float32 (lut: 256 floats on the device).  One launch."""
    if out is None:
        out = torch.empty(x.shape, dtype=F32, device=x.device)
    if out.numel() != x.numel() or lut.numel() != 256:
        raise ValueError("u8_lut_f32: out must match x and lut must hold 256 entries")
    _lib.call("trl_u8_lut_f32", x, out, x.numel(), lut, _stream(), kernels=int(x.numel() > 0))
    return out


# ------------------------------------------------------------------------------------------ frame-stack ring
def frame_ring_write(stack, ring, top, age=None, elapsed=None, hist=None, hist_count=None, size=None):
    """Newest frame of every env's (N, C, ...) uint8 stack -> row *top of ring (T, N, F); age / elapsed: also the age
    byte min(elapsed, C-1); hist / hist_count / size: the (C-1)-deep history of overwritten frames (csrc/frames.cu)."""
    T, N, F = ring.shape
    C = stack.shape[1]
    assert stack.numel() == N * C * F
    _lib.call("trl_frame_ring_write", stack, ring, age, elapsed, hist, hist_count, top, size, N, C, F, T, C - 1,
              _stream())


def frame_hist_advance(hist_count, size, T):
    """Once per step after the step's frame_ring_write calls."""
    _lib.call("trl_frame_hist_advance", hist_count, size, int(T), _stream())


def frame_stack_gather(obs_last, next_last, age, hist, hist_count, idx, rows, top, size, scale, out_obs, out_next,
                       pos=None):
    """out_obs / out_next (rows*N, C, ...) f32 = scale * the frame stacks of ring rows idx[pos*rows + k] (pos None:
    idx[k]), rebuilt from the de-duplicated ring: obs_last / next_last (T, N, F), hist (C-1, N, F)."""
    T, N, F = obs_last.shape
    C = hist.shape[0] + 1
    _lib.call("trl_frame_stack_gather", obs_last, next_last, age, hist, hist_count, idx, pos, int(rows), top, size, N,
              C, F, T, float(scale), out_obs, out_next, _stream(), kernels=int(rows > 0))


# ------------------------------------------------------------------------------------------ K12 peer communication
# Host-side management of the peer-mapped communication blocks (no kernel launches) and the collectives of
# csrc/comm.cu.  peer_* / flags: host arrays of `world` device pointers (distributed.PeerComm.region).
def comm_sizes():
    """(flag pad bytes, cudaIpc handle bytes)."""
    lib = _lib.load()
    return int(lib.trl_comm_flag_bytes()), int(lib.trl_comm_ipc_handle_bytes())


def comm_scratch_doubles(nseg):
    return int(_lib.load().trl_comm_scratch_doubles(int(nseg)))


def comm_ll_recv_bytes(world, nmax):
    return int(_lib.load().trl_comm_ll_recv_bytes(int(world), int(nmax)))


def comm_alloc(nbytes):
    """Device address of a new zeroed communication block of `nbytes`."""
    ptr = ctypes.c_void_p()
    _lib.check(_lib.load().trl_comm_alloc(int(nbytes), ctypes.byref(ptr)), "trl_comm_alloc")
    return ptr.value


def comm_ipc_get(ptr):
    """The cudaIpc handle (bytes) of a block made by comm_alloc."""
    handle = ctypes.create_string_buffer(comm_sizes()[1])
    _lib.check(_lib.load().trl_comm_ipc_get(ptr, handle), "trl_comm_ipc_get")
    return handle.raw


def comm_ipc_open(handle):
    """This process's device address of a peer's block, from its comm_ipc_get handle."""
    ptr = ctypes.c_void_p()
    _lib.check(_lib.load().trl_comm_ipc_open(ctypes.create_string_buffer(bytes(handle), len(handle)),
                                             ctypes.byref(ptr)), "trl_comm_ipc_open")
    return ptr.value


def allreduce_grad(peer_data, flags, rank, world, out, seg_begin, nseg, mask, sumsq3, step_counts, betas, scratch,
                   ticket, seq, zero_local=True):
    """out = the sum over ranks of the peers' flat gradients, with what grad_sumsq computes for it; zero_local: this
    rank's gradient is zeroed once every peer has read it."""
    _lib.call("trl_allreduce_grad", peer_data, flags, int(rank), int(world), out, out.numel(), seg_begin, int(nseg),
              int(mask), sumsq3, step_counts, float(betas[0]), float(betas[1]), scratch, ticket, seq,
              int(bool(zero_local)), _stream())


def allreduce_f64(peer_data, flags, rank, world, out, n, gather, seq):
    """out = the sum over ranks (gather: the (world, n) stack) of the first n doubles of the peers' regions."""
    _lib.call("trl_allreduce_f64", peer_data, flags, int(rank), int(world), out, int(n), int(bool(gather)), seq,
              _stream())
    return out


def allreduce_f64_ll(local, peer_recv, rank, world, out, n, nmax, gather, ll_seq):
    """allreduce_f64 for n <= nmax doubles of `local` in one NVLink traversal (flag-carrying packets)."""
    _lib.call("trl_allreduce_f64_ll", local, peer_recv, int(rank), int(world), out, int(n), int(nmax),
              int(bool(gather)), ll_seq, _stream())
    return out
