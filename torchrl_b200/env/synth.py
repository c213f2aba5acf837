"""Device-resident vectorised envs with the reference's vec-env API: `DeviceVecEnv`, the base of the state-vector
device envs (synthetic, CartPole, Pendulum, Acrobot, Mountain Car), `SelfResettingVecEnv`, the base of those whose
observation is not their state (Pendulum, Acrobot, Mountain Car), and the synthetic env itself.

Stands where ``NormObs(VecEnv(...))`` / ``NormObs(SubProcVecEnv(...))`` stand in the reference
(/root/reference/torchrl/env/get_env.py:70-87): same methods and attributes
(``env_nums``, ``observation_space``, ``action_space``, ``reset``, ``step``, ``partial_reset``,
``seed``, ``train``/``eval``, ``close``, ``_obs_normalizer``, ``_reward_scale``), but all N envs
advance in one CUDA launch and every returned array is a device tensor.
"""
import copy

import numpy as np
import torch

from .. import ops
from ..spaces import Box
from . import synth_spec as spec

F32, F64, U8, I32 = torch.float32, torch.float64, torch.uint8, torch.int32


class DeviceNormalizer:
    """Running mean/var observation normaliser with fp64 state on the device.

    Mirrors Normalizer (/root/reference/torchrl/env/base_wrapper.py:63-100): attributes
    ``_mean``, ``_var``, ``_count``, ``clip``, ``should_estimate``; pickles to NumPy so the
    reference's ``_obs_normalizer_{epoch}.pkl`` snapshot format keeps working
    (/root/reference/torchrl/algo/rl_algo.py:83-89).
    """

    def __init__(self, shape, clip=10., device="cuda"):
        self.shape = tuple(shape) if not isinstance(shape, int) else (shape,)
        dim = int(np.prod(self.shape))
        self._mean = torch.zeros(dim, dtype=F64, device=device)
        self._var = torch.ones(dim, dtype=F64, device=device)
        self._count = torch.full((1,), 1e-4, dtype=F64, device=device)
        self.clip = clip
        self.should_estimate = True

    def stop_update_estimate(self):
        self.should_estimate = False

    def update_estimate(self, data):
        if not self.should_estimate:
            return
        data = data.reshape(-1, self._mean.numel()).contiguous().float()
        sums = ops.obs_norm_moments(data)
        ops.obs_norm_merge(sums, data.shape[0], self._mean, self._var, self._count)

    def filt(self, raw, out=None):
        shp = raw.shape
        res = ops.obs_norm_filt(raw.reshape(-1, self._mean.numel()).contiguous().float(), self._mean, self._var,
                                self.clip, out)
        return res.reshape(shp)

    def inverse(self, raw):
        return raw * torch.sqrt(self._var).float() + self._mean.float()

    def to(self, device):
        self._mean, self._var, self._count = (t.to(device) for t in (self._mean, self._var, self._count))
        return self

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_mean"] = self._mean.cpu().numpy()
        d["_var"] = self._var.cpu().numpy()
        d["_count"] = float(self._count.item())
        return d

    def __setstate__(self, d):
        self.__dict__.update(d)
        dev = "cuda" if torch.cuda.is_available() else "cpu"
        self._mean = torch.as_tensor(np.asarray(d["_mean"], dtype=np.float64)).reshape(-1).to(dev)
        self._var = torch.as_tensor(np.asarray(d["_var"], dtype=np.float64)).reshape(-1).to(dev)
        self._count = torch.full((1,), float(d["_count"]), dtype=F64, device=dev)

    def __deepcopy__(self, memo):
        new = DeviceNormalizer.__new__(DeviceNormalizer)
        new.__dict__.update({k: v for k, v in self.__dict__.items() if not torch.is_tensor(v)})
        new._mean, new._var, new._count = self._mean.clone(), self._var.clone(), self._count.clone()
        return new


class DeviceVecEnv:
    """What the state-vector device envs share: N envs whose raw observation is the fp32 `state` (N, obs_dim), stepped
    by one kernel launch that also keeps the TimeLimit counters, the collector's reset flag and NormObs's batch moments.

    env_param: {"reward_scale": float, "obs_norm": bool} (the reference's "env" config section).
    first_env / total_envs: global index range of this shard (multi-GPU: rank g owns
    [g*N, (g+1)*N) of total_envs; seeds follow VecEnv.seed with the GLOBAL index so the union
    over ranks equals the single-process env set).
    A subclass sets its spaces and launches its kernels in `_step_kernel` (and `_reset_kernel` unless the default reset
    below is its own).
    """

    # half-width of the uniform reset distribution (the collector's in-kernel partial reset reads it too)
    init_scale = spec.INIT_SCALE
    # host mirror of `elapsed` valid (read while lockstep; reset() restores it, partial_reset() invalidates it)
    _host_mirror_ok = True
    # check_actions' message (%s: env_id) for an env whose kernel flags the actions it refuses in `action_error`
    action_error_msg = None

    def __init__(self, env_id, env_nums, env_param, device, first_env, total_envs, max_episode_steps, obs_dim, act_dim,
                 num_ctas):
        env_param = dict(env_param or {})
        self.env_id = env_id
        self.env_nums = int(env_nums)
        self.device = torch.device(device)
        self.obs_dim, self.act_dim = obs_dim, act_dim
        self.first_env = int(first_env)
        self.total_envs = int(total_envs) if total_envs is not None else self.env_nums
        self._max_episode_steps = int(max_episode_steps)
        self._reward_scale = env_param.get("reward_scale", 1)
        self.obs_norm = bool(env_param.get("obs_norm", False))
        self.training = True
        N, o, dev = self.env_nums, obs_dim, self.device
        self.state = torch.zeros(N, o, dtype=F32, device=dev)       # raw observation
        self.elapsed = torch.zeros(N, dtype=I32, device=dev)
        self.episode = torch.zeros(N, dtype=I32, device=dev)
        self.seeds = torch.zeros(N, dtype=I32, device=dev)
        self.reward = torch.zeros(N, dtype=F32, device=dev)
        self.done = torch.zeros(N, dtype=U8, device=dev)
        self.time_limit = torch.zeros(N, dtype=U8, device=dev)
        if self.action_error_msg is not None:
            self.action_error = torch.zeros(1, dtype=I32, device=dev)
        self.obs_out = torch.zeros(N, o, dtype=F32, device=dev)     # what step() returns (normalised if obs_norm)
        self._partial = torch.zeros(num_ctas, 2 * o, dtype=F64, device=dev)
        self.batch_sums = torch.zeros(2 * o, dtype=F64, device=dev)
        self._ticket = torch.zeros(1, dtype=I32, device=dev)
        self.any_reset = torch.zeros(2, dtype=I32, device=dev)
        self._obs_normalizer = DeviceNormalizer((o,), device=dev) if self.obs_norm else None
        self._obs = None
        self._host_elapsed = 0
        # stats merge happens in-kernel; with a DataParallelContext the batch sums are all-reduced
        # over ranks first and merged by a separate launch (global statistics, SURVEY.md 8(e))
        self._dist = None
        self._sums_red = None
        self.seed(0)

    @property
    def dist(self):
        return self._dist

    @dist.setter
    def dist(self, ctx):
        """Attach a DataParallelContext.  With PeerComm (distributed.py) the per-step batch sums move into a
        peer-mapped region so that csrc/comm.cu sums them over ranks in one small kernel (no NCCL launch per step).
        Must happen before the collector captures its step graph."""
        self._dist = ctx
        if ctx is not None and getattr(ctx, "active", False) and getattr(ctx, "peer", None) is not None:
            local, _ = ctx.peer.region("obs_sums", 8 * self.batch_sums.numel(), torch.float64)
            self.batch_sums = local[:self.batch_sums.numel()]
            self.batch_sums.zero_()
            self._sums_red = torch.zeros_like(self.batch_sums)

    def _reduce_sums(self):
        """Sum of `batch_sums` over ranks (identical on every rank)."""
        if self._sums_red is not None:
            return self._dist.peer.all_reduce_f64("obs_sums", self.batch_sums.numel(), self._sums_red)
        return self._dist.all_reduce_sum_(self.batch_sums)

    # ------------------------------------------------------------------ reference API
    def train(self):
        self.training = True

    def eval(self):
        self.training = False

    def close(self):
        pass

    def render(self, *a, **k):
        return None

    def seed(self, seed):
        ops.synth_env_seed(self.seeds, self.episode, seed, self.total_envs, self.first_env)

    def _reset_kernel(self, mask):
        """Every state component from U(-init_scale, init_scale) by the counter hash, as collect_finalize resets."""
        ops.synth_env_reset(self.state, self.elapsed, self.episode, self.seeds, mask, self.init_scale)

    def _observe(self, update):
        """NormObs.observation (/root/reference/torchrl/env/base_wrapper.py:118-121)."""
        if not self.obs_norm:
            self.obs_out.copy_(self.state)
            return self.obs_out
        if update and self.training:
            if self.dist is not None and self.dist.active:
                ops.obs_norm_moments(self.state, self.batch_sums)
                sums = self._reduce_sums()
                nrm = self._obs_normalizer
                ops.obs_norm_merge(sums, self.total_envs, nrm._mean, nrm._var, nrm._count)
            else:
                self._obs_normalizer.update_estimate(self.state)
        return self._obs_normalizer.filt(self.state, out=self.obs_out)

    def reset(self, **kwargs):
        self._reset_kernel(None)
        self._host_elapsed = 0
        self._host_mirror_ok = True
        return self._observe(update=True)

    def partial_reset(self, index_mask, **kwargs):
        """Reset the masked envs and return the RAW observation of all envs -- the reference's
        NormObs does not wrap partial_reset, so VecEnv.partial_reset's un-normalised `_obs`
        comes back (/root/reference/torchrl/env/vecenv.py:47-51; SURVEY.md A.1)."""
        mask = torch.as_tensor(index_mask, device=self.device).reshape(-1).to(U8).contiguous()
        self._reset_kernel(mask)
        self._host_mirror_ok = False
        return self.state

    def launch_step(self, actions, step_count=None, max_episode_frames=0, t_ptr=None):
        """Advance all envs one step: the staging buffers (state, reward, done, time_limit) are updated and, with
        obs_norm, `obs_out` receives what env.step would return.  No host sync; an action the kernel refuses is
        reported by `check_actions`."""
        nrm = self._obs_normalizer
        update = self.obs_norm and self.training and nrm.should_estimate
        distributed = self.dist is not None and self.dist.active
        moments = (self._partial, self.batch_sums, nrm._mean, nrm._var, nrm._count) if update else (None,) * 5
        self._step_kernel(actions, step_count, moments, t_ptr, float(self._reward_scale) if self.training else 1.0,
                          int(max_episode_frames) if step_count is not None else (1 << 30), update and not distributed)
        if update and distributed:
            ops.obs_norm_merge(self._reduce_sums(), self.total_envs, nrm._mean, nrm._var, nrm._count)
        if self.obs_norm:
            ops.obs_norm_filt(self.state, nrm._mean, nrm._var, nrm.clip, self.obs_out)
        return self.obs_out

    def check_actions(self):
        """Raise if any step since the last check received an action the kernel refuses (one host sync, none for an
        env whose kernel accepts every action)."""
        if self.action_error_msg is not None and int(self.action_error.item()) != 0:
            self.action_error.zero_()
            raise ValueError(self.action_error_msg % self.env_id)

    def step(self, actions):
        """obs (N,o), reward (N,1), done (N,1) bool, {'time_limit': (N,) bool} -- device tensors."""
        actions = torch.as_tensor(actions, dtype=F32, device=self.device).reshape(-1)
        if actions.numel() != self.env_nums * self.act_dim:
            raise ValueError("%s.step: %d actions for %d envs" % (self.env_id, actions.numel(), self.env_nums))
        self.launch_step(actions.reshape(self.env_nums, self.act_dim).contiguous())
        if not self.obs_norm:
            self.obs_out.copy_(self.state)
        self.check_actions()
        infos = {"time_limit": self.time_limit.bool()}
        return self.obs_out, self.reward.unsqueeze(-1), self.done.bool().unsqueeze(-1), infos

    def __deepcopy__(self, memo):
        new = type(self).__new__(type(self))
        for k, v in self.__dict__.items():
            if k == "_dist":
                new.__dict__[k] = v                       # the job's communicator is shared, never copied
            elif torch.is_tensor(v):
                new.__dict__[k] = v.clone()
            else:
                new.__dict__[k] = copy.deepcopy(v, memo)
        return new


class SelfResettingVecEnv(DeviceVecEnv):
    """A state-vector device env whose observation is not its state: an fp64 physical state `phys` (N, phys_dim) beside
    the fp32 `state`, and its own reset kernel (`resets_itself`), which the collector launches right after the finalize
    kernel inside the captured step.  A subclass names its ops wrappers by their prefix in `kernels`
    (ops.<kernels>_step, _reset and _num_ctas) and, in `step_extra`, the attributes passed after the step's common
    arguments."""

    # the collector's finalize kernel leaves this env's counters and observation to `collector_reset`
    resets_itself = True
    kernels = None
    step_extra = ()

    def __init__(self, env_id, env_nums, env_param, device, first_env, total_envs, max_episode_steps, obs_dim,
                 phys_dim):
        super().__init__(env_id, env_nums, env_param, device, first_env, total_envs, max_episode_steps, obs_dim, 1,
                         getattr(ops, self.kernels + "_num_ctas")(int(env_nums)))
        self.phys = torch.zeros(self.env_nums, phys_dim, dtype=F64, device=self.device)

    def _reset_kernel(self, mask):
        getattr(ops, self.kernels + "_reset")(self.phys, self.state, self.elapsed, self.episode, self.seeds, mask=mask)

    def collector_reset(self, step_count, cur_ob, t_ptr, raw_obs_after_reset):
        """The collector's partial reset (one launch, capturable): new episodes for the envs whose `step_count` the
        finalize kernel just zeroed, and their next observation in `cur_ob` by collect_finalize's rules."""
        nrm = self._obs_normalizer if self.obs_norm else None
        getattr(ops, self.kernels + "_reset")(
            self.phys, self.state, self.elapsed, self.episode, self.seeds, step_count=step_count,
            next_norm=self.obs_out, cur_ob=cur_ob, any_reset=self.any_reset, t_ptr=t_ptr,
            norm_mean=None if nrm is None else nrm._mean, norm_var=None if nrm is None else nrm._var,
            clip=10.0 if nrm is None else nrm.clip, raw_obs_after_reset=raw_obs_after_reset)

    def _step_kernel(self, actions, step_count, moments, t_ptr, reward_scale, max_episode_frames, merge):
        getattr(ops, self.kernels + "_step")(
            self.phys, self.state, actions.reshape(-1), self.elapsed, step_count, self.reward, self.done,
            self.time_limit, self.action_error, *moments, self._ticket, self.any_reset, t_ptr, reward_scale,
            self._max_episode_steps, max_episode_frames, merge, *(getattr(self, k) for k in self.step_extra))


class SynthVecEnv(DeviceVecEnv):
    """N synthetic envs on one GPU: s' = rho * s + eta * tanh(s A + NormAct(u) B + c) (csrc/env_step.cu)."""

    def __init__(self, env_id, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None,
                 max_episode_steps=spec.MAX_EPISODE_STEPS):
        o, a, self.term_thr = spec.SPECS[env_id]
        super().__init__(env_id, env_nums, env_param, device, first_env, total_envs, max_episode_steps, o, a,
                         ops.synth_env_num_ctas(int(env_nums)))
        hi = np.full((o,), np.inf)
        self.observation_space = Box(-hi, hi)
        ub = np.ones((a,))
        self.action_space = Box(-ub, ub)
        # True when episode boundaries are a deterministic function of the step count
        self.lockstep = not np.isfinite(self.term_thr)
        A, B, c = spec.make_params(o, a)
        self.A = torch.from_numpy(A).to(self.device)
        self.B = torch.from_numpy(B).to(self.device)
        self.c = torch.from_numpy(c).to(self.device)
        self.lb = torch.full((a,), -1.0, dtype=F32, device=self.device)
        self.ub = torch.full((a,), 1.0, dtype=F32, device=self.device)

    def _step_kernel(self, actions, step_count, moments, t_ptr, reward_scale, max_episode_frames, merge):
        ops.synth_env_step(self.state, actions, self.A, self.B, self.c, self.lb, self.ub, self.elapsed, step_count,
                           self.reward, self.done, self.time_limit, *moments, self._ticket, self.any_reset, t_ptr,
                           spec.RHO, spec.ETA, spec.CTRL_COST,
                           float(self.term_thr) if np.isfinite(self.term_thr) else 3.0e38, reward_scale,
                           self._max_episode_steps, max_episode_frames, merge)
