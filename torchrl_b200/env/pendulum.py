"""Device-resident Pendulum-v1 with the vec-env API of SynthVecEnv.

Stands where ``NormAct(VecEnv(gym.make("Pendulum-v1")))`` stands in the reference (/root/reference/torchrl/env/get_env.py:53,
:70-78, env/continuous_wrapper.py:18-20): gym's Pendulum-v1 for all N envs in one launch (csrc/pendulum.cu, defined in
oracle/pendulum.py).  Actions are in [-1, 1] and map to a torque in [-2, 2]; observations are (cos theta, sin theta,
theta_dot) in fp32; the reward is minus gym's cost; there is no terminal state, every episode ends at the 200-step time
limit, so all envs run in lock step.  The physical state (theta, theta_dot) is fp64 (`phys`).  Resets draw theta from
U(-pi, pi) and theta_dot from U(-1, 1) with the counter hash of the synthetic envs; the collector's partial reset is the
env's own kernel (`resets_itself`), launched right after the finalize kernel inside the captured step.

Only v1 is served: Pendulum-v0 moves the angle with the unclipped velocity, which this kernel does not compute.
"""
import numpy as np
import torch

from .. import ops
from ..spaces import Box
from .synth import DeviceNormalizer, SynthVecEnv

F32, F64, U8, I32 = torch.float32, torch.float64, torch.uint8, torch.int32

ENV_ID = "Pendulum-v1"
MAX_EPISODE_STEPS = 200
MAX_SPEED = 8.0


def is_pendulum(env_id):
    return env_id == ENV_ID


class PendulumVecEnv(SynthVecEnv):
    """N Pendulum-v1 envs on one GPU.  env_param / first_env / total_envs / dist: as SynthVecEnv."""

    lockstep = True
    # the collector's finalize kernel leaves this env's counters and observation to `collector_reset`
    resets_itself = True

    def __init__(self, env_nums, env_param=None, device="cuda", first_env=0, total_envs=None, max_episode_steps=None):
        env_param = dict(env_param or {})
        self.env_id = ENV_ID
        self.env_nums = int(env_nums)
        self.device = torch.device(device)
        self.obs_dim, self.act_dim = 3, 1
        self.first_env = int(first_env)
        self.total_envs = int(total_envs) if total_envs is not None else self.env_nums
        self._max_episode_steps = int(max_episode_steps or MAX_EPISODE_STEPS)
        self._reward_scale = env_param.get("reward_scale", 1)
        self.obs_norm = bool(env_param.get("obs_norm", False))
        self.training = True
        self.observation_space = Box(np.array([-1.0, -1.0, -MAX_SPEED]), np.array([1.0, 1.0, MAX_SPEED]))
        self.action_space = Box(-1.0, 1.0, shape=(1,))
        N, o, dev = self.env_nums, self.obs_dim, self.device
        self.phys = torch.zeros(N, 2, dtype=F64, device=dev)        # theta, theta_dot
        self.state = torch.zeros(N, o, dtype=F32, device=dev)       # raw observation
        self.elapsed = torch.zeros(N, dtype=I32, device=dev)
        self.episode = torch.zeros(N, dtype=I32, device=dev)
        self.seeds = torch.zeros(N, dtype=I32, device=dev)
        self.reward = torch.zeros(N, dtype=F32, device=dev)
        self.done = torch.zeros(N, dtype=U8, device=dev)
        self.time_limit = torch.zeros(N, dtype=U8, device=dev)
        self.action_error = torch.zeros(1, dtype=I32, device=dev)
        self.obs_out = torch.zeros(N, o, dtype=F32, device=dev)     # what step() returns (normalised if obs_norm)
        self._partial = torch.zeros(ops.pendulum_num_ctas(N), 2 * o, dtype=F64, device=dev)
        self.batch_sums = torch.zeros(2 * o, dtype=F64, device=dev)
        self._ticket = torch.zeros(1, dtype=I32, device=dev)
        self.any_reset = torch.zeros(2, dtype=I32, device=dev)
        self._obs_normalizer = DeviceNormalizer((o,), device=dev) if self.obs_norm else None
        self._obs = None
        self._host_elapsed = 0
        self._host_mirror_ok = True
        self._dist = None
        self._sums_red = None
        self.seed(0)

    def _reset_kernel(self, mask):
        ops.pendulum_reset(self.phys, self.state, self.elapsed, self.episode, self.seeds, mask=mask)

    def collector_reset(self, step_count, cur_ob, t_ptr, raw_obs_after_reset):
        """The collector's partial reset (one launch, capturable): new episodes for the envs whose `step_count` the
        finalize kernel just zeroed, and their next observation in `cur_ob` by collect_finalize's rules."""
        nrm = self._obs_normalizer if self.obs_norm else None
        ops.pendulum_reset(self.phys, self.state, self.elapsed, self.episode, self.seeds, step_count=step_count,
                           next_norm=self.obs_out, cur_ob=cur_ob, any_reset=self.any_reset, t_ptr=t_ptr,
                           norm_mean=None if nrm is None else nrm._mean, norm_var=None if nrm is None else nrm._var,
                           clip=10.0 if nrm is None else nrm.clip, raw_obs_after_reset=raw_obs_after_reset)

    def launch_step(self, actions, step_count=None, max_episode_frames=0, t_ptr=None):
        """Advance all envs one step: phys/state/reward/done/time_limit staging buffers are updated and, with obs_norm,
        `obs_out` receives what env.step would return.  No host sync; a non-finite action is reported by
        `check_actions`."""
        update = self.obs_norm and self.training and self._obs_normalizer.should_estimate
        nrm = self._obs_normalizer
        distributed = self.dist is not None and self.dist.active
        rs = float(self._reward_scale) if self.training else 1.0
        moments = (self._partial, self.batch_sums, nrm._mean, nrm._var, nrm._count) if update else (None,) * 5
        ops.pendulum_step(self.phys, self.state, actions.reshape(-1), self.elapsed, step_count, self.reward, self.done,
                          self.time_limit, self.action_error, *moments, self._ticket, self.any_reset, t_ptr, rs,
                          self._max_episode_steps, int(max_episode_frames) if step_count is not None else (1 << 30),
                          update and not distributed)
        if update and distributed:
            ops.obs_norm_merge(self._reduce_sums(), self.total_envs, nrm._mean, nrm._var, nrm._count)
        if self.obs_norm:
            ops.obs_norm_filt(self.state, nrm._mean, nrm._var, nrm.clip, self.obs_out)
        return self.obs_out

    def check_actions(self):
        """Raise if any step since the last check received a non-finite action (one host sync)."""
        if int(self.action_error.item()) != 0:
            self.action_error.zero_()
            raise ValueError("%s takes finite actions in [-1, 1]; a NaN or an infinity was passed to step()"
                             % self.env_id)

    def step(self, actions):
        """obs (N,3), reward (N,1), done (N,1) bool, {'time_limit': (N,) bool} -- device tensors."""
        actions = torch.as_tensor(actions, device=self.device).reshape(-1).to(F32).contiguous()
        if actions.numel() != self.env_nums:
            raise ValueError("%s.step: %d actions for %d envs" % (self.env_id, actions.numel(), self.env_nums))
        self.launch_step(actions)
        if not self.obs_norm:
            self.obs_out.copy_(self.state)
        self.check_actions()
        infos = {"time_limit": self.time_limit.bool()}
        return self.obs_out, self.reward.unsqueeze(-1), self.done.bool().unsqueeze(-1), infos
