"""Vectorised rollout collectors on the device (API of /root/reference/torchrl/collector/base.py).

One collector step = policy MLP (PyTorch) -> action sampling kernel -> batched env-step kernel
(+ observation-normaliser statistics) -> filter kernel -> finalize kernel (row store, timeout
bookkeeping, partial reset) -> device-side ring advance.  Nothing returns to the host inside
the T-step loop; the whole step is captured once in a CUDA graph and replayed for every row
(all row indices / RNG offsets are read from device memory, so graph arguments never change).
"""
import copy

import numpy as np
import torch

from .. import ops
from ..env import synth_spec
from ..networks import fused
from ..networks.nets import ZeroNet
from ..policies import distribution as D
from ..spaces import is_box

F32, F64, U8, I32 = torch.float32, torch.float64, torch.uint8, torch.int32


class VecCollector:
    """Off-policy collector (reference: VecCollector, collector/base.py:176-280; the base class
    BaseCollector.__init__ :10-55 supplies the constructor contract)."""

    on_policy = False

    def __init__(self, env, eval_env=None, pf=None, replay_buffer=None, epoch_frames=None, train_render=False, eval_episodes=1,
                 eval_render=False, device='cpu', max_episode_frames=999, use_cuda_graph=True,
                 reference_quirks=True):
        # `eval_env` is optional here (a copy of `env` is made): the reference's a2c / ddpg / dqn example scripts do not
        # pass one although its BaseCollector requires it (collector/base.py:13; SURVEY.md A.4)
        assert pf is not None and replay_buffer is not None and epoch_frames is not None, "pf, replay_buffer, epoch_frames"
        self.pf = pf
        self.replay_buffer = replay_buffer
        self.env = env
        self._host_env = bool(getattr(env, "host_bridge", False))
        self.env.train()
        self.continuous = is_box(self.env.action_space)
        self.train_render = train_render
        if eval_env is not None:
            self.eval_env = eval_env
        else:
            self.eval_env = copy.deepcopy(env)
            if hasattr(env, "_obs_normalizer"):
                self.eval_env._obs_normalizer = env._obs_normalizer
        self.eval_env._reward_scale = 1
        self.eval_episodes = eval_episodes
        self.eval_render = eval_render
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("torchrl_b200 collectors run on a CUDA device (there is no CPU path); got %r" % (device,))
        self.to(self.device)
        self.epoch_frames = epoch_frames
        self.sample_epoch_frames = epoch_frames // self.env.env_nums
        self.max_episode_frames = max_episode_frames
        self.use_cuda_graph = bool(use_cuda_graph)
        self.reference_quirks = bool(reference_quirks)
        # REINFORCE's value function is a ZeroNet: V = 0 needs no launches, `_values` rows stay zero
        self._has_vf = self.on_policy and not isinstance(getattr(self, "vf", None), ZeroNet)

        N = self.env.env_nums
        o = int(np.prod(self.env.observation_space.shape))
        a = self.env.action_space.shape[0] if self.continuous else 1
        self._N, self._o, self._a = N, o, a
        dev = self.device
        if getattr(self.env, "pixel", False):
            self.current_ob = self.env.reset()               # uint8 frame stack, updated in place by the env
        else:
            self.current_ob = torch.empty(N, o, dtype=F32, device=dev)
            self.current_ob.copy_(self.env.reset())
        self.current_step = torch.zeros(N, dtype=I32, device=dev)
        self.train_rew = torch.zeros(N, dtype=F64, device=dev)
        self._epoch_reward = torch.zeros(N, dtype=F64, device=dev)
        self._n_done = torch.zeros(1, dtype=I32, device=dev)
        self._nan_flag = torch.zeros(1, dtype=I32, device=dev)
        self._act = torch.zeros(N, a, dtype=F32, device=dev)
        self._value = torch.zeros(N, dtype=F32, device=dev) if self.on_policy else None
        self._v_next = torch.zeros(N, dtype=F32, device=dev) if self.on_policy else None
        self._eps = None
        self._eps_dev = None
        self._host_step = 0
        self._host_steps = np.zeros(N, dtype=np.int64)      # host mirror of current_step (host envs only)
        self._graphs = {}
        self._eager_steps = 0
        self._side_stream = torch.cuda.Stream(device=self.device)
        self._alloc_buffer()
        self._ret_log = torch.full((self._T, N), float("nan"), dtype=F32, device=dev)

    # ------------------------------------------------------------------ storage
    def _alloc_buffer(self):
        rb, N, o, a = self.replay_buffer, self._N, self._o, self._a
        rb.device = rb.device or self.device
        assert rb.env_nums == N, "replay buffer env_nums must equal the env's env_nums"
        shapes = {"obs": (N, o), "next_obs": (N, o), "acts": (N, a) if self.continuous else (N,),
                  "rewards": (N, 1), "terminals": (N, 1), "time_limits": (N, 1)}
        if self.on_policy:
            shapes["values"] = (N, 1)
        for k, shp in shapes.items():
            if not hasattr(rb, "_" + k):
                rb.allocate(k, shp)
        rb._ensure_device()
        self._T = rb._max_replay_buffer_size
        # epsilon-greedy Q policies on a device env: the host schedule ticks outside the captured step and hands the
        # rate over in a device scalar
        if not self._host_env and not self.continuous and hasattr(self.pf, "tick") and not hasattr(self.pf, "act_only"):
            self._eps_dev = torch.zeros(1, dtype=F32, device=self.device)
            self._eps_host = torch.zeros(1, dtype=F32).pin_memory()

    # ------------------------------------------------------------------ one step
    def _policy_action(self, ob):
        """Sample an action batch for `ob` into self._act (device)."""
        if hasattr(self.pf, "act_only"):
            self.pf.act_only(ob, eps=self._eps, action_out=self._act, nan_flag=self._nan_flag)
        else:
            kw = {} if self._eps_dev is None else {"epsilon": self._eps_dev}
            out = self.pf.explore(ob.unsqueeze(0) if not self.on_policy else ob, **kw)
            act = out["action"]
            self._act.copy_(act.reshape(self._act.shape).to(F32))

    def _finalize(self, v_next):
        env, rb = self.env, self.replay_buffer
        nrm = env._obs_normalizer if getattr(env, "obs_norm", False) else None
        # host envs, and device envs whose observation is not their state (`resets_itself`): the kernel stores rows and
        # the collector's counters and carries the stepped observation forward; the env resets the envs it cut
        own = getattr(env, "resets_itself", False)
        ext = self._host_env or own
        ops.collect_finalize(self.current_ob, env.obs_out, None if ext else env.state, self._act, self._value, v_next,
                             env.reward, env.done, env.time_limit, None if ext else env.elapsed,
                             None if ext else env.episode, None if ext else env.seeds, self.current_step,
                             self.train_rew, self._epoch_reward, self._ret_log, self._n_done,
                             None if ext else env.any_reset, None if nrm is None else nrm._mean,
                             None if nrm is None else nrm._var, self.current_ob, rb._obs, rb._next_obs, rb._acts,
                             rb._values if self.on_policy else None, rb._rewards, rb._terminals, rb._time_limits,
                             rb._top_dev, self.max_episode_frames, getattr(self, "discount", 0.99),
                             getattr(env, "init_scale", synth_spec.INIT_SCALE), nrm.clip if nrm is not None else 10.0,
                             self.on_policy, self.reference_quirks)
        if own:
            env.collector_reset(self.current_step, self.current_ob, rb._top_dev, self.reference_quirks)

    def _step_body(self, bootstrap):
        with torch.no_grad():
            ob = self.current_ob
            side = None
            if self._has_vf:
                # V(ob) is only needed by the finalize kernel: evaluate it on a second stream (a parallel branch of the
                # captured step graph) while the policy forward, the sampling and the env step run on this one
                main = torch.cuda.current_stream(self.device)
                side = self._side_stream
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    self._value.copy_(self.vf(ob).reshape(-1))
            self._policy_action(ob)
            self.env.launch_step(self._act, self.current_step, self.max_episode_frames, self.replay_buffer._top_dev)
            if not getattr(self.env, "obs_norm", False):
                self.env.obs_out.copy_(self.env.state)
            v_next = None
            if bootstrap and self._has_vf:
                if side is not None:
                    main.wait_stream(side)          # one value net, one set of per-stream scratch: V(ob) first
                    side = None
                self._v_next.copy_(self.vf(self.env.obs_out).reshape(-1))
                v_next = self._v_next
            if side is not None:
                main.wait_stream(side)
            self._finalize(v_next)
            if hasattr(self.replay_buffer, "mark_inserted"):
                self.replay_buffer.mark_inserted()    # prioritised ring: the new row enters with the max priority
            ops.counter_advance(None, self.replay_buffer._top_dev, self._T, self.replay_buffer._size_dev)

    def _step_host(self):
        """One collector step over HOST envs behind env/bridge.py (SURVEY.md 8(f).1).  Same order of
        operations as the reference loop (collector/on_policy.py:94-153): act, step, bootstrap the envs cut
        by `max_episode_frames`, store the row, reset finished envs.  Eager: the host env sits in the middle."""
        env = self.env
        with torch.no_grad():
            ob = self.current_ob
            self._policy_action(ob)
            if self._has_vf:
                self._value.copy_(self.vf(ob).reshape(-1))
            env.launch_step(self._act)
            sc = self._host_steps + 1
            mask = env.host_done | (sc >= self.max_episode_frames)
            reset = bool(mask.any())
            v_next = None
            if self._has_vf and reset:
                self._v_next.copy_(self.vf(env.obs_out).reshape(-1))
                v_next = self._v_next
            self._finalize(v_next)
            if reset:
                raw = env.partial_reset(mask)
                if self.reference_quirks or not env.obs_norm:
                    self.current_ob.copy_(raw)              # quirk A.1: raw observations for ALL envs
                else:
                    m = torch.from_numpy(mask).to(self.device)
                    self.current_ob[m] = env._obs_normalizer.filt(raw)[m]
            self._host_steps = np.where(mask, 0, sc)
            if hasattr(self.replay_buffer, "mark_inserted"):
                self.replay_buffer.mark_inserted()
            ops.counter_advance(None, self.replay_buffer._top_dev, self._T, self.replay_buffer._size_dev)
        self.replay_buffer.advance_host(1)

    def _need_bootstrap(self):
        """Host-side prediction of `any(done) or any(current_step >= max_episode_frames)` for this
        step (collector/on_policy.py:132-133).  Exact for lock-step envs (episode ends depend only
        on step counters); otherwise always bootstrap."""
        env = self.env
        if not self.on_policy:
            return False
        if not (getattr(env, "lockstep", False) and env._host_mirror_ok):
            return True
        will_done = env._host_elapsed + 1 >= env._max_episode_steps
        will_surpass = self._host_step + 1 >= self.max_episode_frames
        return bool(will_done or will_surpass)

    def _host_after_step(self):
        """Host mirrors of the step counters (lock-step envs only) and of the ring pointer."""
        env = self.env
        if getattr(env, "lockstep", False) and env._host_mirror_ok:
            el, st = env._host_elapsed + 1, self._host_step + 1
            if el >= env._max_episode_steps or st >= self.max_episode_frames:
                env._host_elapsed, self._host_step = 0, 0       # every env resets on this step
            else:
                env._host_elapsed, self._host_step = el, st
        self.replay_buffer.advance_host(1)

    def _step(self):
        if self._host_env:
            if D.get_noise_mode() == "reference_cpu" and self.continuous and hasattr(self.pf, "act_only"):
                if self._eps is None:
                    self._eps = torch.empty(self._N, self._a, dtype=F32, device=self.device)
                self._eps.copy_(D.draw_reference_noise((self._N, self._a), self.device))
            return self._step_host()
        boot = self._need_bootstrap()
        if self._eps_dev is not None:
            self.pf.tick()
            self._eps_host[0] = float(self.pf.epsilon)
            self._eps_dev.copy_(self._eps_host, non_blocking=True)
        if D.get_noise_mode() == "reference_cpu" and self.continuous and hasattr(self.pf, "act_only"):
            eps = D.draw_reference_noise((self._N, self._a), self.device)
            if self._eps is None:
                self._eps = torch.empty(self._N, self._a, dtype=F32, device=self.device)
            self._eps.copy_(eps)
        if not self.use_cuda_graph:
            self._step_body(boot)
        elif boot in self._graphs:
            self._graphs[boot].replay()
        elif self._eager_steps < 3:
            self._eager_steps += 1          # warm-up: real steps, executed eagerly
            self._step_body(boot)
        else:
            g = ops.CapturedGraph(lambda: self._step_body(boot))
            self._graphs[boot] = g
            g.replay()                      # capture does not execute: run the step now
        self._host_after_step()

    @fused.presplit_scope
    def take_actions(self):
        """One env step for all envs; returns the summed (un-bootstrapped) reward of the step."""
        before = self._epoch_reward.sum()
        self._step()
        return float((self._epoch_reward.sum() - before).item())

    # ------------------------------------------------------------------ epochs
    def start_episode(self):
        pass

    def finish_episode(self):
        pass

    def train_one_epoch(self):
        """T = epoch_frames // env_nums steps (collector/base.py:108-122, :179).  One host sync at the end."""
        top0 = self.replay_buffer._top
        self.rollout_no_sync()
        n_done = int(self._n_done.item())                   # the epoch's only sync
        if int(self._nan_flag.item()) != 0:
            raise FloatingPointError("NaN detected in sampled actions (reference: 'NaN detected. BOOM')")
        if hasattr(self.env, "check_actions"):
            self.env.check_actions()
        self.train_rews = []
        if n_done > 0:
            # finished-episode returns in the reference's order (time-major, env ascending)
            rows = (torch.arange(self.sample_epoch_frames, device=self.device) + top0) % self._T
            log = self._ret_log[rows]
            m = ~torch.isnan(log)
            self.train_rews = [float(x) for x in log[m].cpu().numpy()]
        self.train_epoch_reward = float(self._epoch_reward.sum().item())
        return {'train_rewards': self.train_rews, 'train_epoch_reward': self.train_epoch_reward}

    @fused.presplit_scope
    def rollout_no_sync(self):
        """The T collector steps of one epoch with no host read-back at all (what train_one_epoch
        runs before fetching its summary)."""
        self.env.train()
        self._epoch_reward.zero_()
        self._n_done.zero_()
        self._ret_log.fill_(float("nan"))
        for _ in range(self.sample_epoch_frames):
            self._step()

    @fused.presplit_scope
    def eval_one_epoch(self):
        """Deterministic-policy evaluation episodes on the eval env (collector/base.py:232-280)."""
        eval_env = self.eval_env
        if hasattr(self.env, "_obs_normalizer"):
            eval_env._obs_normalizer = copy.deepcopy(self.env._obs_normalizer)
        eval_env.eval()
        N = eval_env.env_nums
        eval_rews, traj_lens = [], []
        with torch.no_grad():
            for _ in range(self.eval_episodes):
                epi_done = torch.zeros(N, 1, dtype=torch.bool, device=self.device)
                rews = torch.zeros(N, 1, dtype=F64, device=self.device)
                traj_len = torch.zeros(N, 1, dtype=F64, device=self.device)
                eval_obs = eval_env.reset()
                steps = 0
                pixel = getattr(eval_env, "pixel", False)
                while True:
                    # pixel envs hand out uint8 frame stacks: scale them like the training path does
                    act = self.pf.eval_act(eval_env.to_float(eval_obs) if pixel else eval_obs)
                    if not torch.is_tensor(act):
                        act = torch.as_tensor(act, device=self.device)
                    eval_obs, r, done, _ = eval_env.step(act)
                    live = (~epi_done).to(F64)
                    rews = rews + live * r.to(F64)
                    traj_len = traj_len + live
                    epi_done = epi_done | done
                    steps += 1
                    if getattr(eval_env, "lockstep", False):
                        if steps >= eval_env._max_episode_steps:
                            break
                    else:
                        if bool(done.any()):
                            eval_obs = eval_env.partial_reset(done.squeeze(-1))
                        if bool(epi_done.all()):
                            break
                eval_rews += [float(x) for x in rews.reshape(-1).cpu().numpy()]
                traj_lens += [float(x) for x in traj_len.reshape(-1).cpu().numpy()]
        return {"eval_rewards": eval_rews, "eval_traj_length": float(np.mean(traj_lens))}

    def terminate(self):
        self.env.close()
        self.eval_env.close()

    def to(self, device):
        for func in self.funcs.values():
            func.to(device)

    @property
    def funcs(self):
        return {"pf": self.pf}


# the reference's single-env BaseCollector shares the constructor contract; with a device env of
# env_nums == 1 the vectorised collector is the same thing
BaseCollector = VecCollector
