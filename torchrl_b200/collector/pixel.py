"""Collectors for the uint8 pixel env (BASELINE.json config 4): the VecCollector step
(/root/reference/torchrl/collector/base.py:184-230) with frames kept uint8 from the env to the replay ring.

Off-policy step (one captured CUDA graph): ring write obs[t] <- frames | u8->f32 scale | epsilon-greedy Q policy |
env step (frame-stack shift + render, in place) | ring write next_obs[t] <- frames | scalar finalize
(acts / rewards / terminals / time_limits rows, episode returns, timeout + done -> reset mask) | re-render
the reset envs | ring advance.  `epsilon` lives in a device scalar refreshed from the host schedule.  With a
BootstrappedDQNDiscretePolicy the epsilon-greedy stage is the all-heads forward plus one trl_bootstrapped_act launch
(per-env heads redrawn at episode starts, greedy actions, the transition's bootstrap mask row in the `masks` ring key)
and there is no epsilon schedule.

On-policy step (PixelVecOnPolicyCollector, the VecOnPolicyCollector of a pixel env,
/root/reference/torchrl/collector/on_policy.py:94-153): the same graph with V(obs) on a side stream, the policy's
`act_only` sampler (categorical kernel) in place of epsilon-greedy, V(next frames) for the timeout bootstrap (the env
is not lock-step, so every step) and the finalize kernel in on-policy mode (values row, r + discount * V(next_obs) on
rows cut by max_episode_frames, terminals include the cut).
"""
import numpy as np
import torch

from .. import ops
from ..policies import distribution as D
from ..policies.discrete_policies import BootstrappedDQNDiscretePolicy
from .base import VecCollector

F32, F64, U8, I32 = torch.float32, torch.float64, torch.uint8, torch.int32


class PixelVecCollector(VecCollector):
    on_policy = False

    def __init__(self, **kwargs):
        super().__init__(**kwargs)

    def _alloc_buffer(self):
        rb, N = self.replay_buffer, self._N
        rb.device = rb.device or self.device
        assert rb.env_nums == N
        frame = tuple(self.env.observation_space.shape)
        self._dedup = bool(getattr(rb, "frame_dedup", False))
        keys = [("acts", (N,), F32), ("rewards", (N, 1), F32), ("terminals", (N, 1), U8), ("time_limits", (N, 1), U8)]
        if self.on_policy:
            keys.append(("values", (N, 1), F32))
        # Bootstrapped DQN: one Bernoulli mask over the heads per transition, written by the policy's act launch
        self._boot = isinstance(self.pf, BootstrappedDQNDiscretePolicy)
        if self._boot:
            keys.append(("masks", (N, self.pf.head_num), U8))
        assert not (self.on_policy and self._dedup), "the on-policy pixel collector stores full frame stacks"
        if self._dedup:
            # frame-de-duplicated ring (replay_buffers/memory_efficient.py): one frame of obs and one of next_obs per
            # row instead of two C-frame stacks
            if getattr(rb, "_stack", None) is None:
                rb.allocate_frames(frame)
        else:
            keys = [("obs", (N,) + frame, U8), ("next_obs", (N,) + frame, U8)] + keys
        for k, shp, dt in keys:
            if not hasattr(rb, "_" + k):
                rb.allocate(k, shp, dt)
        rb._ensure_device()
        self._T = rb._max_replay_buffer_size
        dev = self.device
        # the scalar finalize kernel wants (N,o)/(T,N,o) observation operands: feed it 1-wide dummies
        self._d_ob = torch.zeros(N, 1, dtype=F32, device=dev)
        self._d_state = torch.zeros(N, 1, dtype=F32, device=dev)
        self._d_rows = torch.zeros(self._T, N, 1, dtype=F32, device=dev)
        self._obs_f = torch.empty((N,) + frame, dtype=F32, device=dev)
        self._next_f = torch.empty((N,) + frame, dtype=F32, device=dev) if self.on_policy else None
        self._any_reset = torch.zeros(2, dtype=I32, device=dev)
        if not self._dedup:
            self._plan_obs = ops.RowCopyPlan([self.env.obs.view(1, -1)], [rb._obs], [ops.row_bytes_of(rb._obs)])
            self._plan_next = ops.RowCopyPlan([self.env.obs.view(1, -1)], [rb._next_obs], [ops.row_bytes_of(rb._next_obs)])
        if self._boot:
            self.pf.ensure_heads(N, dev)
        self._eps_dev = torch.zeros(1, dtype=F32, device=dev)
        self._eps_host = torch.zeros(1, dtype=F32).pin_memory()

    def _o_dim(self):
        return 1

    def _step_body(self, bootstrap):
        env, rb = self.env, self.replay_buffer
        with torch.no_grad():
            if self._dedup:
                rb.write_obs(env.obs, env.elapsed)
            else:
                ops.ring_write(self._plan_obs, rb._top_dev)
            env.to_float(env.obs, self._obs_f)
            side = None
            if self.on_policy:
                if self._has_vf:
                    # V(obs) is only needed by the finalize kernel: a parallel branch of the captured step graph
                    main = torch.cuda.current_stream(self.device)
                    side = self._side_stream
                    side.wait_stream(main)
                    with torch.cuda.stream(side):
                        self._value.copy_(self.vf(self._obs_f).reshape(-1))
                self.pf.act_only(self._obs_f, action_out=self._act, nan_flag=self._nan_flag)
            elif self._boot:
                self.pf.act(self._obs_f, self.current_step, self._act, rb._masks, rb._top_dev)
            else:
                out = self.pf.explore(self._obs_f.unsqueeze(0), epsilon=self._eps_dev)
                self._act.copy_(out["action"].reshape(self._act.shape).to(F32))
            env.launch_step(self._act.reshape(-1))
            if self._dedup:
                rb.write_next_obs(env.obs)
            else:
                ops.ring_write(self._plan_next, rb._top_dev)
            v_next = None
            if side is not None:
                main.wait_stream(side)              # one value net, one set of per-stream scratch: V(obs) first
                self._v_next.copy_(self.vf(env.to_float(env.obs, self._next_f)).reshape(-1))
                v_next = self._v_next
            ops.collect_finalize(self._d_ob, self._d_ob, self._d_state, self._act, self._value, v_next, env.reward,
                                 env.done, env.time_limit, env.elapsed, env.episode, env.seeds, self.current_step,
                                 self.train_rew, self._epoch_reward, self._ret_log, self._n_done, None, None, None,
                                 self._d_ob, self._d_rows, self._d_rows, rb._acts,
                                 rb._values if self.on_policy else None, rb._rewards, rb._terminals,
                                 rb._time_limits, rb._top_dev, self.max_episode_frames,
                                 getattr(self, "discount", 0.0), 0.0, 10.0, self.on_policy, True)
            # envs whose collector step counter was just zeroed need a fresh episode (done or timeout); the
            # finalize kernel already advanced their episode counter
            env._reset(zero_is_mask=self.current_step, episode_bias=1, bump=0)
            if hasattr(rb, "mark_inserted"):
                rb.mark_inserted()                    # prioritised ring: the new row enters with the max priority
            ops.counter_advance(None, rb._top_dev, self._T, rb._size_dev)

    def _need_bootstrap(self):
        return False

    def _step(self):
        boot = self.on_policy
        if not (self.on_policy or self._boot):
            self.pf.tick()                               # host-side epsilon schedule -> device scalar
            self._eps_host[0] = float(self.pf.epsilon)
            self._eps_dev.copy_(self._eps_host, non_blocking=True)
        # "reference_cpu" sampling draws on the host (torch.multinomial): not capturable
        eager = not self.use_cuda_graph or (self.on_policy and D.get_noise_mode() == "reference_cpu")
        if eager:
            self._step_body(boot)
        elif boot in self._graphs:
            self._graphs[boot].replay()
        elif self._eager_steps < 3:
            self._eager_steps += 1
            self._step_body(boot)
        else:
            g = ops.CapturedGraph(lambda: self._step_body(boot))
            self._graphs[boot] = g
            g.replay()
        self.replay_buffer.advance_host(1)
