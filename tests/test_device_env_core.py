"""The parts the state-vector device envs share (csrc/env_common.cuh, DeviceVecEnv in torchrl_b200/env/synth.py): the
step argument rule the synthetic env shares with CartPole and Pendulum, each env class's tensor attributes -- the names,
dtypes and shapes a checkpoint restores by name, so a checkpoint of an earlier build still loads -- and a CartPole and a
Pendulum checkpoint restored after the env has stepped on."""
import ctypes

import numpy as np
import pytest

N = 300     # 10 CTAs of the synthetic step, 2 of the CartPole and Pendulum steps


def test_synth_step_refuses_t_ptr_without_any_reset(native_lib):
    p = ctypes.c_void_p(16)
    assert native_lib.trl_synth_env_step(p, p, p, p, p, p, p, p, None, p, p, p, None, None, None, None, None, None,
                                         None, p, 4, 17, 6, 0.9, 0.5, 0.1, 3e38, 1.0, 1000, 1 << 30, 0, None) == -1
    assert native_lib.trl_last_error() == b"trl_synth_env_step: t_ptr given without the any_reset flag"


def _attrs(env):
    import torch
    return sorted((k, str(v.dtype).replace("torch.", ""), tuple(v.shape)) for k, v in vars(env).items()
                  if torch.is_tensor(v))


COUNTERS = [("done", "uint8", (N,)), ("elapsed", "int32", (N,)), ("episode", "int32", (N,)),
            ("reward", "float32", (N,)), ("seeds", "int32", (N,)), ("time_limit", "uint8", (N,)),
            ("_ticket", "int32", (1,)), ("any_reset", "int32", (2,))]


@pytest.mark.gpu
def test_synth_tensor_attributes():
    from torchrl_b200.env import SynthVecEnv
    want = COUNTERS + [("A", "float32", (17, 17)), ("B", "float32", (6, 17)), ("c", "float32", (17,)),
                       ("lb", "float32", (6,)), ("ub", "float32", (6,)), ("state", "float32", (N, 17)),
                       ("obs_out", "float32", (N, 17)), ("_partial", "float64", (10, 34)),
                       ("batch_sums", "float64", (34,))]
    assert _attrs(SynthVecEnv("SynthHalfCheetah-v0", N, {"obs_norm": True})) == sorted(want)


@pytest.mark.gpu
def test_cartpole_tensor_attributes():
    from torchrl_b200.env.cartpole import CartPoleVecEnv
    want = COUNTERS + [("action_error", "int32", (1,)), ("state", "float32", (N, 4)), ("obs_out", "float32", (N, 4)),
                       ("_partial", "float64", (2, 8)), ("batch_sums", "float64", (8,))]
    assert _attrs(CartPoleVecEnv("CartPole-v1", N, {"obs_norm": True})) == sorted(want)


@pytest.mark.gpu
def test_pendulum_tensor_attributes():
    from torchrl_b200.env.pendulum import PendulumVecEnv
    want = COUNTERS + [("action_error", "int32", (1,)), ("phys", "float64", (N, 2)), ("state", "float32", (N, 3)),
                       ("obs_out", "float32", (N, 3)), ("_partial", "float64", (2, 6)), ("batch_sums", "float64", (6,))]
    assert _attrs(PendulumVecEnv(N, {"obs_norm": True})) == sorted(want)


@pytest.mark.gpu
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1"])
def test_checkpoint_saved_before_a_step_restores_after_it(tmp_path, env_id):
    import torch
    if env_id == "CartPole-v1":
        from tests.test_cartpole_gpu import _dqn
        agent, _, _, env = _dqn("dqn", use_graph=False)
        acts = (torch.arange(env.env_nums, device="cuda") % 2).float()
    else:
        from tests.classic_control_gpu import continuous_agent
        agent, _, _, env = continuous_agent("Pendulum-v1", "td3", 3, 200, False, use_graph=False)
        acts = torch.linspace(-1.0, 1.0, env.env_nums, device="cuda")
    env.reset()
    path = str(tmp_path / "ck.pt")
    agent.save_checkpoint(path)
    saved = {k: v.clone() for k, v in vars(env).items() if torch.is_tensor(v)}
    stepped = [t.clone() for t in env.step(acts)[:3]]
    assert not torch.equal(env.state, saved["state"])
    agent.load_checkpoint(path)
    for k, v in saved.items():
        assert torch.equal(getattr(env, k), v), k
    again = env.step(acts)[:3]
    for a, b in zip(stepped, again):
        assert torch.equal(a, b)
    np.testing.assert_array_equal(env.elapsed.cpu().numpy(), 1)
