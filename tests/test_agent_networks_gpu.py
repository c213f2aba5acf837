"""The network layout of every agent, as literal expectations: which networks a checkpoint saves and in what order
(`networks` decides the order of `state["networks"]`, so a change breaks resume), the (online, target) pairs, the
snapshot names, the fused optimizer's segments with their learning rates, clip norms and eps, and the names of the
tensor attributes a checkpoint saves.  For the off-policy agents also the library launches of every captured update
graph variant: the agents' update bodies may be rearranged in Python, but each graph must hold the same kernels."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _a2c():
    from tests.test_categorical_onpolicy import _pixel_agent
    return _pixel_agent("a2c")[0]


def _ppo():
    from tests.test_ppo_pipeline import _build
    return _build()[0]


def _trpo():
    from tests.test_trpo_categorical_gpu import _pixel_agent
    return _pixel_agent()[0]


def _vmpo():
    from tests.test_vmpo_categorical_gpu import _pixel_agent
    return _pixel_agent()[0]


def _reinforce():
    from tests.test_cartpole_gpu import _on_policy
    return _on_policy("reinforce")[0]


def _continuous(kind):
    def build():
        from tests.test_per_agents_gpu import _agent
        return _agent(kind, per=False)[0]
    return build


def _dqn(kind):
    def build():
        from tests.test_cartpole_gpu import _dqn
        return _dqn(kind)[0]
    return build


def _bootstrapped():
    from tests.test_bootstrapped_gpu import _build
    return _build()[0]


_SAC_TENSORS = ["_alpha_state", "log_alpha"]

# class: (builder, networks, target pairs, snapshots, optimizer lrs, clip norms, eps, tensor attributes)
LAYOUTS = {
    "A2C": (_a2c, ["pf", "vf"], [], [("pf", "pf"), ("vf", "vf")], [3e-4, 3e-4], [0.5, 0.5], [1e-5, 1e-5], []),
    "PPO": (_ppo, ["pf", "vf", "target_pf"], [("pf", "target_pf")], [("pf", "pf"), ("vf", "vf")], [3e-4, 3e-4],
            [0.5, 0.5], [1e-5, 1e-5], []),
    "TRPO": (_trpo, ["pf", "vf"], [], [("pf", "pf"), ("vf", "vf")], [3e-4, 3e-4], [0.5, 0.5], [1e-5, 1e-5], []),
    "VMPO": (_vmpo, ["pf", "vf", "target_pf"], [("pf", "target_pf")], [("pf", "pf"), ("vf", "vf")],
             [3e-4, 3e-4, 3e-4], [0.5, 0.5, 0.0], [1e-5, 1e-5, 1e-5], ["dual"]),
    "Reinforce": (_reinforce, ["pf", "vf"], [], [("pf", "pf")], [3e-3], [0.5], [1e-8], []),
    "DDPG": (_continuous("ddpg"), ["pf", "qf", "target_pf", "target_qf"], [("pf", "target_pf"), ("qf", "target_qf")],
             [("pf", "pf"), ("qf", "qf")], [1e-3, 1e-3], [0.0, 0.0], [1e-8, 1e-8], []),
    "TD3": (_continuous("td3"), ["pf", "qf1", "qf2", "target_pf", "target_qf1", "target_qf2"],
            [("pf", "target_pf"), ("qf1", "target_qf1"), ("qf2", "target_qf2")],
            [("pf", "pf"), ("qf1", "qf1"), ("qf2", "qf2")], [1e-3, 1e-3, 1e-3], [0.0] * 3, [1e-8] * 3, []),
    "TwinSACQ": (_continuous("twin_sac_q"), ["pf", "qf1", "qf2", "target_qf1", "target_qf2"],
                 [("qf1", "target_qf1"), ("qf2", "target_qf2")], [("pf", "pf"), ("qf1", "qf1"), ("qf2", "qf2")],
                 [3e-4, 3e-4, 3e-4], [0.0] * 3, [1e-8] * 3, _SAC_TENSORS),
    "SAC": (_continuous("sac"), ["pf", "qf", "vf", "target_vf"], [("vf", "target_vf")],
            [("pf", "pf"), ("qf", "qf"), ("vf", "vf")], [3e-4, 3e-4, 3e-4], [0.0] * 3, [1e-8] * 3, _SAC_TENSORS),
    "TwinSAC": (_continuous("twin_sac"), ["pf", "qf1", "qf2", "vf", "target_vf"], [("vf", "target_vf")],
                [("pf", "pf"), ("qf1", "qf1"), ("qf2", "qf2"), ("vf", "vf")], [3e-4] * 4, [0.0] * 4, [1e-8] * 4,
                _SAC_TENSORS),
    "DQN": (_dqn("dqn"), ["qf", "target_qf"], [("qf", "target_qf")], [("pf", "qf")], [1e-3], [0.0], [1e-8], []),
    "QRDQN": (_dqn("qrdqn"), ["qf", "target_qf"], [("qf", "target_qf")], [("pf", "qf")], [1e-3], [0.0], [1e-8],
              ["quantile_coefficient"]),
    "BootstrappedDQN": (_bootstrapped, ["qf", "target_qf"], [("qf", "target_qf")], [("pf", "qf")], [1e-3], [0.0],
                        [1e-4], []),
}


def _name(agent, net):
    """The one attribute of `agent` that holds `net`."""
    names = [k for k, v in vars(agent).items() if v is net]
    assert len(names) == 1, names
    return names[0]


def _f32(xs):
    return [float(np.float32(x)) for x in xs]


@pytest.mark.parametrize("cls", sorted(LAYOUTS))
def test_agent_network_layout(cls):
    from torchrl_b200.utils import checkpoint
    build, nets, targets, snapshots, lrs, norms, eps, tensors = LAYOUTS[cls]
    agent = build()
    assert type(agent).__name__ == cls
    assert [_name(agent, n) for n in agent.networks] == nets
    assert [(_name(agent, o), _name(agent, t)) for o, t in agent.target_networks] == targets
    assert [(name, _name(agent, n)) for name, n in agent.snapshot_networks] == snapshots
    opt = agent.opt
    assert opt.nseg == len(lrs) and opt.initial_lrs == lrs
    assert list(opt._max_norm_c) == _f32(norms) and list(opt._eps_c) == _f32(eps)
    assert sorted(checkpoint._tensors(agent)) == tensors


def _per_agent(kind, per):
    def build():
        from tests.test_per_agents_gpu import _agent
        agent, col, _, _ = _agent(kind, per=per)
        return agent, col
    return build


def _offpolicy(kind):
    def build():
        from tests.test_offpolicy import _build_offpolicy
        agent, col, _, _ = _build_offpolicy(kind)
        return agent, col
    return build


def _dqn_col(kind):
    def build():
        from tests.test_cartpole_gpu import _dqn
        agent, col, _, _ = _dqn(kind)
        return agent, col
    return build


def _bootstrapped_col():
    from tests.test_bootstrapped_gpu import _build
    agent, col, _, _ = _build(graph_agent=True, opt_times=4)
    return agent, col


# case: (builder of the agent and its collector, {update-graph variant: library launches it holds})
LAUNCHES = {
    "ddpg": (_per_agent("ddpg", False), {0: 24}),
    "ddpg_per": (_per_agent("ddpg", True), {0: 27}),
    "td3": (_per_agent("td3", False), {0: 24, 1: 36}),
    "td3_per": (_per_agent("td3", True), {0: 27, 1: 39}),
    "td3_ant": (_offpolicy("td3"), {0: 24, 1: 36}),
    "twin_sac_q": (_per_agent("twin_sac_q", False), {0: 42}),
    "twin_sac_q_per": (_per_agent("twin_sac_q", True), {0: 45}),
    "twin_sac_q_ant": (_offpolicy("sac"), {0: 42}),
    "sac": (_per_agent("sac", False), {0: 32}),
    "sac_per": (_per_agent("sac", True), {0: 35}),
    "twin_sac": (_per_agent("twin_sac", False), {0: 40}),
    "twin_sac_per": (_per_agent("twin_sac", True), {0: 43}),
    "dqn": (_dqn_col("dqn"), {0: 12}),
    "qrdqn": (_dqn_col("qrdqn"), {0: 12}),
    "bootstrapped_dqn": (_bootstrapped_col, {0: 7}),
}


@pytest.mark.parametrize("case", sorted(LAUNCHES))
def test_captured_update_launches(case):
    build, want = LAUNCHES[case]
    agent, col = build()
    agent.pretrain()
    for _ in range(3):
        col.train_one_epoch()
        agent.update_per_epoch()
        if set(agent._graphs) >= set(want):
            break
    torch.cuda.synchronize()
    assert {v: g.launches for v, g in agent._graphs.items()} == want
