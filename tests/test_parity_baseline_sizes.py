"""End-to-end parity AT THE BENCHMARK'S SIZES: the device path bench.py times -- wgmma 3xTF32 GEMMs with pre-split
weight planes, the fused MLP tail, skinny-layer kernels, direct gradient writes, CUDA graphs -- against the CPU oracle
port (oracle/ref_port.py, pinned bit-for-bit to the unmodified reference by tests/test_oracle_vs_reference.py) on the
same seeds and the same exploration noise.

BASELINE.json configs[1]: PPO, 4096 SynthHalfCheetah envs, horizon 128, MLP(256,256), minibatches of 4 time rows
(16384 samples).  One epoch with ONE optimisation pass (32 minibatches) keeps the CPU side at ~15 s.

Stated tolerances (fp32 device arithmetic incl. 3xTF32 GEMMs vs float64 NumPy buffers / torch-CPU fp32 nets, after
128 env steps and 32 Adam steps):
  rollout tensors (obs, next_obs, acts, values, rewards) .... 99.9 % of the elements within atol 5e-4 (+ rtol 1e-4),
                                                              every element within 2e-2 (fp32 vs fp64 dynamics drift
                                                              apart over 128 steps for a handful of envs); flags exact
  advantages / returns ..................................... atol 2e-3 (+ rtol 1e-3)
  logged scalars of every minibatch ........................ rtol 5e-3 + atol 5e-4
  parameters after the pass ................................ atol 5e-4
  observation-normaliser state ............................. rtol 1e-5
The measured maxima are written to gpurun_out/parity_baseline_sizes.json.
"""
import json
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dump(name, rec):
    try:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        path = os.path.join(ROOT, "gpurun_out", "parity_baseline_sizes.json")
        cur = json.load(open(path)) if os.path.exists(path) else {}
        cur[name] = rec
        json.dump(cur, open(path, "w"), indent=1)
    except OSError:
        pass


@pytest.mark.gpu
def test_ppo_config2_epoch_matches_reference_port():
    import torch
    from oracle import ref_port
    from torchrl_b200.networks import fused
    from torchrl_b200.policies import set_noise_mode
    from tests.test_ppo_pipeline import _build
    N, T, hidden, rows, oe, seed = 4096, 128, (256, 256), 4, 1, 11
    keys = ("obs", "next_obs", "acts", "values", "rewards", "terminals", "time_limits")
    assert fused.get_matmul_mode() == "tc3"
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    penv, pcol, pagent = ref_port.build_ppo(env_nums=N, horizon=T, hidden=hidden, batch_rows=rows, opt_epochs=oe, seed=seed)
    pagent.current_epoch = 0
    p_out = pcol.train_one_epoch()
    roll = {k: pagent.buffer.data[k].copy() for k in keys}
    pagent.update_per_epoch()
    rec, checks = {}, []
    set_noise_mode("reference_cpu")
    try:
        agent, col, buf, env = _build(N=N, T=T, hidden=hidden, use_graph=True, seed=seed, opt_epochs=oe, batch_rows=rows)
        agent.current_epoch = 0
        out = col.train_one_epoch()
        assert abs(out["train_epoch_reward"] - p_out["train_epoch_reward"]) <= 1e-5 * abs(p_out["train_epoch_reward"]) + 1.0
        for k in keys:
            got = getattr(buf, "_" + k).cpu().numpy().astype(np.float64)
            ref = roll[k].reshape(got.shape)
            rec["rollout/" + k] = float(np.abs(got - ref).max())
            if k in ("terminals", "time_limits"):
                np.testing.assert_array_equal(got, ref, err_msg=k)
            else:
                bad = np.abs(got - ref) > 5e-4 + 1e-4 * np.abs(ref)
                rec["rollout_outliers/" + k] = float(bad.mean())
                checks.append((k, float(bad.mean()) < 1e-3 and rec["rollout/" + k] < 2e-2))
        agent.update_per_epoch()
        advs, rets = buf._advs.cpu().numpy(), buf._estimate_returns.cpu().numpy()
        rec["advs"] = float(np.abs(advs - pagent.buffer.data["advs"]).max())
        rec["returns"] = float(np.abs(rets - pagent.buffer.data["estimate_returns"]).max())
        for name, got, ref in (("advs", advs, pagent.buffer.data["advs"]), ("returns", rets, pagent.buffer.data["estimate_returns"])):
            bad = np.abs(got - ref) > 2e-3 + 1e-3 * np.abs(ref)
            rec[name + "_outliers"] = float(bad.mean())
            checks.append((name, float(bad.mean()) < 1e-3 and rec[name] < 5e-2))
        infos = agent._last_infos
        assert len(infos) == len(pagent.infos) == oe * (T // rows)
        worst, worst_key = 0.0, None
        for u in range(len(infos)):
            for k, v in pagent.infos[u].items():
                err = abs(infos[u][k] - v) / (5e-3 * abs(v) + 5e-4)
                if err > worst:
                    worst, worst_key = err, (u, k, infos[u][k], v)
        rec["infos_worst_over_tolerance"] = worst
        rec["infos_worst_key"] = repr(worst_key)
        checks.append(("infos", worst <= 1.0))
        mine = torch.cat([p.detach().reshape(-1) for p in list(agent.pf.mean_params()) +
                          list(agent.vf.parameters())]).cpu().numpy()
        ref = torch.cat([p.detach().reshape(-1) for p in list(pagent.pf.net.parameters()) +
                         list(pagent.vf.parameters())]).numpy()
        rec["params"] = float(np.abs(mine - ref).max())
        checks.append(("params", rec["params"] < 5e-4))
        nrm = env._obs_normalizer
        rec["norm_mean"] = float(np.abs(nrm._mean.cpu().numpy() - penv.norm.mean).max())
        rec["norm_var_rel"] = float((np.abs(nrm._var.cpu().numpy() - penv.norm.var) / penv.norm.var).max())
        checks.append(("normaliser", rec["norm_mean"] < 1e-5 and rec["norm_var_rel"] < 1e-4))
        assert agent._mb_graph is not None and col._graphs, "the captured-graph path must be the one that ran"
        failed = [name for name, ok in checks if not ok]
        assert not failed, (failed, rec)
    finally:
        set_noise_mode("philox")
        _dump("ppo_config2", rec)
