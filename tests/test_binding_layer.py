"""ops.py is the one Python binding of the C ABI: no other module of the package reaches the library, every wrapper
checks its pointer arguments before it launches, and the launch counter it keeps equals the kernels that ran."""
import ast
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "torchrl_b200")


def _package_sources():
    for dp, _, fns in os.walk(PKG):
        for fn in sorted(fns):
            if fn.endswith(".py"):
                path = os.path.join(dp, fn)
                yield os.path.relpath(path, ROOT), open(path).read()


def test_only_ops_imports_the_library():
    imports_lib = re.compile(r"^\s*(from|import)\s+[\w.]*\b_lib\b|^\s*from\s+[\w.]+\s+import\s+[^#\n]*\b_lib\b", re.M)
    uses_lib = re.compile(r"\b_lib\.")
    allowed = {os.path.join("torchrl_b200", "ops.py"), os.path.join("torchrl_b200", "_lib.py")}
    seen = set()
    for rel, txt in _package_sources():
        if rel in allowed:
            seen.add(rel)
            continue
        assert not imports_lib.search(txt), "%s imports _lib: bind the entry point in ops.py" % rel
        assert not uses_lib.search(txt), "%s reaches _lib: bind the entry point in ops.py" % rel
    assert seen == allowed


def test_only_captured_graph_adds_launches():
    """Every wrapper counts its own kernels through _lib.call; only a graph replay adds a count by hand."""
    sites = []
    entry = [(f, open(os.path.join(ROOT, f)).read()) for f in ("bench.py", "__graft_entry__.py")]
    files = list(_package_sources()) + entry
    for rel, txt in files:
        if "add_launches" not in txt:
            continue
        tree = ast.parse(txt)
        owner = {}
        for cls in (n for n in ast.walk(tree) if isinstance(n, ast.ClassDef)):
            for sub in ast.walk(cls):
                owner[id(sub)] = cls.name
        for node in ast.walk(tree):
            callee = getattr(node.func, "attr", getattr(node.func, "id", None)) if isinstance(node, ast.Call) else None
            if callee == "add_launches":
                sites.append((rel, owner.get(id(node))))
        names = {n.id for n in ast.walk(tree) if isinstance(n, ast.Name)} | {n.attr for n in ast.walk(tree)
                                                                            if isinstance(n, ast.Attribute)}
        if rel == os.path.join("torchrl_b200", "_lib.py"):
            assert "add_launches" not in names, "_lib.py calls add_launches"
        else:
            assert "add_launches" in names
    assert sites and all(s == (os.path.join("torchrl_b200", "ops.py"), "CapturedGraph") for s in sites), sites


# ------------------------------------------------------------------------------------------ GPU
def _launches_and_kernels(fn):
    """(_lib.launch_count() delta, names of the library kernels the profiler saw) of fn()."""
    from torch.profiler import ProfilerActivity, profile

    from torchrl_b200 import _lib
    torch.cuda.synchronize()
    before = _lib.launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    counted = _lib.launch_count() - before
    return counted, [e.name for e in prof.events() if "trl::" in e.name]


def _multi_kernel_calls():
    from torchrl_b200 import ops
    dev = "cuda"
    M, H, K, N = 4096, 256, 17, 6
    g = torch.randn(M, H, device=dev)
    y = torch.tanh(torch.randn(M, H, device=dev))
    x = torch.randn(M, K, device=dev)
    g_out = torch.randn(M, N, device=dev)
    w_out = torch.randn(N, H, device=dev)
    gz = torch.empty(M, H, device=dev)
    db, dw = torch.empty(H, device=dev), torch.empty(H, K, device=dev)
    dw3, db3 = torch.empty(N, H, device=dev), torch.empty(N, device=dev)
    tn = lambda k: torch.empty(ops.skinny_tn_scratch_floats(M, H, k), device=dev)
    da = torch.empty(ops.skinny_dgrad_act_scratch_floats(M, H), device=dev)
    a_tn, b_tn = torch.randn(8192, 256, device=dev), torch.randn(8192, 256, device=dev)
    a_nt, b_nt = torch.randn(512, 256, device=dev), torch.randn(256, 256, device=dev)
    part = tn(K)
    return {
        "skinny_tn": lambda: ops.skinny_tn(g, x, dw, None, False, tn(K)),
        "skinny_act_wgrad": lambda: ops.skinny_act_wgrad(g, y, x, dw, db, 1, tn(K)),
        "skinny_n_dgrad_act_wgrad": lambda: ops.skinny_n_dgrad_act_wgrad(g_out, w_out, y, 1, gz, db, dw3, db3, da,
                                                                         tn(N)),
        "skinny_reduce_jobs": lambda: (ops.skinny_act_wgrad_partial(g, y, x, 1, part),
                                       ops.skinny_reduce_jobs([(1, part, dw, db, M, H, K, 0)])),
        "skinny_reduce_jobs_empty": lambda: ops.skinny_reduce_jobs([]),
        "gemm3_pair_tn_splitk": lambda: ops.gemm3_pair_tn(a_tn, b_tn, splits=8),
        "gemm3_pair_tn": lambda: ops.gemm3_pair_tn(a_tn, b_tn),
        "gemm_tf32x3_tn_splitk": lambda: ops.gemm_tf32x3_tn(a_tn, b_tn, splits=8),
        "gemm_tf32x3_nt_splitk": lambda: ops.gemm_tf32x3_nt(a_nt, b_nt, splits=2),
        "gemm_tf32x3_nt": lambda: ops.gemm_tf32x3_nt(a_nt, b_nt),
        "split_tf32": lambda: ops.split_tf32(a_nt),
    }


@pytest.mark.gpu
def test_multi_kernel_wrappers_count_what_they_launch():
    calls = _multi_kernel_calls()
    for name, fn in calls.items():
        fn()                                            # one-time setup outside the profile
        counted, kernels = _launches_and_kernels(fn)
        assert counted == len(kernels), "%s counted %d launches for %d kernels %s" % (name, counted, len(kernels),
                                                                                      kernels)
    assert _launches_and_kernels(calls["skinny_tn"])[0] == 2


@pytest.mark.gpu
def test_first_layer_backward_counts_what_it_launches(monkeypatch):
    """The _MLPTail backward on its immediate first-layer route (inside transposed_planes, no deferred reduces): the
    dgrad GEMM with the first layer's slab partials in its epilogue, then one slab-sum launch."""
    import torch.nn as nn

    import torchrl_b200.networks as networks
    from torchrl_b200 import ops
    from torchrl_b200.flat import FlatAdam
    from torchrl_b200.networks import fused
    torch.manual_seed(3)
    M = 16384
    net = networks.Net(input_shape=17, output_shape=6, hidden_shapes=[256, 256], append_hidden_shapes=[],
                       base_type=networks.MLPBase, activation_func=nn.Tanh).cuda()
    opt = FlatAdam([net], lrs=[1e-3])
    x = torch.randn(M, 17, device="cuda")
    w = torch.randn(M, 6, device="cuda")
    calls = []
    real = ops.gemm3_pair_dgrad_act_wgrad
    monkeypatch.setattr(ops, "gemm3_pair_dgrad_act_wgrad", lambda *a: calls.append(1) or real(*a))
    for profiled in (False, True):                      # the first pass allocates the scratch buffers
        opt.zero_grad()
        with fused.presplit(), fused.transposed_planes(opt):
            y = net(x)
            if profiled:
                counted, kernels = _launches_and_kernels(lambda: torch.autograd.backward([y], [w]))
            else:
                torch.autograd.backward([y], [w])
    assert len(calls) == 2, "the backward did not take the fused first-layer route"
    assert counted == len(kernels), "counted %d launches for %d kernels %s" % (counted, len(kernels), kernels)


def _finalize_args(**override):
    F32, F64, U8, I32 = torch.float32, torch.float64, torch.uint8, torch.int32
    N, o, a, T = 4, 3, 2, 5
    z = lambda *shape, dtype=F32: torch.zeros(*shape, dtype=dtype, device="cuda")
    args = dict(cur_ob_in=z(N, o), next_norm=z(N, o), state=z(N, o), act=z(N, a), value=None, v_next=None,
                reward=z(N), done=z(N, dtype=U8), tl=z(N, dtype=U8), elapsed=z(N, dtype=I32),
                episode=z(N, dtype=I32), seeds=z(N, dtype=I32), step_count=z(N, dtype=I32), ep_return=z(N, dtype=F64),
                epoch_reward=z(N, dtype=F64), ret_log=z(T, N), n_done=z(1, dtype=I32), any_reset=z(2, dtype=I32),
                norm_mean=None, norm_var=None, cur_ob_out=z(N, o), b_obs=z(T, N, o), b_next_obs=z(T, N, o),
                b_acts=z(T, N, a), b_values=None, b_rewards=z(T, N, 1), b_terminals=z(T, N, 1, dtype=U8),
                b_time_limits=z(T, N, 1, dtype=U8), t_ptr=z(1, dtype=I32), max_episode_frames=1000, discount=0.99,
                init_scale=0.1, clip=10.0, terminal_includes_surpass=False, raw_obs_after_reset=True)
    args.update(override)
    return args


@pytest.mark.gpu
def test_former_raw_sites_reject_bad_operands():
    """Operands that used to reach the kernels as bare addresses are checked now: nothing is launched."""
    from torchrl_b200 import _lib, ops
    from torchrl_b200.env.synth import SynthVecEnv
    from torchrl_b200.replay_buffers.memory_efficient import MemoryEfficientReplayBuffer
    ops.collect_finalize(**_finalize_args())                       # the well-formed call runs
    rb = MemoryEfficientReplayBuffer(64, env_nums=2, device="cuda")
    rb.allocate_frames((4, 8, 8))
    env = SynthVecEnv("SynthHalfCheetah-v0", 4)
    acts = torch.zeros(4, env.act_dim, device="cuda")
    torch.cuda.synchronize()
    before = _lib.launch_count()
    with pytest.raises(TypeError):
        ops.collect_finalize(**_finalize_args(step_count=torch.zeros(4, dtype=torch.int64, device="cuda")))
    with pytest.raises(ValueError):
        rb.gather_rows(torch.zeros(8, dtype=torch.int64, device="cuda")[::2], ["obs", "next_obs"])
    with pytest.raises(TypeError):
        env.launch_step(acts, step_count=torch.zeros(4, dtype=torch.int64, device="cuda"))
    assert _lib.launch_count() == before
