"""The prioritised-replay kernels that serve rings beyond 4096 rows and the importance-weighted critic loss, called
through the C ABI: trl_per_sample_rows (csrc/prioritized.cu) against trl_per_sample and the NumPy oracle, the
deterministic trl_per_update, and trl_twin_mse_loss_weighted (csrc/offpolicy.cu) against fp64.  Conventions are those
of test_data_path_kernels.py: guarded outputs, every case run twice for identical bits."""
import numpy as np
import pytest
import torch

from oracle import ref_numpy as rn
from tests.test_data_path_kernels import (BETA, PER_SIZES, U_TOP, guarded_ints, per_run, twice, uniforms,
                                          wide_priorities)
from tests.test_layer_kernels import U, Guarded, call, same_bits, stream

pytestmark = pytest.mark.gpu
CHUNK = 4096


def scratch_for(capacity):
    from torchrl_b200 import ops
    return torch.empty(ops.per_scratch_doubles(capacity), dtype=torch.float64, device="cuda")


def rows_run(prio, capacity, size, u, b=None, pos=0):
    """trl_per_sample_rows over the first `capacity` entries of prio with *size_ptr = size, draws at position pos."""
    ud = torch.as_tensor(np.asarray(u, dtype=np.float64), device="cuda")
    b = ud.numel() if b is None else b
    sp = torch.tensor([size], dtype=torch.int32, device="cuda")
    pp = torch.tensor([pos], dtype=torch.int32, device="cuda")
    sc = scratch_for(capacity)

    def run():
        idx, w = guarded_ints(b, torch.int64), Guarded(b)
        call("trl_per_sample_rows", prio.data_ptr(), capacity, sp.data_ptr(), ud.data_ptr(), pp.data_ptr(), b, BETA,
             idx.t.data_ptr(), w.t.data_ptr(), sc.data_ptr(), stream())
        return [idx.check("idx"), w.check("weights")]

    return twice(run)


def exact_priorities(rs, size, zero_frac=0.0):
    p = (rs.randint(1, 1025, size) * 2.0 ** -10).astype(np.float32)
    if zero_frac:
        p[rs.rand(size) < zero_frac] = 0.0
    return p


def check_weights(w, rw):
    w = w.cpu().numpy().astype(np.float64)
    assert np.all(np.abs(w - rw) <= (U + 2.0 ** -40) * rw + 2.0 ** -149)


# ------------------------------------------------------------------------------------ bit identity with the one CTA
@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("size", PER_SIZES)
def test_rows_sampler_equals_one_cta_sampler_bit_for_bit(size, wide):
    """up to 4096 rows there is one chunk with offset 0.0 and the same scan order: identical idx and weight bits,
    also when the ring's capacity is larger than the live size"""
    rs = np.random.RandomState(size + 17 * wide)
    p = wide_priorities(rs, size) if wide else exact_priorities(rs, size)
    for b in (1, 7, 1025):
        u = uniforms(rs, b)
        prio = torch.from_numpy(p).cuda()
        idx1, w1 = per_run(prio, size, u, BETA)
        for capacity in (size, 3 * CHUNK + 5):
            big = torch.zeros(capacity, dtype=torch.float32, device="cuda")
            big[:size] = prio
            big[size:] = 7.0                                 # rows past the live size must not matter
            idx2, w2 = rows_run(big, capacity, size, u)
            assert torch.equal(idx1, idx2), "indices differ from trl_per_sample (size %d, b %d)" % (size, b)
            assert same_bits(w1, w2), "weights differ from trl_per_sample (size %d, b %d)" % (size, b)


# ------------------------------------------------------------------------------------ exact regime vs the oracle
@pytest.mark.parametrize("b", [1, 64, 1024])
@pytest.mark.parametrize("size", [4097, 8191, (1 << 16) + 1, 1 << 20, 1 << 24])
def test_rows_sampler_exact_regime_matches_oracle(size, b):
    """priorities j * 2^-10: every partial sum is exact at these sizes (total < 2^34), so the two-level prefix equals
    np.cumsum and the indices equal the oracle's bit for bit"""
    rs = np.random.RandomState(size % 1000 + b)
    p = exact_priorities(rs, size, zero_frac=0.05)
    u = uniforms(rs, b)
    idx, w = rows_run(torch.from_numpy(p).cuda(), size, size, u)
    ridx, rw = rn.per_sample(p, size, u, BETA)
    assert np.array_equal(idx.cpu().numpy(), ridx)
    check_weights(w, rw)


# ------------------------------------------------------------------------------------ zero priorities
def _zero_layout(kind, size):
    p = np.full(size, 0.25, dtype=np.float32)
    if kind == "zero_chunks":
        p[CHUNK:3 * CHUNK] = 0.0                             # two whole chunks
        p[-CHUNK - 100:] = 0.0                               # and a trailing zero chunk and a half
    elif kind == "boundary":
        for c in range(1, size // CHUNK + 1):
            p[c * CHUNK - 3:c * CHUNK + 4] = 0.0             # zeros on both sides of every chunk boundary
    elif kind == "trailing":
        p[-5:] = 0.0
    return p


@pytest.mark.parametrize("kind", ["zero_chunks", "boundary", "trailing"])
def test_rows_sampler_never_draws_a_zero_priority_row(kind):
    size = 5 * CHUNK + 321
    p = _zero_layout(kind, size)
    rs = np.random.RandomState(3)
    for b in (2, 7, 1025):
        u = uniforms(rs, b)
        u[-1] = U_TOP                                        # the last target rounds to the total
        idx, w = rows_run(torch.from_numpy(p).cuda(), size, size, u)
        idx, w = idx.cpu().numpy(), w.cpu().numpy()
        ridx, rw = rn.per_sample(p, size, u, BETA)
        assert np.all(p[idx] > 0) and np.all(np.isfinite(w)) and np.all(w > 0)
        assert idx[-1] == np.flatnonzero(p > 0)[-1]
        assert np.array_equal(idx, ridx)                     # multiples of 2^-2: the exact regime
        check_weights(torch.from_numpy(w), rw)


@pytest.mark.parametrize("size", [CHUNK + 1, 3 * CHUNK + 7, 70000])
def test_rows_sampler_wide_range_draws_positive_rows(size):
    """1e-30 .. 1e30 with zero runs: the draws are never zero-priority rows and the weights are finite"""
    rs = np.random.RandomState(size)
    p = wide_priorities(rs, size)
    u = uniforms(rs, 1025)
    idx, w = rows_run(torch.from_numpy(p).cuda(), size, size, u)
    idx = idx.cpu().numpy()
    assert np.all(p[idx] > 0) and torch.isfinite(w).all()
    assert np.all(np.diff(idx) >= 0), "strata draw rows in order"


# ------------------------------------------------------------------------------------ the live size and position
def test_rows_past_the_size_are_never_read():
    size, capacity = 2 * CHUNK + 99, 6 * CHUNK
    rs = np.random.RandomState(9)
    p = exact_priorities(rs, capacity)
    u = uniforms(rs, 1024)
    base = rows_run(torch.from_numpy(p).cuda(), capacity, size, u)
    poisoned = p.copy()
    poisoned[size:] = 3e38
    got = rows_run(torch.from_numpy(poisoned).cuda(), capacity, size, u)
    assert torch.equal(base[0], got[0]) and same_bits(base[1], got[1])
    ridx, _ = rn.per_sample(p, size, u, BETA)
    assert np.array_equal(base[0].cpu().numpy(), ridx)


def test_graph_replays_follow_the_size_and_position_scalars():
    """one captured launch, then the size scalar and pos changed between replays: each replay equals an eager call"""
    from torchrl_b200 import ops
    capacity, b, U_ = 5 * CHUNK, 256, 4
    rs = np.random.RandomState(4)
    p = torch.from_numpy(exact_priorities(rs, capacity)).cuda()
    u = torch.from_numpy(rs.rand(U_ * b)).cuda()
    sp = torch.tensor([capacity], dtype=torch.int32, device="cuda")
    pp = torch.zeros(1, dtype=torch.int32, device="cuda")
    sc = scratch_for(capacity)
    idx = torch.empty(b, dtype=torch.int64, device="cuda")
    w = torch.empty(b, dtype=torch.float32, device="cuda")
    ops.per_sample_rows(p, sp, u, pp, b, BETA, sc, idx, w)
    torch.cuda.synchronize()
    g = ops.CapturedGraph(lambda: ops.per_sample_rows(p, sp, u, pp, b, BETA, sc, idx, w))
    for size, pos in ((capacity, 0), (100, 3), (CHUNK + 1, 1), (3 * CHUNK, 2), (1, 0)):
        sp.fill_(size)
        pp.fill_(pos)
        g.replay()
        gi, gw = idx.clone(), w.clone()
        ei, ew = rows_run(p, capacity, size, u[pos * b:(pos + 1) * b].cpu().numpy())
        assert torch.equal(gi, ei) and same_bits(gw, ew), (size, pos)


# ------------------------------------------------------------------------------------ launch counts
def profile_new_entry_points():
    """[(wrapper, _lib.launch_count() delta, library kernels the profiler saw)] of one call of each new wrapper, each
    called once before it is profiled."""
    from torchrl_b200 import ops
    from tests.test_binding_layer import _launches_and_kernels
    capacity = 3 * CHUNK
    p = torch.rand(capacity, device="cuda")
    u = torch.rand(64, dtype=torch.float64, device="cuda")
    sp = torch.tensor([capacity], dtype=torch.int32, device="cuda")
    pp = torch.zeros(1, dtype=torch.int32, device="cuda")
    idx, w = torch.empty(64, dtype=torch.int64, device="cuda"), torch.empty(64, device="cuda")
    sc = scratch_for(capacity)
    q1, y = torch.randn(100, device="cuda"), torch.randn(100, device="cuda")
    osc = ops.OffPolicyScratch(100, "cuda")
    calls = {"per_sample_rows": lambda: ops.per_sample_rows(p, sp, u, pp, 64, 0.4, sc, idx, w),
             "twin_mse_loss_weighted": lambda: ops.twin_mse_loss_weighted(q1, q1, y, None, osc)}
    out = []
    for name, fn in calls.items():
        fn()
        counted, kernels = _launches_and_kernels(fn)
        out.append((name, counted, kernels))
    return out


def test_launch_counts():
    """Run in a fresh process, as tests/test_reinforce_gpu.py does, so that what the profiler records does not depend
    on what the suite ran before."""
    import json
    import os
    import subprocess
    import sys
    code = ("import json\nfrom tests.test_per_rows_gpu import profile_new_entry_points\n"
            "print(json.dumps(profile_new_entry_points()))\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-3000:]
    got = {name: (counted, kernels) for name, counted, kernels in json.loads(res.stdout.strip().splitlines()[-1])}
    assert got["per_sample_rows"][0] == len(got["per_sample_rows"][1]) == 2, got
    assert got["twin_mse_loss_weighted"][0] == len(got["twin_mse_loss_weighted"][1]) == 1, got


def test_wrapper_refuses_a_short_scratch():
    from torchrl_b200 import _lib, ops
    capacity = 3 * CHUNK
    p = torch.rand(capacity, device="cuda")
    u = torch.rand(64, dtype=torch.float64, device="cuda")
    sp = torch.tensor([capacity], dtype=torch.int32, device="cuda")
    pp = torch.zeros(1, dtype=torch.int32, device="cuda")
    idx, w = torch.empty(64, dtype=torch.int64, device="cuda"), torch.empty(64, device="cuda")
    before = _lib.launch_count()
    with pytest.raises(ValueError):
        ops.per_sample_rows(p, sp, u, pp, 64, 0.4, scratch_for(capacity)[:10], idx, w)
    assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------ deterministic priority update
def test_per_update_duplicates_take_the_last_draw_like_the_oracle():
    torch.manual_seed(11)
    b, n, R = 512, 6, 40
    td = torch.rand(b, n, device="cuda") * 4
    idx = torch.randint(0, R, (b,), device="cuda").to(torch.int64)
    base = torch.rand(R, device="cuda")

    def run():
        prio, mp = Guarded(R), Guarded(1)
        prio.t.copy_(base)
        mp.t.fill_(0.5)
        call("trl_per_update", prio.t.data_ptr(), idx.data_ptr(), td.data_ptr(), b, n, 0.6, 1e-6, mp.t.data_ptr(),
             stream())
        return [prio.check("prio"), mp.check("max_prio")]

    first = twice(run)
    for _ in range(3):
        again = run()
        assert same_bits(first[0], again[0]) and same_bits(first[1], again[1])
    # each row holds the value the kernel computes for its LAST draw: compare with a duplicate-free call per draw
    distinct = torch.arange(b, dtype=torch.int64, device="cuda")
    cand, mp = Guarded(b), Guarded(1)
    cand.t.zero_()
    mp.t.zero_()
    call("trl_per_update", cand.t.data_ptr(), distinct.data_ptr(), td.data_ptr(), b, n, 0.6, 1e-6, mp.t.data_ptr(),
         stream())
    cand = cand.check()
    want = base.clone()
    ih = idx.cpu().numpy()
    for k in range(b):
        want[ih[k]] = cand[k]
    assert same_bits(first[0], want)
    ref = base.cpu().numpy().copy()
    rmax = rn.per_update(ref, ih, td.cpu().numpy(), 0.6, 1e-6, 0.5)
    got = first[0].cpu().numpy().astype(np.float64)
    assert np.all(np.abs(got - ref) <= (14 * 2.0 ** -53 + 12 * U) * ref)   # test_per_update_matches_fp64's bound
    assert abs(float(first[1].item()) - rmax) <= 12 * U * rmax


# ------------------------------------------------------------------------------------ weighted twin MSE
@pytest.mark.parametrize("twin", [False, True])
@pytest.mark.parametrize("B", [1, 7, 4097, 65537])
def test_weighted_twin_mse_matches_fp64(B, twin):
    from torchrl_b200 import ops
    torch.manual_seed(B + twin)
    q1, q2, y = (torch.randn(B, device="cuda") * 3 for _ in range(3))
    w = torch.rand(B, device="cuda") + 0.05
    sc = ops.OffPolicyScratch(B, "cuda")
    nc = 2 if twin else 1

    def run():
        g1, g2, info, td = Guarded(B), Guarded(B), Guarded(2), Guarded(B * nc)
        call("trl_twin_mse_loss_weighted", q1.data_ptr(), q2.data_ptr() if twin else None, y.data_ptr(), w.data_ptr(),
             B, g1.t.data_ptr(), g2.t.data_ptr() if twin else None, td.t.data_ptr(), info.t.data_ptr(),
             sc.b(3), sc.t(3), stream())
        out = [g1.check("g1"), info.check("info"), td.check("td_out")]
        if twin:
            out.append(g2.check("g2"))
        return out

    out = twice(run)
    g1, info, td = out[0], out[1], out[2]
    assert sc.tickets[3].item() == 0
    qs = [q1, q2] if twin else [q1]
    gs = [g1, out[3]] if twin else [g1]
    wd, yd = w.double(), y.double()
    for k, (q, g) in enumerate(zip(qs, gs)):
        d = q.double() - yd
        d32 = (q - y).double()                               # the kernel's fp32 difference (one rounding)
        assert torch.all((g.double() - 2 * d32 * wd / B).abs() <= 4 * U * (2 * d32 * wd / B).abs())
        loss = (wd * d * d).mean().item()
        assert abs(info[k].item() - loss) <= (8 * U + B * 2.0 ** -50) * loss + 1e-30
        assert same_bits(td.reshape(B, nc)[:, k], (q - y).abs())
    if not twin:
        assert torch.isnan(info[1]) or info[1].item() == 0.0


@pytest.mark.parametrize("twin", [False, True])
def test_weighted_twin_mse_without_weights_is_the_unweighted_kernel(twin):
    from torchrl_b200 import ops
    B = 5000
    torch.manual_seed(2)
    q1, q2, y = (torch.randn(B, device="cuda") for _ in range(3))
    sc = ops.OffPolicyScratch(B, "cuda")
    a1, a2, ai = ops.twin_mse_loss(q1, q2 if twin else None, y, sc)
    b1, b2, bi = ops.twin_mse_loss_weighted(q1, q2 if twin else None, y, None, sc)
    c1, c2, ci = ops.twin_mse_loss_weighted(q1, q2 if twin else None, y, torch.ones(B, device="cuda"), sc,
                                            td_out=torch.empty(B, 2 if twin else 1, device="cuda"))
    for x, yy, z in ((a1, b1, c1), (ai, bi, ci)) + (((a2, b2, c2),) if twin else ()):
        assert same_bits(x, yy) and same_bits(x, z)
