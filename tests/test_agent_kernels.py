"""The agent-specific kernels called straight through the C ABI and compared with float64 or exact restatements of the
same operation: V-MPO's top-half selection and categorical loss, TRPO's Fisher-vector product, tangent bias /
activation step and line-search surrogate (csrc/categorical.cu), Bootstrapped DQN's loss and per-env decision
(csrc/bootstrapped.cu), the Philox path of categorical sampling, the device CartPole (csrc/cartpole.cu), the SAC value
loss (csrc/offpolicy.cu), the Polyak soft update (csrc/optim.cu) and the fp32 transpose (csrc/gemm_tf32x3.cu).

Conventions: those stated at the top of test_loss_kernels.py -- outputs inside guard regions, cross-CTA scratch of
exactly the advertised size filled with +-1e300, tickets back at zero, every call twice with identical bits, exact
results where the arithmetic is exact and a bound derived next to every random check (U = 2^-24; first-order error
analysis, doubled where second-order terms are dropped).  An fp32 library function (expf, logf) is taken to be within
the 2 ulp the CUDA documentation states, and one ulp is at most 2U relative.
The tests without the `gpu` mark check argument validation and the NumPy Philox; nothing is launched there.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import cartpole as CP
from oracle import make_golden_vmpo_categorical as G
from tests.test_layer_kernels import U, Guarded, _host_ptr, _rejects, call, lib, same_bits, stream, twice
from tests.test_loss_kernels import B_EDGES, E53, GUARD, Guarded64, close, exact, poisoned, ptr

TINY = 2.0 ** -147             # absolute error of an fp32 exp / product that underflows into the subnormals
SEL_FILL = 0xA5A5A5A5A5A5A5A5 - (1 << 64)      # the int64 guard of the selection output
MASK_FILL = 0xA5                               # the uint8 guard of the mask ring


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


# ================================================================================================ A. Philox4x32-10
M32 = np.uint64(0xFFFFFFFF)


def philox(ctr, key):
    """NumPy Philox4x32-10 (the round of csrc/common.cuh): ctr 4 arrays of uint32, key 2 arrays -> 4 uint64 arrays"""
    c = [np.asarray(x, np.uint64) & M32 for x in ctr]
    k0, k1 = (np.asarray(x, np.uint64) & M32 for x in key)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & M32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return c


def philox_gen(seed, ctr, stream_id):
    """Philox::gen: key = seed, counter = (ctr_lo, ctr_hi, stream, 0); ctr a uint64 array"""
    ctr = np.asarray(ctr, np.uint64)
    seed = np.uint64(seed)
    return philox([ctr & M32, ctr >> np.uint64(32), np.full(ctr.shape, stream_id, np.uint64), np.zeros(ctr.shape,
                                                                                                      np.uint64)],
                  [seed & M32, seed >> np.uint64(32)])


def unit24(r):
    """(r >> 8) * 2^-24 in fp32, exact: the [0, 1) uniform of the kernels"""
    return (np.asarray(r, np.uint64) >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)


def test_philox_matches_the_random123_known_answers():
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        got = philox([np.array([c], np.uint64) for c in ctr], [np.array([k], np.uint64) for k in key])
        assert [int(g[0]) for g in got] == list(want), [hex(int(g[0])) for g in got]


# ================================================================================================ B. Polyak update
POLYAK_N = [1, 3, 255, 256, 257, 4 * 132 * 256 + 1]       # the last one needs a second grid-stride pass
TAUS = [0.005, 0.001, 0.5, 1.0, 0.0]


def test_polyak_tau_complement_is_exact_in_fp32():
    """The kernel forms 1 - tau as 1.0f - f32(tau); torch multiplies by f32(1.0 - tau).  They are equal for every tau
    the configs use, so the ABI can express torch's product."""
    for tau in TAUS + [0.01, 0.02]:
        assert np.float32(1.0) - np.float32(tau) == np.float32(1.0 - tau), tau


@pytest.mark.gpu
@pytest.mark.parametrize("n", POLYAK_N)
def test_polyak_update_is_bit_exact_against_torch(n):
    """target <- target * (1 - tau) + source * tau bit for bit as torch evaluates it on the CPU (three roundings, no
    fused multiply-add), and the TF32 planes written in the same pass equal trl_split_tf32 of the new target."""
    torch.manual_seed(n)
    for i, tau in enumerate(TAUS):
        t0 = torch.randn(n) * 0.05
        s0 = t0 + torch.randn(n) * 1e-3
        want = t0 * (1.0 - tau) + s0 * tau
        for planes in (False, True):
            tg, hi, lo = Guarded(n), Guarded(n), Guarded(n)
            tg.t.copy_(t0.cuda())
            src = s0.cuda()
            call("trl_polyak_update", tg.t.data_ptr(), src.data_ptr(), n, tau, hi.t.data_ptr() if planes else None,
                 lo.t.data_ptr() if planes else None, stream())
            got = tg.check("target")
            assert same_bits(src.cpu(), s0), "source changed"
            exact(got.cpu(), want, "polyak n=%d tau=%g planes=%d" % (n, tau, planes))
            if planes:
                eh, el = Guarded(n), Guarded(n)
                call("trl_split_tf32", got.data_ptr(), n, eh.t.data_ptr(), el.t.data_ptr(), stream())
                assert same_bits(hi.check("hi"), eh.check("split hi")), "hi plane n=%d tau=%g" % (n, tau)
                assert same_bits(lo.check("lo"), el.check("split lo")), "lo plane n=%d tau=%g" % (n, tau)
            else:
                assert torch.isnan(hi.buf).all() and torch.isnan(lo.buf).all(), "planes written without being asked"


# ================================================================================================ C. transpose
TRANSPOSE_SIZES = [1, 31, 32, 33, 256, 1000]


@pytest.mark.gpu
def test_transpose_is_exact():
    for rows in TRANSPOSE_SIZES:
        for cols in TRANSPOSE_SIZES:
            x = torch.randn(rows, cols, device="cuda")
            out = Guarded(cols, rows)
            r = twice(lambda: [call("trl_transpose_f32", x.data_ptr(), out.t.data_ptr(), rows, cols, stream())
                               or out.check("out")])[0]
            exact(r, x.t().contiguous(), "transpose %dx%d" % (rows, cols))


def test_transpose_refuses_a_tile_grid_beyond_the_launch_limits(native_lib):
    """The row tiles run on grid.y (at most 65535): more than 65535 * 32 rows is an argument error, before any
    launch; so are empty sizes and null pointers."""
    buf = (ctypes.c_float * 64)()
    p = _host_ptr(buf)
    f = native_lib.trl_transpose_f32
    _rejects(native_lib, f(p, p, 65535 * 32 + 1, 1, None), "bad sizes")
    _rejects(native_lib, f(p, p, 1 << 40, 4, None), "bad sizes")
    _rejects(native_lib, f(p, p, 0, 4, None), "bad sizes")
    _rejects(native_lib, f(p, p, 4, 0, None), "bad sizes")
    _rejects(native_lib, f(None, p, 4, 4, None), "null pointer")


# ================================================================================================ D. V-MPO selection
SEL_B = [1, 2, 3, 1023, 1024, 1025, 2049, 65537]
UNIT_STD = np.float32(0.99999)          # f32(UNIT_STD + f32(1e-5)) == 1: the normalisation keeps every bit


def sel_values(kind, B, rs):
    if kind == "low_byte":              # one value and its neighbours within +-300 ulp: the last two radix digits decide
        bits = np.float32(0.75).view(np.int32) + rs.randint(-300, 301, B).astype(np.int32)
        return bits.view(np.float32)
    if kind == "signed_zero":
        return rs.choice(np.float32([-1.0, -0.0, 0.0, 1.0]), B)
    if kind == "inf":
        x = rs.randn(B).astype(np.float32)
        x[rs.rand(B) < 0.2] = np.inf
        x[rs.rand(B) < 0.2] = -np.inf
        return x
    if kind == "subnormal":
        return (rs.randint(-6, 7, B) * 2.0 ** -149).astype(np.float32)
    x = rs.randn(B).astype(np.float32)
    x[rs.rand(B) < 0.3] = np.nan
    return x


def sel_expected(vals, mean, std):
    """positions of the k = B - B // 2 largest normalised values, ties to the lower position, ascending: from
    torch.sort(descending=True, stable=True) on the CPU (NaN first, -0 == +0)"""
    v = torch.from_numpy(np.ascontiguousarray(vals, np.float32))
    advn = (v - float(mean)) / (torch.tensor(np.float32(std)) + 1e-5)
    B = v.numel()
    idx = torch.sort(advn, descending=True, stable=True).indices[:B - B // 2]
    return torch.sort(idx).values.numpy()


def run_select(adv, perm, groups, b, n, table):
    B = b * n
    k = B - B // 2
    sel = Guarded64(groups, k, dtype=torch.int64, fill=SEL_FILL)
    call("trl_vmpo_select", adv.data_ptr(), ptr(perm), groups, b, n, table.data_ptr(), sel.t.data_ptr(), stream())
    got = sel.check("sel")
    assert (got != SEL_FILL).all(), "fewer than k positions written"
    return got.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("B", SEL_B)
def test_vmpo_select_matches_a_stable_torch_sort(B):
    rs = np.random.RandomState(B)
    for kind in ("low_byte", "signed_zero", "inf", "subnormal", "nan"):
        vals = sel_values(kind, B, rs)
        table = dev(np.float32([[0.0, UNIT_STD, 0, 0]]))
        adv = dev(vals)
        got = twice(lambda: [torch.from_numpy(run_select(adv, None, 1, B, 1, table))])[0].numpy()
        np.testing.assert_array_equal(got[0], sel_expected(vals, 0.0, UNIT_STD), err_msg="%s B=%d" % (kind, B))


@pytest.mark.gpu
def test_vmpo_select_several_groups_through_perm():
    """Groups of b time rows of n envs picked through a row permutation (gather_rows order: row-major over (row, env)),
    each with its own statistics row; values mix adjacent floats, +-0 and NaN."""
    rs = np.random.RandomState(3)
    for T, n, b, groups in ((40, 3, 11, 7), (64, 17, 31, 4), (2050, 1, 2049, 2), (8, 1000, 3, 5)):
        vals = sel_values("low_byte", T * n, rs).reshape(T, n)
        vals[rs.rand(T, n) < 0.05] = 0.0
        vals[rs.rand(T, n) < 0.05] = -0.0
        vals[rs.rand(T, n) < 0.02] = np.nan
        perm = np.concatenate([rs.permutation(T) for _ in range(-(-groups * b // T))])[:groups * b].astype(np.int64)
        table = np.float32([[rs.randn() * 0.1, 0.5 + rs.rand(), 0, 0] for _ in range(groups)])
        got = run_select(dev(vals), dev(perm), groups, b, n, dev(table))
        for u in range(groups):
            g = vals[perm[u * b:(u + 1) * b]].reshape(-1)
            np.testing.assert_array_equal(got[u], sel_expected(g, table[u, 0], table[u, 1]),
                                          err_msg="T=%d n=%d b=%d group %d" % (T, n, b, u))


# ================================================================================================ E. V-MPO loss
VMPO_K = [1, 255, 256, 257, 8192, 8193, 70000]
CAT_A = [1, 6, 32]
EDGE_KINDS = ["plain", "saturate", "zero_q", "big"]


def cat_terms(z):
    """fp64 p, l = log(clamp(p, eps, 1 - eps)), the clamp mask, and the first-order bounds of the kernel's fp32 cat_row:
    expf of the rounded difference (U |x - mx| + 4U), two A-term sums, two reciprocals and two products:
    e_p <= p U (|x - mx| + 2A + 8) + TINY; log o clamp is 1 / max(p, eps)-Lipschitz and logf adds 2 ulp:
    e_l <= e_p / max(p, eps) + 4U |l|"""
    z = np.asarray(z, np.float64)
    A = z.shape[-1]
    d = z.max(-1, keepdims=True) - z
    p, l, m = G._cat(z)
    eps = float(np.finfo(np.float32).eps)
    e_p = p * U * (d + 2 * A + 8) + TINY
    # the other exps vanish against 1 in every fp32 sum: the row's maximum gets p = 1 exactly
    e_p = np.where((np.exp(-d).sum(-1, keepdims=True) - 1 < 2.0 ** -26) & (d == 0), 0.0, e_p)
    e_l = e_p / np.maximum(p, eps) + 4 * U * np.abs(l)
    risky = (np.abs(p - eps) <= 2 * e_p) | (np.abs(p - (1 - eps)) <= 2 * e_p)
    return p, l, m, e_p, e_l, risky


def vmpo_case(k, A, kind, rs):
    z = (rs.randn(k, A) * 2).astype(np.float32)
    if kind == "saturate":
        z[::2, 0] += 40.0                                     # p_0 rounds to 1 > 1 - eps: the clamp is active
    zq = (z + rs.randn(k, A) * 0.5).astype(np.float32)
    if kind == "zero_q" and A > 1:
        zq[::97, 1] -= 300.0                                  # q_1 == 0: those rows' KL is inf
        z[1::89, A - 1] -= 300.0                              # p == 0: the term is 0
    acts = rs.randint(0, A, k).astype(np.float32)
    adv = (rs.randn(k) * (30.0 if kind == "big" else 1.0)).astype(np.float32)
    table = np.float32([[0.1, 0.9, 0, 0], [-0.2, 1.3, 0, 0]])
    return z, zq, acts, adv, table


def stats_bound(x, e, what_std=True):
    """bounds of (mean, std, max/min) of values x computed with per-value errors e: the fp64 moments' own rounding
    (k E53 of the magnitudes, and the cancellation of sum x^2 - sum x * mean in the variance), the fp32 casts"""
    n = x.size
    mean = x.mean()
    e_mean = e.mean() + n * E53 * np.abs(x).mean() + U * abs(mean)
    if n < 2:
        return e_mean, None, e.max() + U * np.abs(x).max()
    sd = x.std(ddof=1)
    e_var = 4 * n * E53 * (x * x).sum() / (n - 1)
    e_sd = math.sqrt(n / (n - 1)) * e.max() + (e_var / (2 * sd) if sd > 0 else math.sqrt(e_var)) + 2 * U * sd
    return e_mean, e_sd, e.max() + U * np.abs(x).max()


@pytest.mark.gpu
@pytest.mark.parametrize("per_row", [False, True])
@pytest.mark.parametrize("A", CAT_A)
def test_vmpo_categorical_loss_matches_fp64(A, per_row):
    """All 12 info slots (2 and 3 untouched), g_logits and g_dual against G.vmpo_loss at every CTA and fold edge of k
    -- beyond 32 CTAs the last CTA's lanes loop over the partials, and every CTA recomputes phi's normaliser over all
    k rows -- with the saturated, zero-probability and large-advantage edges and stats_pos NULL (row 0)."""
    for j, k in enumerate(VMPO_K):
        kind = EDGE_KINDS[(j + A) % 4]
        rs = np.random.RandomState(1000 * A + 10 * j + per_row)
        z, zq, acts, adv, table = vmpo_case(k, A, kind, rs)
        row = 0 if j % 3 == 0 else 1
        pos = None if row == 0 else torch.ones(1, dtype=torch.int32, device="cuda")
        eta, alpha = (0.05 if kind == "big" else 0.8), 0.3
        eta_eps, alpha_eps = 0.02, 0.1
        what = "k=%d A=%d %s per_row=%d stats_pos=%s" % (k, A, kind, per_row, pos is not None)
        dz, dzq, da, dadv, dtab = dev(z), dev(zq), dev(acts), dev(adv), dev(table)
        dual = dev(np.float32([eta, alpha]))

        def run(scratch, ticket):
            g, gd, info = Guarded(k, A), Guarded(2), Guarded(12)
            call("trl_vmpo_categorical_loss", dz.data_ptr(), dzq.data_ptr(), da.data_ptr(), dadv.data_ptr(),
                 dtab.data_ptr(), ptr(pos), dual.data_ptr(), k, A, eta_eps, alpha_eps, int(per_row), g.t.data_ptr(),
                 gd.t.data_ptr(), info.t.data_ptr(), scratch, ticket, stream())
            return [g.check("g_logits"), gd.check("g_dual"), info.check("info")]
        g, gd, info = (t.cpu().numpy().astype(np.float64)
                       for t in poisoned(lib().trl_vmpo_categorical_scratch_doubles(k), run))

        advn = G.normalise(adv, table[row, 0], table[row, 1])
        want, gz, geta, galpha = G.vmpo_loss(z, zq, acts, advn, np.float32(eta), np.float32(alpha), eta_eps, alpha_eps,
                                             per_row_kl=per_row)
        p, l, m, e_p, e_l, risky = cat_terms(z)
        q, lq, _, e_q, e_lq, _ = cat_terms(zq)
        assert not risky.any(), "a probability within its error of the clamp: the case cannot decide the mask"
        pz, qz = G._softmax32(z) == 0, G._softmax32(zq) == 0
        live = ~pz & ~qz
        rows, ai = np.arange(k), acts.astype(np.int64)
        logp, e_logp = l[rows, ai], e_l[rows, ai]
        # KL_i = sum_live p (l - lq): the terms' inputs, the subtraction, the product, an A-term fp32 sum
        dl = np.where(live, l - lq, 0.0)
        e_dl = e_l + e_lq + U * np.abs(dl)
        kl_inf = (qz & ~pz).any(-1)
        e_kl = np.where(live, p * e_dl + e_p * np.abs(dl), 0).sum(-1) + (A + 1) * U * np.abs(p * dl).sum(-1)
        kl = np.where(kl_inf, np.inf, (p * dl).sum(-1))
        # phi = expf(x - mx) / se: the difference, expf, the division; se is an fp64 sum of such exps
        x = (advn / np.float32(eta)).astype(np.float64)
        dx = x.max() - x
        ex = np.exp(-dx)
        phi = ex / ex.sum()
        rel_se = U * (ex * (dx + 5)).sum() / ex.sum() + k * E53
        e_phi = phi * (U * (dx + 5) + rel_se + U)
        fin = ~kl_inf
        e_K = e_kl[fin].sum() + k * E53 * np.abs(kl[fin]).sum()
        K = kl[fin].sum()
        if per_row:
            e_K, K = e_K / k, K / k
        e0 = (e_phi * np.abs(logp) + phi * e_logp).sum() / k + alpha * e_K + k * E53 * np.abs(phi * logp).sum() / k

        def slot(i, key, bound):
            w = want[key]
            if not np.isfinite(w):
                assert (np.isnan(info[i]) and np.isnan(w)) or info[i] == w, "%s %s: %r vs %r" % (key, what, info[i], w)
            else:
                close(info[i:i + 1], w, 2 * bound + U * abs(w), "%s %s" % (key, what))
        slot(0, "Training/policy_loss", e0)
        slot(1, "Training/alpha_loss", alpha * e_K)
        assert np.isnan(info[2]) and np.isnan(info[3]), "info slots 2, 3 must stay unwritten"
        em, es, ex_ = stats_bound(logp, e_logp)
        slot(4, "logprob/mean", em)
        if k == 1:
            assert np.isnan(info[5])
        else:
            slot(5, "logprob/std", es)
        slot(6, "logprob/max", ex_)
        slot(7, "logprob/min", ex_)
        if per_row:
            if kl_inf.any():
                for i, key in zip(range(8, 11), ("mean", "std", "max")):
                    slot(i, "KL/" + key, 0.0)
                if fin.any():
                    slot(11, "KL/min", stats_bound(kl[fin], e_kl[fin])[2])
            else:
                em, es, ex_ = stats_bound(kl, e_kl)
                slot(8, "KL/mean", em)
                if k > 1:
                    slot(9, "KL/std", es)
                slot(10, "KL/max", ex_)
                slot(11, "KL/min", ex_)
        else:
            assert np.isnan(info[9]) and info[8] == info[10] == info[11], what
            slot(8, "KL/mean", e_K)
        # g_dual: eta_eps + log mean exp(x) - sum phi advn / eta, and alpha_eps - K
        e_g0 = rel_se + (e_phi * np.abs(advn)).sum() / eta + k * E53 * np.abs(phi * advn).sum() / eta
        close(gd[0:1], geta, 2 * e_g0 + U * abs(geta) + 4 * U * (abs(x.max()) + 1), "dL/deta " + what)
        if np.isinf(galpha):
            assert gd[1] == galpha, what
        else:
            close(gd[1:2], galpha, 2 * e_K + U * abs(galpha) + U * alpha_eps, "dL/dalpha " + what)
        # g_logits: -(phi / k) m_a (delta_a - p) + c p (g - sum_j p_j g_j), g = l - lq + m on the live terms
        ca = np.where(m[rows, ai] > 0, -phi / k, 0.0)
        e_ca = np.where(m[rows, ai] > 0, e_phi / k + U * np.abs(ca), 0.0)
        delta = (np.arange(A)[None, :] == ai[:, None]).astype(np.float64)
        t1 = (delta - p) * ca[:, None]
        e_t1 = np.abs(delta - p) * e_ca[:, None] + np.abs(ca)[:, None] * e_p + 2 * U * np.abs(t1)
        gj = np.where(live, l - lq + m, 0.0)
        e_gj = np.where(live, e_dl + U * np.abs(gj), 0.0)
        spg = (p * gj).sum(-1, keepdims=True)
        e_spg = (p * e_gj + e_p * np.abs(gj)).sum(-1, keepdims=True) + (A + 1) * U * np.abs(p * gj).sum(-1,
                                                                                                        keepdims=True)
        c = alpha / k if per_row else alpha
        t2 = c * p * (gj - spg)
        e_t2 = c * (e_p * np.abs(gj - spg) + p * (e_gj + e_spg)) + 4 * U * np.abs(t2)
        assert np.isfinite(g).all(), what
        close(torch.from_numpy(g), gz, 2 * (e_t1 + e_t2) + U * np.abs(gz), "g_logits " + what)


# ================================================================================================ F. TRPO kernels
FVP_M = [1, 255, 256, 257, 70000]
FVP_A = [1, 2, 31, 32]


@pytest.mark.gpu
@pytest.mark.parametrize("A", FVP_A)
def test_categorical_fisher_vp_matches_fp64(A):
    """g = scale * p * (t - <p, t>) with p a max-subtracted softmax, logits spread so that some p underflow to 0;
    scale = 0 gives exact zeros.  Bound: e_p <= p U (|x - mx| + A + 4) + TINY (expf, an A-term sum, a reciprocal, a
    product); <p, t> adds A U sum |p t| and sum e_p |t|; the difference, the product and the scaling one rounding
    each."""
    for j, M in enumerate(FVP_M):
        rs = np.random.RandomState(100 * A + j)
        z = (rs.randn(M, A) * (40.0 if j % 2 else 3.0)).astype(np.float32)
        t = rs.randn(M, A).astype(np.float32)
        for scale in (0.37, 0.0):
            dz, dt = dev(z), dev(t)
            out = Guarded(M, A)
            got = twice(lambda: [call("trl_categorical_fisher_vp", dz.data_ptr(), dt.data_ptr(), M, A, scale,
                                      out.t.data_ptr(), stream()) or out.check("g")])[0].cpu().double().numpy()
            what = "M=%d A=%d scale=%g" % (M, A, scale)
            if scale == 0.0:
                assert (got == 0).all(), what
                continue
            zz = z.astype(np.float64)
            d = zz.max(-1, keepdims=True) - zz
            p = np.exp(-d) / np.exp(-d).sum(-1, keepdims=True)
            e_p = p * U * (d + A + 4) + TINY
            tt = t.astype(np.float64)
            pt = (p * tt).sum(-1, keepdims=True)
            e_pt = (e_p * np.abs(tt)).sum(-1, keepdims=True) + A * U * np.abs(p * tt).sum(-1, keepdims=True)
            want = scale * p * (tt - pt)
            e = scale * (e_p * np.abs(tt - pt) + p * (e_pt + U * np.abs(tt - pt))) + 2 * U * np.abs(want)
            if j % 2:
                assert (got == 0).any(), "wide logits should underflow some p to 0"
            close(torch.from_numpy(got), want, 2 * e + TINY, what)


TANGENT_SHAPES = [(S, C) for S in (1, 2, 3, 400) for C in (1, 3, 7, 32)]


def tangent_expected(t, db, y, C, S, act):
    tb = t.view(-1, C, S) + db.view(1, C, 1)
    if act == 1:
        tb = tb * (1 - y.view(-1, C, S) * y.view(-1, C, S))
    elif act == 2:
        tb = tb * (y.view(-1, C, S) > 0)
    return tb.reshape(-1)


def tangent_run(t, db, y, M, C, S, act, t_off=0, y_off=0):
    """t (and y) copied into NaN-guarded buffers shifted by t_off (y_off) elements; returns t after the call"""
    n = M * C * S
    tg = Guarded(n, offset=t_off)
    tg.t.copy_(t.cuda())
    yd = None
    if y is not None:
        yb = torch.full((n + 8,), float("nan"), device="cuda")
        yd = yb[4 + y_off:4 + y_off + n]
        yd.copy_(y.cuda())
    dbd = db.cuda()
    call("trl_tangent_bias_act", tg.t.data_ptr(), dbd.data_ptr(), ptr(yd), M, C, S, act, stream())
    out = tg.check("t").cpu()
    assert same_bits(dbd.cpu(), db), "db changed"
    if yd is not None:
        assert same_bits(yd.cpu(), y), "y changed"
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("S,C", TANGENT_SHAPES)
def test_tangent_bias_act_is_bit_exact_against_torch(S, C):
    """(t + db[c]) * (1 - y*y), (t + db[c]) * (y > 0) and t + db[c] bit for bit as torch evaluates them on the CPU:
    the float4 path (n % 4 == 0, aligned) and the scalar path, forced by a one-element offset of t or of y and by
    n % 4 != 0; a channel change inside a float4 when S < 4."""
    torch.manual_seed(10 * S + C)
    for M in (1, 4, 5, 33):
        n = M * C * S
        t = torch.randn(n)
        db = torch.randn(C)
        y = torch.tanh(torch.randn(n))
        y[::5] = 0.0
        for act in (0, 1, 2):
            want = tangent_expected(t, db, y, C, S, act)
            yy = y if act else None
            for t_off, y_off in ((0, 0), (1, 0), (0, 1)):
                if act == 0 and y_off:
                    continue
                got = tangent_run(t, db, yy, M, C, S, act, t_off, y_off)
                exact(got, want, "S=%d C=%d M=%d act=%d offsets=(%d,%d) n%%4=%d" % (S, C, M, act, t_off, y_off, n % 4))


@pytest.mark.gpu
def test_tangent_bias_act_over_several_grid_stride_passes():
    """n ~ 5e6 is more than two passes of the 2112-CTA float4 grid (2112 * 256 * 4) and nine of the scalar one."""
    torch.manual_seed(7)
    for M, C, S, t_off in ((1221, 32, 128, 0), (1221, 32, 128, 1), (555557, 3, 3, 0)):
        n = M * C * S
        t, db, y = torch.randn(n), torch.randn(C), torch.tanh(torch.randn(n))
        for act in (1, 2):
            got = tangent_run(t, db, y, M, C, S, act, t_off)
            exact(got, tangent_expected(t, db, y, C, S, act), "n=%d act=%d t_off=%d" % (n, act, t_off))


SURR_M = [1, 256, 257, 8193, 70000]


@pytest.mark.gpu
@pytest.mark.parametrize("M", SURR_M)
def test_categorical_surrogate_matches_fp64(M):
    """out = -mean(exp(logp - logp_old) * advn) with A = 32, sentinel scratch of ceil(M / 256) doubles, the output in
    a guard.  Per row: logp within e_l (cat_terms), the difference U |d|, expf 4U, the product U: e_term <=
    |advn| r (e_l + U |d| + 4U) + U |term|; the fp64 sum adds M E53 sum |term|."""
    A = 32
    rs = np.random.RandomState(M)
    z = (rs.randn(M, A) * 2).astype(np.float32)
    z[::3, 5] += 40.0
    acts = rs.randint(0, A, M).astype(np.float32)
    p, l, m, e_p, e_l, _ = cat_terms(z)
    logp = l[np.arange(M), acts.astype(np.int64)]
    old = (logp + rs.randn(M) * 0.2).astype(np.float32)
    advn = rs.randn(M).astype(np.float32)
    dz, da, do, dv = dev(z), dev(acts), dev(old), dev(advn)

    def run(scratch, ticket):
        out = Guarded(1)
        call("trl_categorical_surrogate", dz.data_ptr(), da.data_ptr(), do.data_ptr(), dv.data_ptr(), M, A,
             out.t.data_ptr(), scratch, ticket, stream())
        return [out.check("out")]
    got = poisoned(-(-M // 256), run)[0]
    d = logp - old.astype(np.float64)
    r = np.exp(d)
    term = r * advn
    e = np.abs(advn) * r * (e_l[np.arange(M), acts.astype(np.int64)] + U * np.abs(d) + 4 * U) + U * np.abs(term)
    want = -term.mean()
    close(got, want, 2 * e.mean() + M * E53 * np.abs(term).mean() + U * abs(want), "surrogate M=%d" % M)


@pytest.mark.gpu
def test_categorical_surrogate_is_nan_for_an_invalid_action():
    """An action that is not an integer in [0, A) has no log-probability: cat_pick gives NaN and so does the score."""
    M, A = 300, 32
    z = torch.randn(M, A, device="cuda")
    old, advn = torch.zeros(M, device="cuda"), torch.ones(M, device="cuda")
    for bad in (32.0, -1.0, 1.5, float("nan")):
        acts = torch.zeros(M, device="cuda")
        acts[77] = bad

        def run(scratch, ticket):
            out = Guarded(1)
            call("trl_categorical_surrogate", z.data_ptr(), acts.data_ptr(), old.data_ptr(), advn.data_ptr(), M, A,
                 out.t.data_ptr(), scratch, ticket, stream())
            return [out.check("out")]
        assert torch.isnan(poisoned(-(-M // 256), run)[0]).all(), "action %r" % bad


# ================================================================================================ G. Bootstrapped DQN
BOOT_B = [1, 255, 256, 257, 8193, 70000]
BOOT_H = [1, 10, 32]
BOOT_A = [2, 18, 33]


def boot_loss_run(pred, nxt, acts, rew, term, masks, B, H, A, gamma):
    def run(scratch, ticket):
        g, info = Guarded(H, B, A), Guarded(3)
        call("trl_bootstrapped_dqn_loss", pred.data_ptr(), nxt.data_ptr(), acts.data_ptr(), rew.data_ptr(),
             term.data_ptr(), masks.data_ptr(), B, H, A, gamma, g.t.data_ptr(), info.t.data_ptr(), scratch, ticket,
             stream())
        return [g.check("grad"), info.check("info")]
    return poisoned(lib().trl_offpolicy_scratch_doubles(B), run)


@pytest.mark.gpu
@pytest.mark.parametrize("H", BOOT_H)
@pytest.mark.parametrize("B", BOOT_B)
def test_bootstrapped_dqn_loss_matches_fp64(B, H):
    """loss = mean_b sum_h m_bh (Q_h(s, a) - y_h)^2 / H, y_h = r + gamma (1 - d) max Q'_h; mask and terminal bytes 2
    and 255 count as on / terminal; gamma 0 and 1; every grad element written.  Bounds: y within 3U |gamma max| + U |y|
    (two products and the sum, contracted or not), d = q - y adds U |d|; the gradient 2 d / B / H adds 3U |g|; the
    loss sums fp64 squares of fp32 d: 2 |d| e_d + U d^2 per term."""
    A = BOOT_A[(B + H) % 3]
    for gamma in (0.99, 0.0, 1.0):
        rs = np.random.RandomState(B * 7 + H + int(gamma * 100))
        pred = rs.randn(H, B, A).astype(np.float32)
        nxt = rs.randn(H, B, A).astype(np.float32)
        acts = rs.randint(0, A, B).astype(np.float32)
        rew = rs.randn(B).astype(np.float32)
        term = rs.choice(np.uint8([0, 0, 0, 1, 2, 255]), B)
        masks = rs.choice(np.uint8([0, 0, 1, 2, 255]), (B, H))
        g, info = boot_loss_run(dev(pred), dev(nxt), dev(acts), dev(rew), dev(term), dev(masks), B, H, A, gamma)
        g, info = g.cpu().double().numpy(), info.cpu().double().numpy()
        what = "B=%d H=%d A=%d gamma=%g" % (B, H, A, gamma)
        a = acts.astype(np.int64)
        q = pred.astype(np.float64)[:, np.arange(B), a]                       # (H, B)
        mx = nxt.astype(np.float64).max(-1)
        nd = (term == 0).astype(np.float64)
        gm = gamma * nd[None, :] * mx
        y = rew.astype(np.float64)[None, :] + gm
        dd = q - y
        e_d = 3 * U * np.abs(gm) + U * np.abs(y) + U * np.abs(dd)
        on = (masks.T != 0).astype(np.float64)
        loss = (on * dd * dd).sum() / (B * H)
        e_loss = (on * (2 * np.abs(dd) * e_d + U * dd * dd)).sum() / (B * H) + B * E53 * loss
        close(info[0:1], loss, 2 * e_loss + U * loss, "loss " + what)
        qm = q.mean()
        close(info[1:2], qm, B * E53 * np.abs(q).mean() + U * abs(qm), "mean q " + what)
        rm = rew.astype(np.float64).mean()
        close(info[2:3], rm, B * E53 * np.abs(rew).mean() + U * abs(rm), "mean reward " + what)
        want = np.zeros((H, B, A))
        want[:, np.arange(B), a] = on * 2 * dd / B / H
        e_g = np.zeros((H, B, A))
        e_g[:, np.arange(B), a] = on * 2 * (e_d + 3 * U * np.abs(dd)) / B / H
        assert (g[e_g == 0] == 0).all(), "off-action / masked-off gradient " + what
        close(torch.from_numpy(g), want, 2 * e_g, "grad " + what)


@pytest.mark.gpu
def test_bootstrapped_dqn_loss_drops_nan_in_the_target_max():
    """Pinned: the target's max over a' is fmaxf, which drops a NaN entry (torch.max would propagate it); a row of
    NaN only gives NaN.  DESIGN.md lists this as a deviation."""
    B, H, A = 5, 2, 3
    pred = torch.zeros(H, B, A, device="cuda")
    nxt = torch.tensor([1.0, 2.0, 3.0], device="cuda").repeat(H, B, 1)
    nxt[0, 0, 2] = float("nan")                   # max of (1, 2, nan) -> 2
    nxt[0, 1, 0] = float("nan")                   # max of (nan, 2, 3) -> 3
    nxt[1, 2, :] = float("nan")                   # all NaN -> NaN
    acts, rew = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda")
    term = torch.zeros(B, dtype=torch.uint8, device="cuda")
    masks = torch.ones(B, H, dtype=torch.uint8, device="cuda")
    g, info = boot_loss_run(pred, nxt, acts, rew, term, masks, B, H, A, 1.0)
    g = g.cpu()
    coef = np.float32(1.0 / B) / np.float32(H)                # 2 d coef, coef = (1 / B) / H in fp32
    assert g[0, 0, 0].item() == np.float32(2 * -2.0) * coef
    assert g[0, 1, 0].item() == np.float32(2 * -3.0) * coef
    assert torch.isnan(g[1, 2, 0]) and torch.isnan(info[0].cpu())


def act_expected(q, cur, head0, seed, ctr, H, A, p, u_head=None, u_mask=None):
    """heads, actions and mask rows of trl_bootstrapped_act: Philox draws (seed, (ctr << 32) + n, 0xB0075 + k / 4)[k % 4]
    with k = 0 the head draw and k = 1 + j the mask draw of head j, unless uniforms are given"""
    N = cur.size
    if u_head is None:
        c = (np.uint64(ctr) << np.uint64(32)) + np.arange(N, dtype=np.uint64)
        draws = {s: philox_gen(seed, c, 0xB0075 + s) for s in range((H + 1 + 3) // 4)}
        u = np.stack([unit24(draws[k // 4][k % 4]) for k in range(H + 1)], 1)
        u_head, u_mask = u[:, 0], u[:, 1:]
    h = np.minimum((u_head * np.float32(H)).astype(np.int64), H - 1)        # the product rounds in fp32
    head = np.where(cur == 0, h, head0)
    action = q[head, np.arange(N)].argmax(-1).astype(np.float32)             # the first maximum
    return head.astype(np.int32), action, (u_mask < np.float32(p)).astype(np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 255, 256, 257, 70000])
def test_bootstrapped_act_philox_draws_are_bit_exact(N):
    """Heads, actions and masks from the NumPy Philox, bit for bit, for H up to 32 (nine stream ids); the counter
    advances by exactly one per launch; only ring row *top is written, and heads only where current_step == 0."""
    T = 3
    for H, A in ((1, 2), (5, 18), (32, 7)):
        rs = np.random.RandomState(N + H)
        q = np.round(rs.randn(H, N, A) * 2).astype(np.float32)             # ties: the first maximum wins
        cur = np.where(rs.rand(N) < 0.5, 0, rs.randint(1, 50, N)).astype(np.int32)
        head0 = rs.randint(0, H, N).astype(np.int32)
        seed, ctr0 = 0x1234_5678_9ABC + N, 7 + H
        top = 1
        dq, dcur = dev(q), dev(cur)
        head = Guarded64(N, dtype=torch.int32, fill=-7)
        head.t.copy_(dev(head0))
        action = Guarded(N)
        ring = torch.full((T, N, H), MASK_FILL, dtype=torch.uint8, device="cuda")
        dtop = torch.tensor([top], dtype=torch.int32, device="cuda")
        counter = torch.tensor([ctr0], dtype=torch.int64, device="cuda")
        ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
        for launch in range(2):
            ctr = ctr0 + launch
            call("trl_bootstrapped_act", dq.data_ptr(), dcur.data_ptr(), head.t.data_ptr(), action.t.data_ptr(),
                 ring.data_ptr(), dtop.data_ptr(), None, None, seed, counter.data_ptr(), ticket.data_ptr(), N, H, A, 0.5,
                 stream())
            wh, wa, wm = act_expected(q, cur, head0, seed, ctr, H, A, 0.5)
            what = "N=%d H=%d launch %d" % (N, H, launch)
            np.testing.assert_array_equal(head.check("head").cpu().numpy(), wh, err_msg=what)
            np.testing.assert_array_equal(action.check("action").cpu().numpy(), wa, err_msg=what)
            r = ring.cpu().numpy()
            np.testing.assert_array_equal(r[top], wm, err_msg=what)
            assert (np.delete(r, top, 0) == MASK_FILL).all(), "a ring row other than *top was written " + what
            assert int(counter.item()) == ctr + 1, "the counter advances by one per launch"
            assert int(ticket.item()) == 0
            head0 = wh
        if N > 1000:
            assert 0.45 < wm.mean() < 0.55 and len(np.unique(wh)) == H
    call("trl_bootstrapped_act", dq.data_ptr(), dcur.data_ptr(), head.t.data_ptr(), action.t.data_ptr(),
         ring.data_ptr(), dtop.data_ptr(), None, None, seed, counter.data_ptr(), ticket.data_ptr(), 0, H, A, 0.5,
         stream())
    assert int(counter.item()) == ctr0 + 2, "N = 0 launches nothing and leaves the counter"


@pytest.mark.gpu
def test_bootstrapped_act_given_uniforms_and_u_equal_to_p():
    """u == p gives mask 0 (u < p); the head is min(floor(f32(u * H)), H - 1), u = 1 - 2^-24 included."""
    N, H, A, p = 300, 7, 5, 0.5
    rs = np.random.RandomState(0)
    q = rs.randn(H, N, A).astype(np.float32)
    cur = np.zeros(N, np.int32)
    u_head = rs.rand(N).astype(np.float32)
    u_head[:3] = [0.0, np.float32(1 - 2.0 ** -24), np.float32(3 / 7)]
    u_mask = rs.rand(N, H).astype(np.float32)
    u_mask[::4] = np.float32(p)
    head = torch.zeros(N, dtype=torch.int32, device="cuda")
    action = Guarded(N)
    ring = torch.full((2, N, H), MASK_FILL, dtype=torch.uint8, device="cuda")
    dtop = torch.tensor([0], dtype=torch.int32, device="cuda")
    dq, dcur, duh, dum = dev(q), dev(cur), dev(u_head), dev(u_mask)
    call("trl_bootstrapped_act", dq.data_ptr(), dcur.data_ptr(), head.data_ptr(), action.t.data_ptr(), ring.data_ptr(),
         dtop.data_ptr(), duh.data_ptr(), dum.data_ptr(), 0, None, None, N, H, A, p, stream())
    wh, wa, wm = act_expected(q, cur, cur, 0, 0, H, A, p, u_head, u_mask)
    np.testing.assert_array_equal(head.cpu().numpy(), wh)
    np.testing.assert_array_equal(action.check().cpu().numpy(), wa)
    np.testing.assert_array_equal(ring[0].cpu().numpy(), wm)
    assert (ring[0].cpu().numpy()[::4] == 0).all() and (ring[1].cpu().numpy() == MASK_FILL).all()


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 255, 256, 257, 70000])
def test_categorical_sample_philox_draws_are_bit_exact(M):
    """The Philox path draws u = (r[0] >> 8) 2^-24 of (seed, (ctr << 32) + m, stream 0): it must give the same bits as
    the explicit-uniform path fed the NumPy draws, and the counter is only read."""
    for A in (1, 6, 32):
        rs = np.random.RandomState(M + A)
        z = dev((rs.randn(M, A) * 2).astype(np.float32))
        seed, ctr = 987654321 + A, 3 + M
        counter = torch.tensor([ctr], dtype=torch.int64, device="cuda")
        c = (np.uint64(ctr) << np.uint64(32)) + np.arange(M, dtype=np.uint64)
        u = dev(unit24(philox_gen(seed, c, 0)[0]))
        outs = []
        for uu in (None, u):
            act, lp = Guarded(M), Guarded(M)
            call("trl_categorical_sample", z.data_ptr(), ptr(uu), seed, counter.data_ptr(), M, A, act.t.data_ptr(),
                 lp.t.data_ptr(), None, stream())
            outs.append((act.check("action"), lp.check("log_prob")))
        assert same_bits(outs[0][0], outs[1][0]) and same_bits(outs[0][1], outs[1][1]), "M=%d A=%d" % (M, A)
        assert int(counter.item()) == ctr


# ================================================================================================ H. CartPole
CART_N = [1, 256, 257, 8193, 70000]


def cart_states(N, rs):
    return np.stack([rs.uniform(-2.3, 2.3, N), rs.randn(N), rs.uniform(-0.19, 0.19, N), 1.5 * rs.randn(N)],
                    1).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("N", CART_N)
def test_cartpole_step_and_normobs_merge(N):
    """One step with statistics and merge_stats: states within one ulp of oracle/cartpole.py (equal for >= 99.99 %),
    flags exact away from the thresholds; invalid actions (NaN, 0.5) set action_error and leave the state bit for bit,
    -0.0 is a valid push left; batch_sums and the Chan-merged norm_* against fp64 of the states the kernel wrote,
    with partials of exactly (num_ctas, 8) sentinel doubles; the any_reset double buffer through t_ptr."""
    rs = np.random.RandomState(N)
    s0 = cart_states(N, rs)
    a = rs.randint(0, 2, N).astype(np.float32)
    a[rs.rand(N) < 0.1] = -0.0
    bad = np.zeros(N, bool)
    if N > 1:
        bad[rs.choice(N, max(1, N // 50), replace=False)] = True
        a[bad] = np.where(rs.rand(int(bad.sum())) < 0.5, np.nan, 0.5)
    max_steps = 200
    el0 = rs.randint(0, max_steps, N).astype(np.int32)
    mean0, var0, cnt0 = rs.randn(4) * 0.1, 0.5 + rs.rand(4), 1000.0
    ncta = lib().trl_cartpole_num_ctas(N)
    assert ncta == -(-N // 256)
    da = dev(a)

    def run(scratch, ticket):
        st = Guarded(N, 4)
        st.t.copy_(dev(s0))
        el = dev(el0)
        rew, done, tl = Guarded(N), Guarded64(N, dtype=torch.uint8, fill=MASK_FILL), \
            Guarded64(N, dtype=torch.uint8, fill=MASK_FILL)
        err = torch.zeros(1, dtype=torch.int32, device="cuda")
        bs = Guarded64(8)
        nm, nv, nc = dev(mean0), dev(var0), dev(np.array([cnt0]))
        any_reset = torch.tensor([5, 0], dtype=torch.int32, device="cuda")
        t_ptr = torch.tensor([3], dtype=torch.int32, device="cuda")
        call("trl_cartpole_step", st.t.data_ptr(), da.data_ptr(), el.data_ptr(), None, rew.t.data_ptr(),
             done.t.data_ptr(), tl.t.data_ptr(), err.data_ptr(), scratch, bs.t.data_ptr(), nm.data_ptr(), nv.data_ptr(),
             nc.data_ptr(), ticket, any_reset.data_ptr(), t_ptr.data_ptr(), N, 1.0, max_steps, 1 << 30, 1, stream())
        return [st.check("state"), rew.check("reward"), done.check("done").int(), tl.check("time_limit").int(), el, err,
                bs.check("batch_sums"), nm, nv, nc, any_reset]
    st, rew, done, tl, el, err, bs, nm, nv, nc, anyr = (t.cpu().numpy() for t in poisoned(ncta * 8, run))
    assert err[0] == int(bad.any())
    np.testing.assert_array_equal(st[bad].view(np.uint32), s0[bad].view(np.uint32))
    good = ~bad
    av = np.where(a == 1.0, 1.0, 0.0).astype(np.float32)
    ws, wr, wd, wtl, wel = CP.step(s0, av, el0, max_steps)
    ws = np.where(bad[:, None], s0, ws)
    diff = np.abs(st.astype(np.float64) - ws.astype(np.float64))
    ulp = np.spacing(np.abs(ws)).astype(np.float64)
    assert (diff <= ulp).all() and (st == ws).mean() >= 0.9999
    np.testing.assert_array_equal(el, el0 + 1)
    np.testing.assert_array_equal(rew, np.ones(N, np.float32))
    wd = np.where(bad, (el0 + 1) >= max_steps, wd)
    far = ~((np.abs(np.abs(ws[:, 0].astype(np.float64)) - CP.X_THRESHOLD) <= ulp[:, 0]) |
            (np.abs(np.abs(ws[:, 2].astype(np.float64)) - CP.THETA_THRESHOLD) <= ulp[:, 2]))
    np.testing.assert_array_equal(done[far] != 0, np.asarray(wd, bool)[far])
    np.testing.assert_array_equal(tl != 0, (done != 0) & (el == max_steps))
    assert anyr[1] == int(done.any()) and anyr[0] == 0, anyr
    # the moments: fp64 sums along a tree of depth <= 5 + 8 + ceil(ncta / 32) + 5
    x = st.astype(np.float64)
    depth = 18 + -(-ncta // 32)
    s, q = (np.array([math.fsum(c) for c in v.T]) for v in (x, x * x))      # correctly rounded references
    e_s, e_q = depth * E53 * np.abs(x).sum(0), depth * E53 * q
    close(torch.from_numpy(bs[:4]), s, e_s, "batch sums N=%d" % N)
    close(torch.from_numpy(bs[4:]), q, e_q, "batch sums of squares N=%d" % N)
    bm = s / N
    bv = np.maximum(q / N - bm * bm, 0.0)
    e_bm = e_s / N + E53 * np.abs(bm)
    e_bv = e_q / N + 2 * np.abs(bm) * e_bm + 4 * E53 * (q / N + bm * bm)
    tot = cnt0 + N
    delta = bm - mean0
    m2 = var0 * cnt0 + bv * N + delta * delta * cnt0 * N / tot
    e_mean = e_bm * N / tot + 4 * E53 * (np.abs(mean0) + np.abs(delta))
    e_var = (e_bv * N + 2 * np.abs(delta) * e_bm * cnt0 * N / tot) / tot + 8 * E53 * m2 / tot
    close(torch.from_numpy(nm), mean0 + delta * N / tot, 2 * e_mean, "norm_mean N=%d" % N)
    close(torch.from_numpy(nv), m2 / tot, 2 * e_var, "norm_var N=%d" % N)
    assert nc[0] == tot


@pytest.mark.gpu
def test_cartpole_step_without_statistics():
    """partial = NULL: no moments (and no ticket needed); the step and the any_reset flag are unchanged, without t_ptr
    slot 0 is written and slot 1 cleared."""
    N = 1000
    rs = np.random.RandomState(1)
    s0 = cart_states(N, rs)
    s0[0, 0] = 2.39
    s0[0, 1] = 5.0                                             # leaves the track
    a = rs.randint(0, 2, N).astype(np.float32)
    st = dev(s0)
    el = torch.zeros(N, dtype=torch.int32, device="cuda")
    rew, err = torch.zeros(N, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    done, tl = (torch.zeros(N, dtype=torch.uint8, device="cuda") for _ in range(2))
    anyr = torch.tensor([0, 1], dtype=torch.int32, device="cuda")
    da = dev(a)
    call("trl_cartpole_step", st.data_ptr(), da.data_ptr(), el.data_ptr(), None, rew.data_ptr(), done.data_ptr(),
         tl.data_ptr(), err.data_ptr(), None, None, None, None, None, None, anyr.data_ptr(), None, N, 2.0, 500,
         1 << 30, 1, stream())
    ws, wr, wd, wtl, wel = CP.step(s0, a, np.zeros(N), 500, 2.0)
    got = st.cpu().numpy()
    assert (np.abs(got.astype(np.float64) - ws) <= np.spacing(np.abs(ws))).all()
    np.testing.assert_array_equal(rew.cpu().numpy(), wr)
    assert done[0].item() == 1 and err.item() == 0
    assert anyr.tolist() == [1, 0]


# ================================================================================================ I. SAC value loss
@pytest.mark.gpu
@pytest.mark.parametrize("B", B_EDGES)
def test_sac_v_loss_under_guards_and_sentinels(B):
    """The fp64 cases of test_sac_v.py (its restatement and bounds) with every output in a guard, +-1e300 scratch of
    exactly trl_offpolicy_scratch_doubles(B), the ticket back at zero and identical bits on repeat."""
    from tests.test_sac_v import _np_sac_v
    for twin, rep, dev_alpha in ((True, True, True), (True, False, True), (False, True, False), (False, False, True)):
        rs = np.random.RandomState(B + 7 * twin + 3 * rep)
        lp, q1, q2, v = (rs.randn(B).astype(np.float32) for _ in range(4))
        q2[::3] = q1[::3]
        la = dev(np.float32([-0.4])) if dev_alpha else None
        alpha = float(torch.exp(la).item()) if dev_alpha else 1.0
        dl, d1, d2, dv = dev(lp), dev(q1), dev(q2), dev(v)

        def run(scratch, ticket):
            g_lp, g1, g2, g_v, info = Guarded(B), Guarded(B), Guarded(B), Guarded(B), Guarded(6)
            call("trl_sac_v_loss", dl.data_ptr(), d1.data_ptr(), d2.data_ptr() if twin else None, dv.data_ptr(),
                 ptr(la), 1.0, int(rep), B, g_lp.t.data_ptr(), g1.t.data_ptr(), g2.t.data_ptr() if twin else None,
                 g_v.t.data_ptr(), info.t.data_ptr(), scratch, ticket, stream())
            out = [g_lp.check("g_logp"), g1.check("g_qn1"), g_v.check("g_v"), info.check("info")]
            if twin:
                out.append(g2.check("g_qn2"))
            else:
                assert torch.isnan(g2.buf).all(), "g_qn2 written without a second critic"
            return out
        outs = [t.cpu().numpy() for t in poisoned(lib().trl_offpolicy_scratch_doubles(B), run)]
        g_lp, g1, g_v, info = outs[:4]
        loss, vl, e_lp, e1, e2, e_v, st = _np_sac_v(lp, q1, q2 if twin else None, v, alpha, rep)
        what = "B=%d twin=%d rep=%d" % (B, twin, rep)
        assert abs(info[0] - loss) <= 1e-5 * max(1.0, abs(loss)), what
        assert abs(info[1] - vl) <= 1e-5 * max(1.0, abs(vl)), what
        np.testing.assert_allclose(info[[2, 4, 5]], [st[0], st[2], st[3]], rtol=1e-5, atol=1e-6, err_msg=what)
        if B == 1:
            assert np.isnan(info[3])
        else:
            np.testing.assert_allclose(info[3], st[1], rtol=1e-5, err_msg=what)
        np.testing.assert_allclose(g_lp, e_lp, rtol=1e-5, atol=5e-6 / B, err_msg=what)
        np.testing.assert_allclose(g1, e1, rtol=1e-6, atol=0, err_msg=what)
        np.testing.assert_allclose(g_v, e_v, rtol=1e-5, atol=5e-6 / B, err_msg=what)
        if twin:
            np.testing.assert_allclose(outs[4], e2, rtol=1e-6, atol=0, err_msg=what)


# ================================================================================================ J. validation
def test_agent_kernels_reject_bad_arguments(native_lib):
    buf = (ctypes.c_float * 256)()
    p = _host_ptr(buf)
    p = p + (-p % 16)
    L = native_lib
    _rejects(L, L.trl_polyak_update(p, p, -1, 0.005, None, None, None), "negative size")
    _rejects(L, L.trl_polyak_update(None, p, 8, 0.005, None, None, None), "null pointer")
    _rejects(L, L.trl_polyak_update(p, p, 8, 0.005, p, None, None), "given together")
    assert L.trl_polyak_update(None, None, 0, 0.005, None, None, None) == 0
    for g, b, n in ((0, 4, 1), (1, 0, 1), (1, 4, 0), (1, 1 << 16, 1 << 15)):
        _rejects(L, L.trl_vmpo_select(p, None, g, b, n, p, p, None), "bad sizes")
    _rejects(L, L.trl_vmpo_select(p, None, 1, 4, 1, None, p, None), "null pointer")
    for k, a in ((0, 6), (8, 0), (8, 33)):
        _rejects(L, L.trl_vmpo_categorical_loss(p, p, p, p, p, None, p, k, a, 0.0, 0.0, 0, p, p, p, p, p, None),
                 "bad sizes")
    _rejects(L, L.trl_vmpo_categorical_loss(p, p, p, p, None, None, p, 8, 6, 0.0, 0.0, 0, p, p, p, p, p, None),
             "null pointer")
    for a in (0, 33):
        _rejects(L, L.trl_categorical_fisher_vp(p, p, 8, a, 1.0, p, None), "bad sizes")
        _rejects(L, L.trl_categorical_surrogate(p, p, p, p, 8, a, p, p, p, None), "bad sizes")
    _rejects(L, L.trl_categorical_fisher_vp(p, p, -1, 4, 1.0, p, None), "bad sizes")
    _rejects(L, L.trl_categorical_surrogate(p, p, p, p, 0, 4, p, p, p, None), "bad sizes")
    _rejects(L, L.trl_categorical_surrogate(p, p, p, p, 8, 4, p, None, p, None), "null pointer")
    for M, C, S, act in ((-1, 1, 1, 0), (1, 0, 1, 0), (1, 1, 0, 0), (1, 1, 1, 3)):
        _rejects(L, L.trl_tangent_bias_act(p, p, p, M, C, S, act, None), "bad sizes")
    _rejects(L, L.trl_tangent_bias_act(p, p, None, 4, 1, 1, 1, None), "null pointer")
    for B, H, A in ((0, 1, 2), (4, 0, 2), (4, 1, 1)):
        _rejects(L, L.trl_bootstrapped_dqn_loss(p, p, p, p, p, p, B, H, A, 0.99, p, p, p, p, None), "bad sizes")
    _rejects(L, L.trl_bootstrapped_dqn_loss(p, p, p, p, p, None, 4, 1, 2, 0.99, p, p, p, p, None), "null pointer")
    act = L.trl_bootstrapped_act
    _rejects(L, act(p, p, p, p, p, p, None, None, 0, p, p, -1, 2, 2, 0.5, None), "bad sizes")
    _rejects(L, act(p, p, p, p, p, p, None, None, 0, p, p, 4, 0, 2, 0.5, None), "bad sizes")
    _rejects(L, act(p, p, p, p, p, p, None, None, 0, p, p, 4, 2, 2, 1.5, None), "outside [0, 1]")
    _rejects(L, act(p, p, p, p, p, p, p, None, 0, p, p, 4, 2, 2, 0.5, None), "u_head and u_mask")
    _rejects(L, act(p, p, p, p, p, p, None, None, 0, p, None, 4, 2, 2, 0.5, None), "rng_counter and ticket")
    _rejects(L, L.trl_categorical_sample(p, None, 0, None, 8, 4, p, None, None, None), "needs u or rng_counter")
    step = L.trl_cartpole_step
    _rejects(L, step(*[p] * 8, p, None, p, p, p, None, None, None, 8, 1.0, 200, 100, 0, None), "without a ticket")
    _rejects(L, step(*[p] * 8, p, None, None, p, p, p, None, None, 8, 1.0, 200, 100, 1, None), "merge_stats needs")
    _rejects(L, step(*[p] * 8, None, None, None, None, None, None, None, p, 8, 1.0, 200, 100, 0, None),
             "t_ptr given without")
    _rejects(L, step(*[p] * 8, None, None, None, None, None, None, None, None, 8, 1.0, 0, 100, 0, None), "bad sizes")
    _rejects(L, step(p, None, *[p] * 6, None, None, None, None, None, None, None, None, 8, 1.0, 200, 100, 0, None),
             "null pointer")
