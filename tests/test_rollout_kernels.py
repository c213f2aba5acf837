"""The rollout-side kernels called straight through the C ABI and compared with float64 / exact restatements of the same
operation: the GAE and discounted-return scans (trl_gae_scan, trl_discount_return: the serial kernel, the chunked kernel
with one or four envs per lane in csrc/gae.cu, the persistent TMA kernel in csrc/gae_tma.cu and the automatic choice
between them), the synthetic continuous-control env (trl_synth_env_step, trl_synth_env_reset, trl_synth_env_seed in
csrc/env_step.cu, against oracle/synth_env.py) and the synthetic Atari env (trl_synth_atari_step, trl_synth_atari_reset
in csrc/atari_env.cu, against oracle/synth_atari.py).

Conventions (those of test_layer_kernels.py, test_loss_kernels.py and test_data_path_kernels.py):
  * every output is a view inside a guard region that must be unchanged after the call: NaN for float outputs, the byte
    0xA5 for byte and integer outputs;
  * every case runs twice and both runs must give identical bits; the cross-CTA scratch of the env step is exactly as
    long as its size query says and runs once filled with +1e300 and once with -1e300;
  * every ticket is back at zero after each call, and every input is bit-unchanged;
  * small-integer and dyadic cases must match the exact result bit for bit; random cases are checked against float64
    with a bound derived next to each check (U = 2^-24, first-order error analysis, doubled for the dropped
    second-order terms).
The tests without the `gpu` mark check argument validation; nothing is launched there.

Assumption stated here once: tanhf (the env dynamics' tanh, built without fast-math) is within 2 ulp of tanh, the
maximum error the CUDA Math API documents for it.

Found by these tests and fixed with them: trl_synth_env_step computed its shared-memory size in `int`, so an obs_dim of
23138 or more wrapped it negative and passed the 227 KB check (test_synth_env_rejects_bad_arguments); and it compared
only the dynamic shared memory with both limits, leaving out the kernel's own static shared memory.  A size that fits
227 KB alone failed in cudaFuncSetAttribute instead of being refused as an argument error
(test_synth_env_step_at_the_shared_memory_limit), and a size just under 48 KB alone, (81, 4), got no opt-in and its
launch failed (test_synth_env_step_matches_fp64[33-81-4]).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import ref_numpy as rn
from oracle import synth_atari as oa
from oracle import synth_env as se
from tests.test_data_path_kernels import GuardedBytes
from tests.test_layer_kernels import U, Guarded, _host_ptr, _rejects, assert_within, call, lib, same_bits, stream, \
    twice
from tests.test_loss_kernels import Guarded64, Scratch

TRL_EINVAL, TRL_EUNSUPPORTED = -1, -3
E53 = 2.0 ** -53
M32 = 0xFFFFFFFF
SMEM_LIMIT = 227 * 1024
F32 = lambda v: float(np.float32(v))       # a constant as the kernels see it


def u32_dev(a):
    """uint32 values as the int32 device tensor the kernels read as unsigned"""
    return torch.from_numpy(np.asarray(a, dtype=np.uint32).view(np.int32).copy()).cuda()


def u32_host(t):
    return t.cpu().numpy().view(np.uint32).astype(np.int64)


def unchanged(before, after, what):
    for i, (b, a) in enumerate(zip(before, after)):
        assert torch.equal(b.reshape(-1).view(torch.uint8), a.reshape(-1).view(torch.uint8)), \
            "%s: input %d was modified" % (what, i)


def as_bytes(t):
    """a byte output as int32, so that twice() can compare it word by word"""
    return t.to(torch.int32)


# ======================================================================================== A. GAE and discounted returns
GAE, DISC = "gae", "disc"
GAE_T = [1, 2, 3, 4, 5, 63, 64, 65, 127, 128, 129, 256, 257, 1000]
GAE_N = [1, 3, 4, 5, 31, 32, 33, 127, 128, 129]
TC = 4                       # timesteps per warp chunk, in both kernels (gae.cu TC template argument, gae_tma.cu kTC)


def dev_array(a, dtype, off=0):
    """a 1-D device copy of `a` starting `off` bytes past a 16-byte boundary (torch allocations are 512 B aligned)"""
    a = np.ascontiguousarray(a).reshape(-1)
    nbytes = a.size * np.dtype(a.dtype).itemsize
    buf = torch.zeros(nbytes + off + 16, dtype=torch.uint8, device="cuda")
    t = buf[off:off + nbytes].view(dtype)
    t.copy_(torch.from_numpy(a))
    return t


class Rollout:
    """A time-major (T, N) rollout on the device; the float arrays start `foff` bytes and the flag arrays `boff` bytes
    past a 16-byte boundary."""

    def __init__(self, r, v, term, tl, lv, foff=0, boff=0):
        self.T, self.N = r.shape
        self.host = (r, v, term, tl, lv)
        f = lambda x: dev_array(np.asarray(x, dtype=np.float32), torch.float32, foff)
        b = lambda x: dev_array(np.asarray(x, dtype=np.uint8), torch.uint8, boff)
        self.dev = [f(r), f(v), b(term), b(tl), f(lv)]

    def columns(self, n):
        r, v, term, tl, lv = self.host
        return Rollout(r[:, :n], v[:, :n], term[:, :n], tl[:, :n], lv[:n])


def scan_args(mode, ro, adv, ret, gamma, tau, filt, variant, T=None, N=None):
    T = ro.T if T is None else T
    N = ro.N if N is None else N
    ptrs = [x.data_ptr() for x in ro.dev] + [adv, ret]
    if mode == GAE:
        return "trl_gae_scan", ptrs + [T, N, gamma, tau, int(filt), variant, stream()]
    return "trl_discount_return", ptrs + [T, N, gamma, int(filt), variant, stream()]


def scan(mode, ro, gamma, tau, filt, variant, out_off=0):
    """(adv, ret) of one mode and variant; run twice (identical bits), outputs guarded, inputs unchanged.
    out_off: the outputs start that many floats past a 16-byte boundary."""
    before = [x.clone() for x in ro.dev]

    def run():
        adv, ret = Guarded(ro.T, ro.N, offset=out_off), Guarded(ro.T, ro.N, offset=out_off)
        name, args = scan_args(mode, ro, adv.t.data_ptr(), ret.t.data_ptr(), gamma, tau, filt, variant)
        call(name, *args)
        return [adv.check("%s adv (variant %d)" % (mode, variant)), ret.check("%s ret (variant %d)" % (mode, variant))]

    out = twice(run)
    unchanged(before, ro.dev, "%s variant %d" % (mode, variant))
    return out


def variants_for(N):
    return (0, 1, 2, 3, 4) if N % 128 == 0 else (0, 1, 2, 3)


def oracle(mode, ro, gamma, tau, filt):
    r, v, term, tl, lv = ro.host
    if mode == GAE:
        return rn.gae(r, v, term, tl, lv, gamma, tau, filt)
    return rn.discount_return(r, v, term, tl, lv, gamma, filt)


def exact_rollout(T, N, seed, chain=16, p=0.1):
    """Small-integer rewards, values and last values in [-8, 8].
    chain = 16: every env has a terminal at least every 16 steps (the last one within 16 steps of the end), so with
    gamma, tau in {1, 1/2} every result is a sum of at most 16 integer multiples of powers of 1/2: |x| <= 3 * 8 * 2 <
    2^6 and its last bit is >= 2^-15, 21 bits, exact in fp32 in any association.
    chain = None: no forced terminals, for gamma = tau = 1 only.  The sums then hold up to T + 1 integers, |x| <=
    24 T + 8 < 2^24, exact at any length, and with p = 0.01 many carries run across whole 64-step tiles and 128-step
    spans.
    Flags also sit on step 0, on step T-1 and on both flags of one step, in fixed envs."""
    rs = np.random.RandomState(seed)
    r = rs.randint(-8, 9, (T, N)).astype(np.float32)
    v = rs.randint(-8, 9, (T, N)).astype(np.float32)
    lv = rs.randint(-8, 9, N).astype(np.float32)
    term = rs.rand(T, N) < p
    tl = rs.rand(T, N) < p
    if chain is not None:
        phase = rs.randint(0, chain, N)
        term |= (np.arange(T)[:, None] + phase[None, :]) % chain == chain - 1
    term[0, 0::3] = True
    tl[T - 1, 0::2] = True
    term[T - 1, 1::4] = True
    term[T // 2, 0::5] = tl[T // 2, 0::5] = True
    return r, v, term.astype(np.uint8), tl.astype(np.uint8), lv


# (mode, gamma, tau): gamma = tau = 1 makes every coefficient 0 or 1 (long carries, chain = None); gamma = 1,
# tau = 1/2 tells gamma from gamma*tau (dyadic, chain = 16)
UNIT_COEFS = [(GAE, 1.0, 1.0), (DISC, 1.0, None)]
DYADIC_COEFS = [(GAE, 1.0, 0.5), (DISC, 0.5, None)]


def longest_carry(term):
    """the longest run of steps without a terminal, over all envs"""
    best = 0
    run = np.zeros(term.shape[1], dtype=np.int64)
    for t in range(term.shape[0]):
        run = np.where(term[t] != 0, 0, run + 1)
        best = max(best, int(run.max()))
    return best


def exact_cases(T, Ns, seed):
    unit = Rollout(*exact_rollout(T, max(Ns), seed, chain=None, p=0.01))
    dyadic = Rollout(*exact_rollout(T, max(Ns), seed + 1))
    if T > 128:
        assert longest_carry(unit.host[2]) > 128, "no carry crosses a whole 128-step span"
    cases = [(unit, c) for c in UNIT_COEFS] + [(dyadic, c) for c in DYADIC_COEFS]
    refs = [(full, mode, g, tau, f, oracle(mode, full, g, tau, bool(f))) for full, (mode, g, tau) in cases
            for f in (0, 1)]
    for N in Ns:
        for full, mode, g, tau, f, (ea, er) in refs:
            ro = full if N == full.N else full.columns(N)
            for variant in variants_for(N):
                a, r = scan(mode, ro, g, tau or 0.0, f, variant)
                what = "%s g=%s tau=%s filter=%d T=%d N=%d variant %d" % (mode, g, tau, f, T, N, variant)
                for got, want, name in ((a, ea[:, :N], "adv"), (r, er[:, :N], "ret")):
                    bad = got.cpu().numpy().astype(np.float64) != want
                    assert not bad.any(), "%s %s: %d entries differ from the exact result (first at %s)" % (
                        what, name, int(bad.sum()), tuple(np.argwhere(bad)[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("T", GAE_T)
def test_scan_exact_small_envs(T):
    """Every variant, both modes, filter on and off, N in GAE_N, against the float64 oracle bit for bit.  T covers one
    step, the 4-step chunk, the 64-step TMA tile (65-row value box) and the 128-step span of the chunked kernel on both
    sides; N = 128 runs the TMA kernel with one group, the other N the ragged vector and warp tails."""
    exact_cases(T, GAE_N, seed=T)


@pytest.mark.gpu
@pytest.mark.parametrize("T,N", [(1, 16896), (64, 17024), (65, 16896), (129, 17024), (257, 17024), (1000, 16896)])
def test_scan_exact_many_groups(T, N):
    """The TMA kernel with exactly one group per SM (N = 16896 = 132 groups) and with more groups than SMs (N = 17024,
    133 groups) over one tile, a ragged earliest tile and several tiles; the chunked kernels at the same sizes."""
    exact_cases(T, [N], seed=T + N)


def scan64(mode, ro, g, gt, filt):
    """float64 restatement with the constants the kernel holds (g = f32(gamma), gt = f32(f32(gamma) f32(tau))) and the
    error bound of the fp32 kernels, per element.

    x_t = a_t + b_t x_{t+1}.  a_t is evaluated from at most three roundings of operands whose magnitudes sum to
    alpha_t (|r| + g|V_{t+1}|nt + |V| for GAE, |r| + tl|V| for returns): |a^ - a| <= 3 U alpha_t.  b_t is exact.
    Magnitudes: X_t = alpha_t + beta_t X_{t+1}, Y_t = |x_t| + beta_t Y_{t+1} (beta = |b|, Y_T = |x_T|).
      * serial: x_t = fma(b, x_{t+1}, a^) rounds once, U|x_t|: error <= U (3 X_t + Y_t);
      * a chunk of TC steps composed as (ca, cb) and applied with one fma: ca's partial sums equal
        x_s - (prod b) x_e, adding TC U |x_e| at the chunk end e; cb is a product of TC factors, (TC - 1) U cb |x_e|;
        the fma adds U |x_s0| at the chunk start.  Each step is the start of one chunk and the end of the next, so
        each Y term carries at most 1 + 1 + (2 TC - 1) = 2 TC + 1 = 9 (both kernels use TC = 4; the tile-to-tile and
        span-to-span carries go through shared memory unrounded):
            |x^_t - x_t| <= U (3 X_t + 9 Y_t), doubled: 2 U (3 X_t + 9 Y_t);
      * the output that adds or subtracts V rounds once more: + 2 U |out|."""
    r, v, term, tl, lv = (np.asarray(x, dtype=np.float64) for x in ro.host)
    T = r.shape[0]
    nt = 1.0 - term
    x = lv.copy() if mode == DISC else np.zeros_like(lv)
    X = np.zeros_like(lv)
    Y = np.abs(x)
    xs, Xs, Ys = np.empty_like(r), np.empty_like(r), np.empty_like(r)
    vnext = lv
    for t in range(T - 1, -1, -1):
        if mode == GAE:
            m = 1.0 - tl[t] if filt else 1.0
            a = m * (r[t] + nt[t] * g * vnext - v[t])
            b = m * gt * nt[t]
            alpha = m * (np.abs(r[t]) + g * np.abs(vnext) * nt[t] + np.abs(v[t]))
        elif filt:
            a = r[t] + tl[t] * v[t]
            b = nt[t] * g * (1.0 - tl[t])
            alpha = np.abs(r[t]) + tl[t] * np.abs(v[t])
        else:
            a, b, alpha = r[t], nt[t] * g, np.abs(r[t])
        x = a + b * x
        X = alpha + b * X
        Y = np.abs(x) + b * Y
        xs[t], Xs[t], Ys[t] = x, X, Y
        vnext = v[t]
    err = 2 * U * (3 * Xs + (2 * TC + 1) * Ys)
    if mode == GAE:
        adv, ret = xs, xs + v
        return adv, ret, err, err + 2 * U * np.abs(ret)
    adv, ret = xs - v, xs
    return adv, ret, err + 2 * U * np.abs(adv), err


RANDOM_SHAPES = [(1, 5), (5, 129), (64, 128), (65, 33), (128, 4096), (129, 1024), (257, 17024), (1000, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("T,N", RANDOM_SHAPES)
def test_scan_random_within_fp64_bound(T, N):
    """gae_inputs-style data (gamma 0.99, tau 0.95, 2 % terminals, 1 % time limits): every variant within the bound of
    scan64 of the float64 result.  For these rollouts the bound is below the former blanket tolerance (rtol 1e-4,
    atol 2e-5 for GAE, 3e-5 for returns) at 90-98 % of the elements, and its median is 0.1-0.25 of it."""
    from oracle.make_golden import gae_inputs
    v, r, term, tl, lv = gae_inputs(T, N, seed=3 * T + N, p_term=0.02, p_tl=0.01)
    ro = Rollout(r[..., 0], v[..., 0], term[..., 0], tl[..., 0], lv[:, 0])
    g = F32(0.99)
    gt = F32(np.float32(0.99) * np.float32(0.95))
    for mode in (GAE, DISC):
        atol = 2e-5 if mode == GAE else 3e-5
        for f in (0, 1):
            ea, er, ba, br = scan64(mode, ro, g, gt, bool(f))
            if T * N >= 4096:
                blanket = 1e-4 * np.abs(ea) + atol
                assert np.median(ba / blanket) < 0.5 and (ba < blanket).mean() > 0.8
            dev = lambda x: torch.from_numpy(x).cuda()
            for variant in variants_for(N):
                a, rt = scan(mode, ro, 0.99, 0.95, f, variant)
                what = "%s filter=%d T=%d N=%d variant %d" % (mode, f, T, N, variant)
                assert_within(a, dev(ea), dev(ba), what + " adv")
                assert_within(rt, dev(er), dev(br), what + " ret")


def dispatch_rollout(N, foff, boff, seed):
    from oracle.make_golden import gae_inputs
    v, r, term, tl, lv = gae_inputs(129, N, seed=seed, p_term=0.02, p_tl=0.01)
    return Rollout(r[..., 0], v[..., 0], term[..., 0], tl[..., 0], lv[:, 0], foff=foff, boff=boff)


# (N, float arrays' byte offset, flag arrays' byte offset, the variant that 1 must pick); the threshold for the TMA
# and 4-wide kernels is N >= 2 * 128 * 132 = 33792 (gae.cu dispatch)
DISPATCH = [(33792, 0, 0, 4), (33796, 0, 0, 2), (33793, 0, 0, 3), (33664, 0, 0, 3), (33792, 16, 4, 2),
            (33792, 4, 4, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,foff,boff,picked", DISPATCH)
def test_scan_dispatch_picks_the_documented_kernel(N, foff, boff, picked):
    """Variant 1 equals the forced variant it is meant to pick, bit for bit, and differs in bits from each kernel it
    must not pick.  T = 129 makes the three associations differ: the serial kernel (variant 0) steps one fma at a
    time, the chunked kernels compose 4-step chunk maps over 128-step spans, the TMA kernel (variant 4) over 64-step
    tiles.  The differ-checks prove that each equality could have failed.
    The 4-wide (2) and scalar (3) chunked kernels run the same per-element arithmetic, so bits cannot tell them apart:
    they must agree bitwise, and the cases that pick 2 or 3 only establish that variant 1 took the chunked kernel.
    Variant 4 refuses a ragged N and misaligned arrays with TRL_EUNSUPPORTED and writes nothing."""
    ro = dispatch_rollout(N, foff, boff, seed=N + foff + boff)
    out_off = foff // 4
    tma_ok = N % 128 == 0 and foff % 16 == 0 and boff % 16 == 0
    # kernels of a different association that variant 1 must not have run
    others = (0, 3) if picked == 4 else ((0, 4) if tma_ok else (0,))
    for mode in (GAE, DISC):
        for f in (0, 1):
            auto = scan(mode, ro, 0.99, 0.95, f, 1, out_off)
            forced = scan(mode, ro, 0.99, 0.95, f, picked, out_off)
            for x, y, name in zip(auto, forced, ("adv", "ret")):
                assert same_bits(x, y), "%s filter=%d N=%d: variant 1 is not variant %d (%s)" % (mode, f, N, picked, name)
            for other in others:
                alt = scan(mode, ro, 0.99, 0.95, f, other, out_off)
                assert not same_bits(auto[0], alt[0]), \
                    "%s filter=%d N=%d: variant 1 cannot be told from variant %d" % (mode, f, N, other)
            v2 = scan(mode, ro, 0.99, 0.95, f, 2, out_off)
            v3 = scan(mode, ro, 0.99, 0.95, f, 3, out_off)
            for x, y in zip(v2, v3):
                assert same_bits(x, y), "%s: variants 2 and 3 differ" % mode
        if not tma_ok:
            adv, ret = Guarded(ro.T, N, offset=out_off), Guarded(ro.T, N, offset=out_off)
            name, args = scan_args(mode, ro, adv.t.data_ptr(), ret.t.data_ptr(), 0.99, 0.95, 1, 4)
            rc = getattr(lib(), name)(*args)
            assert rc == TRL_EUNSUPPORTED, rc
            assert "TMA" in lib().trl_last_error().decode()
            torch.cuda.synchronize()
            assert torch.isnan(adv.buf).all() and torch.isnan(ret.buf).all(), "variant 4 wrote after refusing"


ISO_ENVS = [0, 3, 4, 7, 127, 128, 131, 255]     # first / last lane of a 4-wide vector, first / last env of a group


@pytest.mark.gpu
@pytest.mark.parametrize("array", ["rewards", "values"])
def test_scan_keeps_envs_apart(array):
    """A NaN at (t, n) of `array` may change env n at steps <= t only; every other env, and env n after t, stays
    bit-equal to the clean run -- for every variant, both modes.  n is the first and the last lane of a 4-wide
    vector and the first and the last env of a 128-env group."""
    from oracle.make_golden import gae_inputs
    T, N, t = 129, 256, 70
    v, r, term, tl, lv = gae_inputs(T, N, seed=11, p_term=0.02, p_tl=0.01)
    host = [r[..., 0], v[..., 0], term[..., 0], tl[..., 0], lv[:, 0]]
    clean_ro = Rollout(*host)
    clean = {(m, var): scan(m, clean_ro, 0.99, 0.95, 1, var) for m in (GAE, DISC) for var in variants_for(N)}
    k = 0 if array == "rewards" else 1
    for n in ISO_ENVS:
        dirty = [h.copy() for h in host]
        dirty[k][t, n] = np.nan
        ro = Rollout(*dirty)
        for (m, var), ref in clean.items():
            for got, want, name in zip(scan(m, ro, 0.99, 0.95, 1, var), ref, ("adv", "ret")):
                keep = torch.ones(T, N, dtype=torch.bool, device="cuda")
                keep[:t + 1, n] = False
                assert same_bits(got[keep], want[keep]), \
                    "%s variant %d: a NaN at (%d, %d) of %s leaked beyond env %d's earlier steps (%s)" % (
                        m, var, t, n, array, n, name)
                if name == "adv":
                    assert torch.isnan(got[t, n]), "%s variant %d: the poisoned step is not NaN" % (m, var)


@pytest.mark.gpu
def test_scan_degenerate_sizes_write_nothing():
    """T = 0 or N = 0: every variant returns 0 and writes nothing."""
    ro = Rollout(*exact_rollout(4, 8, seed=1))
    for T, N in ((0, 8), (4, 0), (0, 0)):
        for mode in (GAE, DISC):
            for variant in (0, 1, 2, 3, 4):
                adv, ret = Guarded(4, 8), Guarded(4, 8)
                name, args = scan_args(mode, ro, adv.t.data_ptr(), ret.t.data_ptr(), 0.99, 0.95, 1, variant, T=T, N=N)
                call(name, *args)
                torch.cuda.synchronize()
                assert torch.isnan(adv.buf).all() and torch.isnan(ret.buf).all(), (mode, variant, T, N)


def test_scan_rejects_bad_arguments(native_lib):
    buf = (ctypes.c_float * 64)()
    p = _host_ptr(buf)
    p16 = p + (-p % 16)
    ptrs = [p16] * 7
    for name, extra in (("trl_gae_scan", [0.99, 0.95]), ("trl_discount_return", [0.99])):
        fn = getattr(native_lib, name)
        _rejects(native_lib, fn(*ptrs, -1, 4, *extra, 1, 1, None), "negative size")
        _rejects(native_lib, fn(*ptrs, 4, -1, *extra, 1, 1, None), "negative size")
        for i in range(7):
            nul = list(ptrs)
            nul[i] = None
            _rejects(native_lib, fn(*nul, 4, 4, *extra, 1, 1, None), "null pointer")
        _rejects(native_lib, fn(*ptrs, 4, 4, *extra, 1, 5, None), "variant 5")
        _rejects(native_lib, fn(*ptrs, 4, 4, *extra, 1, -1, None), "variant -1")
        assert fn(*([None] * 7), 0, 4, *extra, 1, 5, None) == 0      # nothing to do: no pointer or variant is read


# ================================================================================== B. synthetic continuous-control env
def env_smem(o, a):
    return lib().trl_synth_env_smem_bytes(o, a)


O_MAX = 210                  # the largest obs_dim whose shared memory fits 227 KB with act_dim 1 (checked below)
ENV_SHAPES = [(2, 1), (17, 6), (111, 8), (129, 3), (O_MAX, 1)]
# (81, 4) needs 49144 B of dynamic shared memory: under 48 KB alone, over it with the kernel's static shared memory,
# so the step must opt in.  It runs first: the opt-in is kept per process, and a larger size set earlier would cover it.
ENV_CASES = ([(33, 81, 4), (4097, 81, 4)] + [(N, o, a) for o, a in ENV_SHAPES for N in (1, 33, 4097)] +
             [(N, 17, 6) for N in (31, 32, 65537)] + [(65537, 111, 8), (65537, 129, 3)])
MAX_STEPS = 7


class EnvCase:
    """Random fp32 states and dyadic actions.  Actions are multiples of 2^-16 in [-1.25, 1.25] and ub - lb is 2 or 4,
    so NormAct's lb + (act + 1) / 2 (ub - lb) and its clip are exact in fp32 and the oracle sees the kernel's u."""

    def __init__(self, N, o, a, seed, thr=0.9, scale=1.5):
        rs = np.random.RandomState(seed)
        self.N, self.o, self.a = N, o, a
        self.A, self.B, self.c = se.make_params(o, a)
        self.s = (scale * rs.randn(N, o)).astype(np.float32)
        self.act = (rs.randint(-5 * 2 ** 14, 5 * 2 ** 14 + 1, (N, a)) / 2.0 ** 16).astype(np.float32)
        self.lb = rs.choice([-1.0, -0.5, -2.0], a).astype(np.float32)
        self.ub = (self.lb + rs.choice([2.0, 4.0], a)).astype(np.float32)
        self.elapsed = rs.choice([0, 3, MAX_STEPS - 2, MAX_STEPS - 1, MAX_STEPS, MAX_STEPS + 3], N).astype(np.int32)
        self.thr = thr
        self.reward_scale = 0.37
        d = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
        self.dev = [d(x) for x in (self.act, self.A, self.B, self.c, self.lb, self.ub)]

    def u(self):
        lb, ub = self.lb.astype(np.float64), self.ub.astype(np.float64)
        return np.clip(lb + (self.act + 1.0) * 0.5 * (ub - lb), lb, ub)


def env_step(case, partial=None, batch_sums=None, norm=(None, None, None), ticket=None, any_reset=None, t_ptr=None,
             step_count=None, max_frames=1 << 30, merge=0, thr=None):
    """one trl_synth_env_step on fresh guarded copies of the case's state; returns the guarded outputs"""
    N, o = case.N, case.o
    state = Guarded(N, o)
    state.t.copy_(torch.from_numpy(case.s))
    reward = Guarded(N)
    done, tlim = GuardedBytes(N), GuardedBytes(N)
    elapsed = GuardedBytes(4 * N, dtype=torch.int32)
    elapsed.t.copy_(torch.from_numpy(case.elapsed))
    p = lambda t: None if t is None else t.data_ptr()
    act, A, B, c, lb, ub = case.dev
    call("trl_synth_env_step", state.t.data_ptr(), act.data_ptr(), A.data_ptr(), B.data_ptr(), c.data_ptr(),
         lb.data_ptr(), ub.data_ptr(), elapsed.t.data_ptr(), p(step_count), reward.t.data_ptr(), done.t.data_ptr(),
         tlim.t.data_ptr(), p(partial), p(batch_sums), *[p(x) for x in norm], p(ticket), p(any_reset), p(t_ptr), N, o,
         case.a, se.RHO, se.ETA, se.CTRL_COST, case.thr if thr is None else thr, case.reward_scale, MAX_STEPS,
         max_frames, merge, stream())
    return state, reward, done, tlim, elapsed


def env_outputs(outs):
    state, reward, done, tlim, elapsed = outs
    return [state.check("state"), reward.check("reward"), as_bytes(done.check("done")),
            as_bytes(tlim.check("time_limit")), elapsed.check("elapsed")]


@pytest.mark.gpu
@pytest.mark.parametrize("N,o,a", ENV_CASES)
def test_synth_env_step_matches_fp64(N, o, a):
    """State, reward, done, time_limit and elapsed against oracle/synth_env.dynamics from the same fp32 state.

    z = c + s A + u B is one fma chain of o + a terms: |z^ - z| <= (o + a) U S with S = |c| + sum|s A| + sum|u B|.
    tanhf adds 2 ulp <= 4 U |tanh z|, and tanh is 1-Lipschitz.  s' = rho s + eta tanh(z) with rho = f32(0.8) (within
    U rho |s| of the oracle's 0.8), two products and a sum: U (3 rho |s| + 2 eta |t|).  Doubled:
        |s'^ - s'| <= 2 (eta (o + a) U S + U (3 rho |s| + 6 eta |t|)).
    reward = (s'_0 - ctrl sum u^2) * scale: the fma chain of a squares adds a U sum u^2, f32(0.1) and the product
    2 U ctrl sum u^2, the difference U |r|, the scale f32(0.37) and its product 2 U |r scale|; doubled.
    done must equal |s'^_1| > thr or elapsed >= max exactly, and match the oracle wherever | |s'_1| - thr | exceeds
    the state bound.  time_limit is set exactly when elapsed reaches max_episode_steps, whether or not the dynamics
    end the episode on that step too."""
    if o == O_MAX:
        assert env_smem(O_MAX, 1) <= SMEM_LIMIT < env_smem(O_MAX + 1, 1)
    if (o, a) == (81, 4):
        assert 48 * 1024 - 16 < env_smem(o, a) <= 48 * 1024
    case = EnvCase(N, o, a, seed=N + 7 * o + a)
    before = [x.clone() for x in case.dev]
    s2, rew, done, tlim, el = twice(lambda: env_outputs(env_step(case)))
    unchanged(before, case.dev, "env step")

    s = case.s.astype(np.float64)
    u = case.u()
    A, B, c = (x.astype(np.float64) for x in (case.A, case.B, case.c))
    want_s, want_r, want_dd = se.dynamics(s, u, case.A, case.B, case.c, F32(case.thr))
    S = np.abs(c) + np.abs(s) @ np.abs(A) + np.abs(u) @ np.abs(B)
    t = np.abs(np.tanh(s @ A + u @ B + c))
    rho = se.RHO
    bound_s = 2 * (se.ETA * (o + a) * U * S + U * (3 * rho * np.abs(s) + 6 * se.ETA * t))
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    assert_within(s2, dev(want_s), dev(bound_s), "state N=%d o=%d a=%d" % (N, o, a))

    usq = (u * u).sum(1)
    ctrl, rsc = se.CTRL_COST, case.reward_scale
    r_pre = want_r
    bound_r = 2 * (rsc * (bound_s[:, 0] + ctrl * (a + 2) * U * usq + U * np.abs(r_pre)) + 2 * U * np.abs(r_pre * rsc))
    assert_within(rew, dev(want_r * F32(rsc)), dev(bound_r), "reward")

    el_want = case.elapsed + 1
    got_s = s2.cpu().numpy()
    done_exact = (np.abs(got_s[:, 1]) > np.float32(case.thr)) | (el_want >= MAX_STEPS)
    np.testing.assert_array_equal(done.cpu().numpy(), done_exact.astype(np.int32))
    clear = np.abs(np.abs(want_s[:, 1]) - F32(case.thr)) > bound_s[:, 1]
    done_ref = want_dd | (el_want >= MAX_STEPS)
    np.testing.assert_array_equal(done.cpu().numpy()[clear], done_ref[clear].astype(np.int32))
    np.testing.assert_array_equal(tlim.cpu().numpy(), (el_want == MAX_STEPS).astype(np.int32))
    np.testing.assert_array_equal(el.cpu().numpy(), el_want)
    if N >= 4097:
        at_limit = el_want == MAX_STEPS
        assert (at_limit & want_dd & clear).any() and (at_limit & ~want_dd & clear).any()


@pytest.mark.gpu
def test_synth_env_step_at_the_shared_memory_limit():
    """obs_dim 137, act_dim 178 needs exactly 227 KB of dynamic shared memory, which leaves no room for the kernel's
    own static shared memory: the step must refuse it with an argument error rather than fail at the launch (it used to
    return the CUDA error of cudaFuncSetAttribute)."""
    assert env_smem(137, 178) == SMEM_LIMIT
    case = EnvCase(33, 137, 178, seed=5)
    N, o = case.N, case.o
    state, reward = Guarded(N, o), Guarded(N)
    done, tlim = GuardedBytes(N), GuardedBytes(N)
    elapsed = GuardedBytes(4 * N, dtype=torch.int32)
    act, A, B, c, lb, ub = case.dev
    rc = lib().trl_synth_env_step(state.t.data_ptr(), act.data_ptr(), A.data_ptr(), B.data_ptr(), c.data_ptr(),
                                  lb.data_ptr(), ub.data_ptr(), elapsed.t.data_ptr(), None, reward.t.data_ptr(),
                                  done.t.data_ptr(), tlim.t.data_ptr(), None, None, None, None, None, None, None, None,
                                  N, o, case.a, 0.8, 0.5, 0.1, 1.0, 1.0, 10, 1 << 30, 0, stream())
    _rejects(lib(), rc, "shared memory")
    torch.cuda.synchronize()
    assert torch.isnan(state.buf).all() and torch.isnan(reward.buf).all()


MOMENT_CASES = [(N, o, a) for o, a in ((2, 1), (17, 6), (111, 8), (129, 3)) for N in (1, 33, 4097)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,o,a", MOMENT_CASES)
def test_synth_env_step_moments(N, o, a):
    """The NormObs batch moments of the step: `partial` exactly trl_synth_env_num_ctas(N) * 2 o doubles inside +-1e300
    sentinels (both runs identical bits), batch_sums within N E53 sum|x| of math.fsum, and the Chan merge into
    norm_mean / norm_var / norm_count as in the float64 formula.  o = 2, 17 and 111 fold the partials in P parts
    (2 o <= 256), o = 129 walks the CTAs serially.  merge_stats = 0 leaves norm_* untouched; batch_sums = NULL still
    merges, to the same bits."""
    case = EnvCase(N, o, a, seed=3 * N + o)
    ncta = lib().trl_synth_env_num_ctas(N)
    assert ncta == -(-N // 32)
    rs = np.random.RandomState(o)
    mean0, var0, cnt0 = rs.randn(o), rs.rand(o) + 0.5, 37.0

    def run(fill, merge=1, sums=True):
        part = Scratch(ncta * 2 * o, fill)
        bs = Guarded64(2 * o)
        nm, nv, nc = Guarded64(o), Guarded64(o), Guarded64(1)
        nm.t.copy_(torch.from_numpy(mean0))
        nv.t.copy_(torch.from_numpy(var0))
        nc.t.fill_(cnt0)
        ticket = GuardedBytes(4, dtype=torch.int32)
        ticket.t.zero_()
        outs = env_step(case, part.t, bs.t if sums else None, (nm.t, nv.t, nc.t), ticket.t, merge=merge)
        part.check()
        assert int(ticket.check("ticket").item()) == 0, "the ticket is not back at zero"
        return env_outputs(outs) + [bs.check("batch_sums"), nm.check("norm_mean"), nv.check("norm_var"),
                                    nc.check("norm_count")]

    first, second = run(1e300), run(-1e300)
    for i, (x, y) in enumerate(zip(first, second)):
        assert same_bits(x, y), "output %d differs between the +1e300 and the -1e300 scratch" % i
    x = first[0].cpu().numpy().astype(np.float64)
    sums = first[5].cpu().numpy()
    ref = np.array([math.fsum(x[:, j]) for j in range(o)] + [math.fsum(x[:, j] ** 2) for j in range(o)])
    mag = np.concatenate([np.abs(x).sum(0), (x * x).sum(0)])
    assert (np.abs(sums - ref) <= N * E53 * mag).all(), "batch_sums beyond N E53 sum|x|"
    bm, bv = x.mean(0), x.var(0)
    tot = cnt0 + N
    delta = bm - mean0
    want_var = (var0 * cnt0 + bv * N + delta ** 2 * cnt0 * N / tot) / tot
    want_mean = mean0 + delta * N / tot
    np.testing.assert_allclose(first[6].cpu().numpy(), want_mean, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(first[7].cpu().numpy(), want_var, rtol=1e-9, atol=1e-12)
    assert first[8].item() == tot

    no_merge = run(1e300, merge=0)
    for got, init in ((no_merge[6], mean0), (no_merge[7], var0), (no_merge[8], np.array([cnt0]))):
        assert torch.equal(got.cpu(), torch.from_numpy(init)), "merge_stats = 0 changed norm_*"
    assert same_bits(no_merge[5], first[5])
    no_sums = run(-1e300, sums=False)
    assert torch.isnan(no_sums[5]).all(), "batch_sums = NULL: something was written to the guarded stand-in"
    for i in (6, 7, 8):
        assert same_bits(no_sums[i], first[i]), "batch_sums = NULL changed the merge"


@pytest.mark.gpu
@pytest.mark.parametrize("t", [0, 1, None])
def test_synth_env_step_any_reset_flag(t):
    """any_reset[t & 1] (slot 0 when t_ptr is NULL) becomes the OR over envs of done | (step_count + 1 >=
    max_episode_frames), and the slot of the next step, (t + 1) & 1, is cleared.  Cases: no env resets, only the
    surpass flag of the last env is set, the dynamics end episodes; without step_count."""
    N = 4097
    case = EnvCase(N, 17, 6, seed=21)
    case.elapsed[:] = 0
    slot = 0 if t is None else t & 1
    t_dev = None if t is None else torch.tensor([t], dtype=torch.int32, device="cuda")
    frames = 50
    counts = np.zeros(N, dtype=np.int32)
    only_last = counts.copy()
    only_last[-1] = frames - 1
    for thr, sc, want in ((3e38, counts, 0), (3e38, only_last, 1), (0.9, counts, 1), (3e38, None, 0),
                          (0.9, None, 1)):
        def run():
            flag = GuardedBytes(8, dtype=torch.int32)
            flag.t.fill_(0x5A5A)
            flag.t[slot] = 0
            sc_dev = None if sc is None else torch.from_numpy(sc).cuda()
            outs = env_step(case, any_reset=flag.t, t_ptr=t_dev, step_count=sc_dev, max_frames=frames, thr=thr)
            return env_outputs(outs) + [flag.check("any_reset")]

        outs = twice(run)
        done, flag = outs[2].cpu().numpy(), outs[5].cpu().numpy()
        surpass = False if sc is None else ((sc + 1) >= frames).any()
        assert int(bool(done.any() or surpass)) == want
        assert flag[slot] == want and flag[1 - slot] == 0, (thr, sc is not None, flag)


def reset_inputs(N, o, seed):
    rs = np.random.RandomState(seed)
    seeds = rs.randint(0, 2 ** 32, N, dtype=np.uint64).astype(np.uint32)
    episodes = rs.randint(0, 2 ** 32, N, dtype=np.uint64).astype(np.uint32)
    episodes[:3] = [0, M32, M32 - 1]
    state0 = rs.randn(N, o).astype(np.float32)
    elapsed0 = rs.randint(0, 1000, N).astype(np.int32)
    mask = (rs.rand(N) < 0.5).astype(np.uint8)
    mask[:2] = 1
    return seeds, episodes, state0, elapsed0, mask


@pytest.mark.gpu
@pytest.mark.parametrize("o", [1, 33, 111])
@pytest.mark.parametrize("masked", [True, False])
def test_synth_env_reset_matches_reset_state(o, masked):
    """Reset rows equal oracle reset_state cast to fp32 bit for bit, their episode counter advances (wrapping at
    2^32) and elapsed is 0; rows outside the mask keep state, elapsed and episode.  obs_dim 1, 33 and 111: the lanes
    of a warp stride over the features."""
    N = 1000
    seeds, episodes, state0, elapsed0, mask = reset_inputs(N, o, seed=o)
    sel = mask.astype(bool) if masked else np.ones(N, dtype=bool)
    seeds_d, mask_d = u32_dev(seeds), torch.from_numpy(mask).cuda()

    def run():
        state = Guarded(N, o)
        state.t.copy_(torch.from_numpy(state0))
        elapsed, episode = GuardedBytes(4 * N, dtype=torch.int32), GuardedBytes(4 * N, dtype=torch.int32)
        elapsed.t.copy_(torch.from_numpy(elapsed0))
        episode.t.copy_(u32_dev(episodes))
        call("trl_synth_env_reset", state.t.data_ptr(), elapsed.t.data_ptr(), episode.t.data_ptr(), seeds_d.data_ptr(),
             mask_d.data_ptr() if masked else None, N, o, se.INIT_SCALE, stream())
        return [state.check("state"), elapsed.check("elapsed"), episode.check("episode")]

    state, elapsed, episode = twice(run)
    want = state0.copy()
    want[sel] = se.reset_state(seeds[sel], episodes[sel], o).astype(np.float32)
    assert np.array_equal(state.cpu().numpy().view(np.int32), want.view(np.int32))
    np.testing.assert_array_equal(elapsed.cpu().numpy(), np.where(sel, 0, elapsed0))
    np.testing.assert_array_equal(u32_host(episode), np.where(sel, (episodes.astype(np.int64) + 1) & M32, episodes))
    assert same_bits(seeds_d, u32_dev(seeds)) and torch.equal(mask_d.cpu(), torch.from_numpy(mask))


@pytest.mark.gpu
@pytest.mark.parametrize("N,seed,n_total,first", [(1, 0, 1, 0), (1000, 0x9E3779B9, 3000000017, 0xFFFFFF00),
                                                  (257, M32, M32, M32)])
def test_synth_env_seed_is_exact(N, seed, n_total, first):
    """seeds[i] = seed * n_total + first_env + i modulo 2^32 and episodes 0, inside 0xA5 guards."""
    def run():
        seeds, episode = GuardedBytes(4 * N, dtype=torch.int32), GuardedBytes(4 * N, dtype=torch.int32)
        episode.t.fill_(-1)
        call("trl_synth_env_seed", seeds.t.data_ptr(), episode.t.data_ptr(), N, seed, n_total, first, stream())
        return [seeds.check("seeds"), episode.check("episode")]

    seeds, episode = twice(run)
    want = (((seed * n_total + first) & M32) + np.arange(N, dtype=np.int64)) & M32
    np.testing.assert_array_equal(u32_host(seeds), want)
    assert (episode == 0).all()


def test_synth_env_rejects_bad_arguments(native_lib):
    """Sizes, null pointers, statistics without a ticket or without norm_*, and an obs_dim beyond 227 KB of shared
    memory -- including obs_dim 23138 and up, whose byte count used to overflow int and pass the check."""
    buf = (ctypes.c_float * 64)()
    p = _host_ptr(buf)
    p16 = p + (-p % 16)
    fn = native_lib.trl_synth_env_step

    def step(N=4, o=17, a=6, ptrs=None, partial=None, norm=None, ticket=None, merge=0):
        ptrs = ptrs or [p16] * 8
        st, act, A, B, c, lb, ub, el = ptrs[:8]
        nm = norm or [None] * 3
        return fn(st, act, A, B, c, lb, ub, el, None, p16, p16, p16, partial, None, *nm, ticket, None, None, N, o, a,
                  0.8, 0.5, 0.1, 1.0, 1.0, 10, 1 << 30, merge, None)

    _rejects(native_lib, step(N=-1), "bad sizes")
    _rejects(native_lib, step(o=1), "bad sizes")
    _rejects(native_lib, step(a=0), "bad sizes")
    for i in range(8):
        ptrs = [p16] * 8
        ptrs[i] = None
        _rejects(native_lib, step(ptrs=ptrs), "null pointer")
    _rejects(native_lib, step(partial=p16), "ticket")
    _rejects(native_lib, step(partial=p16, ticket=p16, merge=1), "merge_stats")
    assert native_lib.trl_synth_env_smem_bytes(O_MAX, 1) <= SMEM_LIMIT < native_lib.trl_synth_env_smem_bytes(O_MAX + 1, 1)
    _rejects(native_lib, step(o=O_MAX + 1, a=1), "227 KB")
    for o in (23138, 46341, 65536, 1 << 30):
        assert native_lib.trl_synth_env_smem_bytes(o, 1) > SMEM_LIMIT
        _rejects(native_lib, step(o=o, a=1), "227 KB")
    rs = native_lib.trl_synth_env_reset
    _rejects(native_lib, rs(p16, p16, p16, p16, None, -1, 4, 0.1, None), "bad sizes")
    _rejects(native_lib, rs(p16, p16, p16, p16, None, 4, 0, 0.1, None), "bad sizes")
    _rejects(native_lib, rs(p16, p16, None, p16, None, 4, 4, 0.1, None), "null pointer")
    _rejects(native_lib, native_lib.trl_synth_env_seed(p16, p16, -1, 1, 1, 0, None), "bad size")
    _rejects(native_lib, native_lib.trl_synth_env_seed(p16, None, 4, 1, 1, 0, None), "null pointer")


# ================================================================================================ C. synthetic Atari env
LAT_KEYS = ("bx", "by", "vx", "vy", "px")
FRAME = 84 * 84
ATARI_MAX = 9


def lat_array(lat):
    return np.stack([lat[k] for k in LAT_KEYS], 1).astype(np.int32)


def random_latent(N, rs):
    """balls anywhere in the field, half of them near the paddle row (hits and misses), all velocities"""
    by = np.where(rs.rand(N) < 0.5, rs.randint(0, 80, N), rs.randint(66, 80, N))
    return {"bx": rs.randint(0, 81, N), "by": by, "vx": rs.choice([-2, -1, 1, 2], N), "vy": rs.choice([-2, -1, 1, 2], N),
            "px": rs.randint(0, 73, N)}


def atari_buffers(obs0, lat0, el0):
    N = obs0.shape[0]
    obs = GuardedBytes(N * 4 * FRAME)
    obs.t.copy_(torch.from_numpy(obs0.reshape(-1)))
    latent = GuardedBytes(4 * 5 * N, dtype=torch.int32)
    latent.t.copy_(torch.from_numpy(lat_array(lat0).reshape(-1)))
    elapsed = GuardedBytes(4 * N, dtype=torch.int32)
    elapsed.t.copy_(torch.from_numpy(el0))
    return obs, latent, elapsed


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 255, 4099])
def test_synth_atari_step_bit_exact(N):
    """One step against oracle/synth_atari.py bit for bit, every action 0..5 (env n takes (n + k) % 6 in step k of
    two), walls, hits and misses, elapsed around max_steps; obs, latent, elapsed, reward, done and time_limit inside
    0xA5 guards."""
    rs = np.random.RandomState(N)
    for k in range(2):
        lat0 = random_latent(N, rs)
        obs0 = rs.randint(0, 256, (N, 4, 84, 84)).astype(np.uint8)
        el0 = rs.choice([0, 5, ATARI_MAX - 2, ATARI_MAX - 1, ATARI_MAX + 2], N).astype(np.int32)
        act = ((np.arange(N) + k) % 6).astype(np.float32)
        act_d = torch.from_numpy(act).cuda()

        def run():
            obs, latent, elapsed = atari_buffers(obs0, lat0, el0)
            reward = GuardedBytes(4 * N, dtype=torch.float32)
            done, tlim = GuardedBytes(N), GuardedBytes(N)
            call("trl_synth_atari_step", obs.t.data_ptr(), latent.t.data_ptr(), act_d.data_ptr(), elapsed.t.data_ptr(),
                 reward.t.data_ptr(), done.t.data_ptr(), tlim.t.data_ptr(), N, ATARI_MAX, stream())
            return [obs.check("obs").view(torch.int32), latent.check("latent"), elapsed.check("elapsed"),
                    reward.check("reward"), as_bytes(done.check("done")), as_bytes(tlim.check("time_limit"))]

        obs, latent, elapsed, reward, done, tlim = twice(run)
        assert torch.equal(act_d.cpu(), torch.from_numpy(act))
        lat, r, miss = oa.step_latent(lat0, act)
        want_obs = np.concatenate([obs0[:, 1:], oa.render(lat)[:, None]], axis=1)
        np.testing.assert_array_equal(obs.view(torch.uint8).cpu().numpy().reshape(N, 4, 84, 84), want_obs)
        np.testing.assert_array_equal(latent.cpu().numpy().reshape(N, 5), lat_array(lat))
        el = el0 + 1
        np.testing.assert_array_equal(elapsed.cpu().numpy(), el)
        np.testing.assert_array_equal(reward.cpu().numpy(), r.astype(np.float32))
        dn = miss | (el >= ATARI_MAX)
        np.testing.assert_array_equal(done.cpu().numpy(), dn.astype(np.int32))
        np.testing.assert_array_equal(tlim.cpu().numpy(), (dn & (el == ATARI_MAX)).astype(np.int32))
        if N >= 255:
            assert (r == 1).any() and miss.any() and (el == ATARI_MAX).any()


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 255, 4099])
@pytest.mark.parametrize("use_mask,use_zero,bias,bump", [(False, False, 0, 1), (True, False, 0, 1),
                                                         (False, True, 1, 0), (True, True, 1, 0)])
def test_synth_atari_reset_bit_exact(N, use_mask, use_zero, bias, bump):
    """Reset of the envs selected by `mask` (uint8, nonzero: reset) and `zero_is_mask` (int32, zero: reset) against
    oracle reset_latent / render with episode index episode - episode_bias (modulo 2^32), then episode += bump.
    (1, 0) is the collector's combination: its finalize kernel has already advanced the episode.  Envs not selected
    keep obs, latent, elapsed and episode."""
    rs = np.random.RandomState(N + 2 * bias)
    lat0 = random_latent(N, rs)
    obs0 = rs.randint(0, 256, (N, 4, 84, 84)).astype(np.uint8)
    el0 = rs.randint(0, 1000, N).astype(np.int32)
    seeds = rs.randint(0, 2 ** 32, N, dtype=np.uint64).astype(np.uint32)
    episodes = rs.randint(0, 2 ** 32, N, dtype=np.uint64).astype(np.uint32)
    episodes[0] = 0
    mask = (rs.rand(N) < 0.5).astype(np.uint8) * rs.randint(1, 256, N).astype(np.uint8)
    mask[0] = 1
    zero = np.where(rs.rand(N) < 0.5, 0, rs.choice([1, -3, 7], N)).astype(np.int32)
    zero[0] = 0
    sel = np.ones(N, dtype=bool)
    if use_mask:
        sel &= mask != 0
    if use_zero:
        sel &= zero == 0
    seeds_d, mask_d, zero_d = u32_dev(seeds), torch.from_numpy(mask).cuda(), torch.from_numpy(zero).cuda()

    def run():
        obs, latent, elapsed = atari_buffers(obs0, lat0, el0)
        episode = GuardedBytes(4 * N, dtype=torch.int32)
        episode.t.copy_(u32_dev(episodes))
        call("trl_synth_atari_reset", obs.t.data_ptr(), latent.t.data_ptr(), elapsed.t.data_ptr(), episode.t.data_ptr(),
             seeds_d.data_ptr(), mask_d.data_ptr() if use_mask else None, zero_d.data_ptr() if use_zero else None,
             bias, bump, N, stream())
        return [obs.check("obs").view(torch.int32), latent.check("latent"), elapsed.check("elapsed"),
                episode.check("episode")]

    obs, latent, elapsed, episode = twice(run)
    ep = (episodes.astype(np.int64) - bias) & M32
    fresh = oa.reset_latent(seeds[sel].astype(np.uint64), ep[sel].astype(np.uint64))
    want_lat = lat_array(lat0)
    want_lat[sel] = lat_array(fresh)
    want_obs = obs0.copy()
    want_obs[sel] = np.repeat(oa.render(fresh)[:, None], 4, axis=1)
    np.testing.assert_array_equal(obs.view(torch.uint8).cpu().numpy().reshape(N, 4, 84, 84), want_obs)
    np.testing.assert_array_equal(latent.cpu().numpy().reshape(N, 5), want_lat)
    np.testing.assert_array_equal(elapsed.cpu().numpy(), np.where(sel, 0, el0))
    np.testing.assert_array_equal(u32_host(episode), np.where(sel, (episodes.astype(np.int64) + bump) & M32, episodes))
    assert torch.equal(mask_d.cpu(), torch.from_numpy(mask)) and torch.equal(zero_d.cpu(), torch.from_numpy(zero))


def test_synth_atari_rejects_bad_arguments(native_lib):
    buf = (ctypes.c_float * 64)()
    p = _host_ptr(buf)
    p16 = p + (-p % 16)
    step, reset = native_lib.trl_synth_atari_step, native_lib.trl_synth_atari_reset
    _rejects(native_lib, step(p16, p16, p16, p16, p16, p16, p16, -1, 10, None), "bad size")
    _rejects(native_lib, step(p16, p16, None, p16, p16, p16, p16, 4, 10, None), "null pointer")
    _rejects(native_lib, step(p16 + 4, p16, p16, p16, p16, p16, p16, 4, 10, None), "16-byte aligned")
    assert step(None, None, None, None, None, None, None, 0, 10, None) == 0
    _rejects(native_lib, reset(p16, p16, p16, p16, p16, None, None, 0, 1, -1, None), "bad size")
    _rejects(native_lib, reset(p16, p16, p16, None, p16, None, None, 0, 1, 4, None), "null pointer")
