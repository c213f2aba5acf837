"""The kernels that move and build the training data, called straight through the C ABI and compared with exact NumPy /
torch restatements: the row gather and ring writes (csrc/gather.cu), prioritised sampling, priority update and insert
(csrc/prioritized.cu), the frame-de-duplicated pixel ring (csrc/frames.cu), the collector step's row store and partial
reset, the step counter advance and the tanh-Gaussian action sample (csrc/collect.cu) and the pixel widening
(csrc/atari_env.cu).

Conventions (those of test_layer_kernels.py and test_loss_kernels.py):
  * every output is a view inside a guard region that must be unchanged after the call: NaN for float outputs, the byte
    0xA5 for byte and integer outputs (NaN cannot be stored there);
  * every device counter or ticket has a stated value after each call;
  * every case runs twice and both runs must give identical bits;
  * byte and index results must match the reference exactly; a float result is exact where the arithmetic is exact
    (a byte times a float32 scale is one rounding on both sides), else within a bound derived next to the check.
The tests without the `gpu` mark check argument validation; nothing is launched there.
"""
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import ref_numpy as rn
from tests.test_layer_kernels import U, Guarded, _host_ptr, _rejects, call, same_bits, stream

GUARD = 64
SENTINEL = 0xA5
E53 = 2.0 ** -53
vp = ctypes.c_void_p


# ------------------------------------------------------------------------------------------------------------- helpers
class GuardedBytes:
    """nbytes of output inside GUARD bytes of 0xA5 on each side, starting `offset` bytes past a 16-byte boundary;
    `t` views them as `dtype` (offset must then be a multiple of its size)."""

    def __init__(self, nbytes, offset=0, dtype=torch.uint8):
        self.nbytes, self.lo = int(nbytes), GUARD + offset
        self.buf = torch.full((self.lo + self.nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.bytes = self.buf[self.lo:self.lo + self.nbytes]
        self.t = self.bytes.view(dtype)

    def check(self, what="output"):
        assert (self.buf[:self.lo] == SENTINEL).all() and (self.buf[self.lo + self.nbytes:] == SENTINEL).all(), \
            "%s: a write landed outside the output" % what
        return self.t


def guarded_ints(n, dtype, fill=None):
    g = GuardedBytes(n * torch.tensor([], dtype=dtype).element_size(), dtype=dtype)
    if fill is not None:
        g.t.fill_(fill)
    return g


def dev_bytes(nbytes, offset=0, gen=None):
    """random bytes starting `offset` bytes past a 16-byte boundary"""
    buf = torch.randint(0, 256, (nbytes + offset + 16,), dtype=torch.uint8, device="cuda", generator=gen)
    return buf[offset:offset + nbytes]


def twice(run):
    """run() -> list of output tensors; a second run must reproduce every byte (test_layer_kernels.twice compares
    32-bit words, which byte outputs of odd length do not have)"""
    first = [t.clone() for t in run()]
    second = run()
    for i, (a, b) in enumerate(zip(first, second)):
        assert a.shape == b.shape and torch.equal(a.contiguous().reshape(-1).view(torch.uint8),
                                                  b.contiguous().reshape(-1).view(torch.uint8)), \
            "output %d differs between two identical calls" % i
    return first


def i32(*v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def keys_table(tensors):
    return (vp * len(tensors))(*[t.data_ptr() for t in tensors])


def i64_table(vals):
    return (ctypes.c_int64 * len(vals))(*vals)


# ============================================================================================== A. row copy (gather.cu)
ROW_BYTES = [1, 3, 4, 12, 15, 16, 17, 16384, 16385, (1 << 24) + 8]
OFFSETS = [0, 1, 4, 8]


def gather_case(rbs, idx, src_rows, offset=0, pos=None, rows=None):
    """trl_row_gather of len(rbs) keys, each checked against dst[k] = src[idx[k]] byte for byte"""
    rows = idx.shape[-1] if rows is None else rows
    srcs = [dev_bytes(src_rows * rb, offset) for rb in rbs]
    sel = idx if pos is None else idx[int(pos.item())]

    def run():
        dsts = [GuardedBytes(rows * rb, offset) for rb in rbs]
        call("trl_row_gather", len(rbs), keys_table(srcs), keys_table([d.bytes for d in dsts]), i64_table(rbs),
             idx.data_ptr(), None if pos is None else pos.data_ptr(), rows, stream())
        return [d.check("key %d" % i) for i, d in enumerate(dsts)]

    outs = twice(run)
    for i, (s, o, rb) in enumerate(zip(srcs, outs, rbs)):
        want = s.view(src_rows, rb)[sel].reshape(-1) if rows else s[:0]
        assert torch.equal(o, want), "key %d (row_bytes %d, offset %d): %d bytes differ" % (
            i, rb, offset, int((o != want).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("offset", OFFSETS)
@pytest.mark.parametrize("rb", ROW_BYTES)
def test_row_gather_row_sizes_and_alignments(rb, offset):
    """one key: every copy width (16 B, 4 B, byte) and the chunk split of long rows (16384 B per CTA, capped at ~8
    waves: 2^24 + 8 bytes over 3 rows hits the cap), with duplicate indices and the last source row"""
    src_rows = 5
    idx = torch.tensor([src_rows - 1, 0, src_rows - 1, 2], dtype=torch.int64, device="cuda")
    gather_case([rb], idx, src_rows, offset)


@pytest.mark.gpu
@pytest.mark.parametrize("nkeys", [1, 3, 8])
def test_row_gather_many_keys_in_one_launch(nkeys):
    rbs = [17, 16, 1, 16385, 4, 12, 15, 3][:nkeys]
    torch.manual_seed(nkeys)
    idx = torch.randint(0, 40, (37,), dtype=torch.int64, device="cuda")
    idx[-1] = 39
    gather_case(rbs, idx, 40)
    gather_case(rbs, idx, 40, offset=4)


@pytest.mark.gpu
def test_row_gather_position_table():
    """idx[(*pos_ptr) * rows + k]: only row `pos` of the table is used"""
    torch.manual_seed(1)
    table = torch.randint(0, 50, (3, 21), dtype=torch.int64, device="cuda")
    for p in (0, 2):
        gather_case([12, 17], table, 50, pos=i32(p))


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [0, 1, 65535, 65536, 70001])
def test_row_gather_row_counts(rows):
    """grid y is limited to 65535: batches beyond it are strided inside the kernel"""
    torch.manual_seed(rows)
    idx = torch.randint(0, 1000, (max(rows, 1),), dtype=torch.int64, device="cuda")
    gather_case([4, 12, 1], idx[:rows] if rows else idx, 1000, rows=rows)


@pytest.mark.gpu
def test_ring_write_at_device_row():
    """dst[*row_ptr] = src for every key; no other row changes"""
    T, rbs = 7, [12, 16385, 3]
    srcs = [dev_bytes(rb) for rb in rbs]
    for row in (0, 3, T - 1):
        rp = i32(row)

        def run():
            dsts = [GuardedBytes(T * rb) for rb in rbs]
            for d in dsts:
                d.bytes.fill_(7)
            call("trl_ring_write", len(rbs), keys_table(srcs), keys_table([d.bytes for d in dsts]), i64_table(rbs),
                 rp.data_ptr(), stream())
            return [d.check() for d in dsts]

        for s, o, rb in zip(srcs, twice(run), rbs):
            want = torch.full((T, rb), 7, dtype=torch.uint8, device="cuda")
            want[row] = s
            assert torch.equal(o.view(T, rb), want)
        assert int(rp.item()) == row


def _ring_advance_run(T, rbs, steps, with_size, graph):
    """`steps` calls of trl_ring_write_advance, each with new source bytes; checks row, size and ticket after every
    call against the model row = (row + 1) % T, size = min(size + 1, T).  Returns the ring contents."""
    gen = torch.Generator(device="cuda")
    gen.manual_seed(T * 1000 + steps)
    srcs = [torch.zeros(rb + 16, dtype=torch.uint8, device="cuda")[:rb] for rb in rbs]
    dsts = [GuardedBytes(T * rb) for rb in rbs]
    for d in dsts:
        d.bytes.zero_()
    row, size, tk = i32(0), i32(0), i32(0)
    model = [torch.zeros(T, rb, dtype=torch.uint8, device="cuda") for rb in rbs]

    def launch():
        call("trl_ring_write_advance", len(rbs), keys_table(srcs), keys_table([d.bytes for d in dsts]), i64_table(rbs),
             row.data_ptr(), T, size.data_ptr() if with_size else None, tk.data_ptr(), stream())

    g = None
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            launch()
    r, s = 0, 0
    for _ in range(steps):
        for src, m in zip(srcs, model):
            src.copy_(torch.randint(0, 256, src.shape, dtype=torch.uint8, device="cuda", generator=gen))
            m[r] = src
        if g is not None:
            g.replay()
        else:
            launch()
        r, s = (r + 1) % T, min(s + 1, T)
        assert int(row.item()) == r, "row index %d, want %d" % (int(row.item()), r)
        assert int(size.item()) == (s if with_size else 0)
        assert int(tk.item()) == 0, "ticket not back at zero"
    for d, m in zip(dsts, model):
        assert torch.equal(d.check().view(m.shape), m), "ring contents differ from the model"
    return [d.bytes.clone() for d in dsts]


@pytest.mark.gpu
@pytest.mark.parametrize("with_size", [True, False])
@pytest.mark.parametrize("T", [1, 2, 7])
def test_ring_write_advance_laps_and_graph(T, with_size):
    """several laps; a 4 MB key copied by hundreds of CTAs still lands at the OLD row in every key (the last CTA
    advances the row only after all have read it); eager calls and one graph replayed T+3 times agree bit for bit"""
    rbs = [12, 4 << 20, 17]
    eager = _ring_advance_run(T, rbs, T + 3, with_size, graph=False)
    graphed = _ring_advance_run(T, rbs, T + 3, with_size, graph=True)
    for a, b in zip(eager, graphed):
        assert torch.equal(a, b)
    _ring_advance_run(T, [16, 3], 3 * T + 2, with_size, graph=False)


# ========================================================================== B. prioritised replay (prioritized.cu)
PER_SIZES = [1, 2, 31, 1023, 1024, 1025, 2047, 4095, 4096]
PER_B = [1, 7, 1024, 1025, 5000]
U_TOP = 1.0 - 2.0 ** -53        # np.random.rand can return it; (b - 1 + U_TOP) rounds to b
BETA = 0.375                    # exact in fp32: the kernel and the oracle raise to the same power


def per_run(prio, size, u, beta):
    ud = torch.as_tensor(u, dtype=torch.float64, device="cuda")
    b = ud.numel()

    def run():
        idx, w = guarded_ints(b, torch.int64), Guarded(b)
        call("trl_per_sample", prio.data_ptr(), size, ud.data_ptr(), b, beta, idx.t.data_ptr(), w.t.data_ptr(), stream())
        return [idx.check("idx"), w.check("weights")]

    return twice(run)


def uniforms(rs, b):
    u = rs.rand(b)
    u[0] = 0.0
    u[-1] = U_TOP
    if b > 2:
        u[b // 2] = U_TOP
    return u


@pytest.mark.gpu
@pytest.mark.parametrize("b", PER_B)
@pytest.mark.parametrize("size", PER_SIZES)
def test_per_sample_exact_regime_matches_oracle_bit_for_bit(size, b):
    """priorities j * 2^-10, j in 1..1024: every fp64 partial sum is exact in any order, so the kernel's scan equals
    np.cumsum and the indices equal the oracle's bit for bit.  The weights are (size p/total)^-beta / max_w in fp64
    (pow within a few ulp, 2^-40 relative covers it) rounded once to fp32 (U)."""
    rs = np.random.RandomState(size * 7 + b)
    p = (rs.randint(1, 1025, size) * 2.0 ** -10).astype(np.float32)
    prio = torch.from_numpy(p).cuda()
    u = uniforms(rs, b)
    idx, w = per_run(prio, size, u, BETA)
    ridx, rw = rn.per_sample(p, size, u, BETA)
    assert np.array_equal(idx.cpu().numpy(), ridx), "indices differ from the oracle"
    assert np.all(np.abs(w.cpu().numpy().astype(np.float64) - rw) <= (U + 2.0 ** -40) * rw)


@pytest.mark.gpu
@pytest.mark.parametrize("b", [2, 7, 1025])
def test_per_sample_never_draws_a_zero_priority_row(b):
    """trailing zero priorities: the last stratum's target (b - 1 + u)/b * total rounds to the total for u = 1 - 2^-53,
    which no prefix exceeds; the draw must be the last row with a positive priority, with a finite weight"""
    size = 100
    p = np.full(size, 0.5, dtype=np.float32)
    p[-3:] = 0.0
    p[10:13] = 0.0
    u = np.full(b, 0.5)
    u[-1] = U_TOP
    idx, w = per_run(torch.from_numpy(p).cuda(), size, u, BETA)
    ridx, rw = rn.per_sample(p, size, u, BETA)
    idx, w = idx.cpu().numpy(), w.cpu().numpy()
    assert idx[-1] == size - 4 and ridx[-1] == size - 4, "last draw %d (oracle %d), want row %d" % (
        idx[-1], ridx[-1], size - 4)
    assert np.all(p[idx] > 0) and np.all(np.isfinite(w)) and np.all(w > 0)
    assert np.array_equal(idx, ridx)
    assert np.all(np.abs(w - rw) <= (U + 2.0 ** -40) * rw)


def wide_priorities(rs, size):
    """1e-30 .. 1e30, runs of equal priorities, zero rows inside and at the end"""
    p = (10.0 ** rs.uniform(-30, 30, size)).astype(np.float32)
    for _ in range(max(1, size // 64)):
        a = rs.randint(0, size)
        p[a:a + rs.randint(1, 9)] = p[a]
        z = rs.randint(0, size)
        p[z:z + rs.randint(1, 4)] = 0.0
    if size > 1:
        p[-min(3, size - 1):] = 0.0
    if not (p > 0).any():
        p[0] = 1.0
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("b", [7, 1025, 5000])
@pytest.mark.parametrize("size", [2, 31, 1025, 4096])
def test_per_sample_wide_range_lands_in_the_exact_stratum(size, b):
    """The scan's fp64 prefix is not np.cumsum's when the sums round.  With S_i the EXACT inclusive prefix (fractions)
    and t the target computed from the exact total, the drawn row i must satisfy S_{i-1} - tol <= t <= S_i + tol, tol =
    (per-thread run (<= 4) + 15 scan levels + 4 for the target) * 2^-53 * S_total: a row other than the oracle's only
    when t is within that rounding of a row boundary.  A zero-priority row is never drawn; the weights follow
    (p_i / min positive p)^-beta within U + the fp64 rounding of the ratio and the two pows."""
    rs = np.random.RandomState(size + 31 * b)
    p = wide_priorities(rs, size)
    u = uniforms(rs, b)
    idx, w = per_run(torch.from_numpy(p).cuda(), size, u, BETA)
    idx, w = idx.cpu().numpy(), w.cpu().numpy().astype(np.float64)
    assert np.all(p[idx] > 0), "a zero-priority row was drawn"
    S = np.empty(size + 1, dtype=object)
    S[0] = Fraction(0)
    acc = Fraction(0)
    for i, v in enumerate(p):
        acc += Fraction(float(v))
        S[i + 1] = acc
    total = float(acc)
    tol = Fraction((4 + 15 + 4) * E53 * total)
    for k in range(b):
        t = Fraction((k + float(u[k])) / b * total)
        i = int(idx[k])
        assert S[i] - tol <= t <= S[i + 1] + tol, "draw %d: row %d's interval misses the target" % (k, i)
    pmin = float(p[p > 0].min())
    rw = (p[idx].astype(np.float64) / pmin) ** -BETA
    assert np.all(np.abs(w - rw) <= (U + 2.0 ** -40) * rw + 2.0 ** -149)
    ridx, _ = rn.per_sample(p, size, u, BETA)
    assert np.all(p[ridx] > 0), "the oracle drew a zero-priority row"


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 10000])
def test_per_update_matches_fp64(n):
    """prio[idx_k] = (mean |td_k| + eps)^alpha: the fp64 mean (tree sum, <= 14 levels: 14 * 2^-53 relative), its fp32
    rounding (U), the fp32 + eps (U) and powf (alpha * 2U from the input, 4 ulp = 8U of its own).  Rows not drawn
    keep their bits; max_prio becomes max(old, new priorities) exactly and never decreases."""
    torch.manual_seed(n)
    R, b, alpha, eps = 300, 37, 0.625, 1e-6          # alpha exact in fp32
    idx = torch.randperm(R, device="cuda")[:b].to(torch.int64)
    td = torch.randn(b, n, device="cuda") * 3
    base = torch.rand(R, device="cuda") + 0.1
    for m0 in (0.5, 1e6):
        mp0 = torch.tensor([m0], dtype=torch.float32, device="cuda")

        def run():
            prio, mp = Guarded(R), Guarded(1)
            prio.t.copy_(base)
            mp.t.copy_(mp0)
            call("trl_per_update", prio.t.data_ptr(), idx.data_ptr(), td.data_ptr(), b, n, alpha, eps, mp.t.data_ptr(),
                 stream())
            return [prio.check("prio"), mp.check("max_prio")]

        prio, mp = twice(run)
        r = (td.double().abs().mean(1) + float(np.float32(eps))) ** alpha
        got = prio[idx].double()
        assert torch.all((got - r).abs() <= (14 * E53 + (2 + alpha * 2 + 8) * U) * r), "priorities beyond the bound"
        keep = torch.ones(R, dtype=torch.bool, device="cuda")
        keep[idx] = False
        assert same_bits(prio[keep], base[keep]), "a row that was not drawn changed"
        assert float(mp.item()) == max(m0, float(prio[idx].max())) >= m0


@pytest.mark.gpu
def test_per_update_duplicate_rows_take_one_candidate():
    """duplicate rows in a batch are written unordered: the row ends up with one of its candidates' values (each
    candidate computed by a duplicate-free call), and max_prio is the maximum of all candidates"""
    torch.manual_seed(5)
    b, n = 64, 9
    td = torch.rand(b, n, device="cuda") * 4
    idx = torch.randint(0, 8, (b,), device="cuda").to(torch.int64)
    distinct = torch.arange(b, dtype=torch.int64, device="cuda")

    def update(rows, R):
        def run():
            prio, mp = Guarded(R), Guarded(1)
            prio.t.zero_()
            mp.t.zero_()
            call("trl_per_update", prio.t.data_ptr(), rows.data_ptr(), td.data_ptr(), b, n, 0.6, 1e-6, mp.t.data_ptr(),
                 stream())
            return [prio.check("prio"), mp.check("max_prio")]
        return run

    cand, m1 = twice(update(distinct, b))
    # the duplicate call is not repeated for bits: which duplicate lands last is unordered by contract
    prio, mp = update(idx, 8)()
    for row in range(8):
        c = cand[idx == row]
        if c.numel():
            assert (c == prio[row]).any(), "row %d holds none of its candidates" % row
        else:
            assert prio[row].item() == 0
    assert same_bits(mp, cand.max().reshape(1)) and same_bits(m1, mp)


@pytest.mark.gpu
def test_per_insert_writes_only_the_device_row():
    T = 33
    base = torch.rand(T, device="cuda")
    mp = torch.tensor([2.5], device="cuda")
    for row in (0, T - 1):
        rp = i32(row)

        def run():
            prio = Guarded(T)
            prio.t.copy_(base)
            call("trl_per_insert", prio.t.data_ptr(), rp.data_ptr(), mp.data_ptr(), stream())
            return [prio.check()]

        (got,) = twice(run)
        want = base.clone()
        want[row] = 2.5
        assert same_bits(got, want) and int(rp.item()) == row and mp.item() == 2.5


# ================================================================================== C. frame ring (frames.cu)
class FrameModel:
    """N envs producing C-frame stacks with FrameStack semantics (a reset repeats the first frame C times; each env
    resets independently at random), started mid-episode; records the full (T, N, C, F) obs / next_obs ring the
    de-duplicated one must rebuild, and the newest-frame sequence the history is checked against."""

    def __init__(self, N, C, F, T, seed, p_done=0.15, resets=True):
        self.N, self.C, self.F, self.T = N, C, F, T
        self.g = torch.Generator(device="cuda")
        self.g.manual_seed(seed)
        self.p_done = p_done if resets else 0.0
        self.elapsed = torch.randint(0, 2 * C, (N,), dtype=torch.int32, device="cuda", generator=self.g)
        if not resets:
            self.elapsed.fill_(C - 1 + 5)
        st = self.frames(C)
        for n in range(N):                     # the first C-1-elapsed frames repeat the episode's first frame
            first = max(0, C - 1 - int(self.elapsed[n]))
            st[n, :first] = st[n, first]
        self.stack = st.contiguous()
        self.obs = torch.zeros(T, N, C, F, dtype=torch.uint8, device="cuda")
        self.next = torch.zeros_like(self.obs)
        self.newest = [self.stack[:, j].clone() for j in range(C - 1)]     # seeded: the frames older than row 0
        self.top = self.size = self.writes = 0
        self.reset_rows = set()

    def frames(self, k):
        return torch.randint(0, 256, (self.N, k, self.F), dtype=torch.uint8, device="cuda", generator=self.g)

    def step(self):
        """-> (obs stack, elapsed, next_obs stack) of this step; advances the model"""
        obs, el = self.stack.clone(), self.elapsed.clone()
        nxt = torch.cat([self.stack[:, 1:], self.frames(1)], 1).contiguous()
        self.obs[self.top], self.next[self.top] = obs, nxt
        self.newest.append(obs[:, -1].clone())
        if (el == 0).any():
            self.reset_rows.add(self.top)
        done = torch.rand(self.N, device="cuda", generator=self.g) < self.p_done
        first = self.frames(1)
        self.stack = torch.where(done[:, None, None], first.expand(-1, self.C, -1), nxt).contiguous()
        self.elapsed = torch.where(done, torch.zeros_like(el), el + 1)
        self.top, self.size, self.writes = (self.top + 1) % self.T, min(self.size + 1, self.T), self.writes + 1
        return obs, el, nxt

    def pushes(self):
        return max(0, self.writes - self.T)

    def hist_want(self, m):
        """the frame m steps older than the oldest ring row"""
        return self.newest[self.C - 1 + self.pushes() - m]


class FrameRing:
    """the device ring driven through the C ABI the way MemoryEfficientReplayBuffer drives it"""

    def __init__(self, N, C, F, T):
        self.N, self.C, self.F, self.T = N, C, F, T
        z = lambda *s: torch.zeros(*s, dtype=torch.uint8, device="cuda")
        self.obs, self.next, self.age, self.hist = z(T, N, F), z(T, N, F), z(T, N), z(C - 1, N, F)
        self.hc, self.top, self.size = i32(0), i32(0), i32(0)

    def step(self, obs, elapsed, nxt):
        N, C, F, T = self.N, self.C, self.F, self.T
        call("trl_frame_ring_write", obs.data_ptr(), self.obs.data_ptr(), self.age.data_ptr(), elapsed.data_ptr(),
             self.hist.data_ptr(), self.hc.data_ptr(), self.top.data_ptr(), self.size.data_ptr(), N, C, F, T, C - 1,
             stream())
        call("trl_frame_hist_advance", self.hc.data_ptr(), self.size.data_ptr(), T, stream())
        call("trl_frame_ring_write", nxt.data_ptr(), self.next.data_ptr(), None, None, None, None, self.top.data_ptr(),
             None, N, C, F, T, C - 1, stream())
        call("trl_step_advance", self.top.data_ptr(), T, self.size.data_ptr(), None, stream())

    def gather(self, idx, scale, rows=None, pos=None):
        rows = idx.shape[-1] if rows is None else rows
        n = rows * self.N * self.C * self.F

        def run():
            o1, o2 = Guarded(n), Guarded(n)
            call("trl_frame_stack_gather", self.obs.data_ptr(), self.next.data_ptr(), self.age.data_ptr(),
                 self.hist.data_ptr(), self.hc.data_ptr(), idx.data_ptr(), None if pos is None else pos.data_ptr(),
                 rows, self.top.data_ptr(), self.size.data_ptr(), self.N, self.C, self.F, self.T, scale,
                 o1.t.data_ptr(), o2.t.data_ptr(), stream())
            return [o1.check("obs"), o2.check("next_obs")]

        return [o.view(rows, self.N, self.C, self.F) for o in twice(run)]


def check_counters_and_history(ring, model):
    assert int(ring.top.item()) == model.top and int(ring.size.item()) == model.size
    assert int(ring.hc.item()) == model.pushes(), "hist_count %d, want %d" % (int(ring.hc.item()), model.pushes())
    hc = model.pushes()
    for m in range(1, model.C):
        slot = (hc - m) % (model.C - 1)
        assert torch.equal(ring.hist[slot], model.hist_want(m)), "history slot %d (frame %d back) differs" % (slot, m)


def sample_rows(model, rs):
    """every valid row when the output is small, else a subset that keeps the oldest row, the newest row and the rows
    right after a reset"""
    valid = list(range(model.size))
    cap = max(3, (1 << 22) // (model.N * model.C * model.F))
    if len(valid) > cap:
        must = {model.top % model.T if model.size == model.T else 0, (model.top - 1) % model.T}
        must |= set(sorted(model.reset_rows & set(valid))[:2])
        rest = [r for r in valid if r not in must]
        valid = sorted(must) + list(rs.choice(rest, cap - len(must), replace=False))
    valid.append(valid[0])                   # a duplicate
    return torch.tensor(valid, dtype=torch.int64, device="cuda")


def check_gather(ring, model, scale, rs):
    idx = sample_rows(model, rs)
    o1, o2 = ring.gather(idx, scale)
    s = torch.tensor(scale, dtype=torch.float32, device="cuda")
    assert torch.equal(o1, model.obs[idx].float() * s), "obs stacks differ from the full-stack model"
    assert torch.equal(o2, model.next[idx].float() * s), "next_obs stacks differ from the full-stack model"
    # device-position form: row 1 of a two-row table
    table = torch.stack([idx.flip(0), idx])
    p1, p2 = ring.gather(table, scale, rows=idx.numel(), pos=i32(1))
    assert torch.equal(p1, o1) and torch.equal(p2, o2)


FRAME_CASES = [(C, T, F, N) for i, (C, T) in enumerate((C, T) for C in (2, 3, 4, 8) for T in sorted({1, 2, 3, C - 1, 64}))
               for F, N in [[(16, 3), (48, 33), (7056, 1), (48, 1), (16, 33)][i % 5]]]


@pytest.mark.gpu
@pytest.mark.parametrize("C,T,F,N", FRAME_CASES)
def test_frame_ring_rebuilds_every_stack(C, T, F, N):
    """after 0, 1/4, 1, 1.5 and 4 laps every sampled row (the oldest one, rows right after a reset, the newest) gathers
    bit for bit to scale * the full-stack model, for obs and next_obs; the history and hist_count equal the model's
    frames older than the oldest row after every step"""
    model, ring = FrameModel(N, C, F, T, seed=C * 1000 + T * 10 + N), FrameRing(N, C, F, T)
    rs = np.random.RandomState(C + T + F + N)
    checkpoints = sorted({max(1, T // 4), T, T + (T + 1) // 2, 4 * T})
    ring.gather(torch.zeros(1, dtype=torch.int64, device="cuda"), 1.0, rows=0)      # empty ring: rows = 0
    for step in range(1, 4 * T + 1):
        ring.step(*model.step())
        check_counters_and_history(ring, model)
        if step in checkpoints:
            for scale in (1.0 / 255.0, 1.0):
                check_gather(ring, model, scale, rs)
    assert ring.age.max() <= C - 1


@pytest.mark.gpu
def test_frame_stack_gather_past_the_grid_y_limit():
    """rows * N = 65536 samples (grid y is limited to 65535; the kernel strides over the rest)"""
    C, T, F, N = 2, 8, 16, 1
    model, ring = FrameModel(N, C, F, T, seed=9), FrameRing(N, C, F, T)
    for _ in range(T + 3):
        ring.step(*model.step())
    idx = torch.randint(0, T, (65536,), dtype=torch.int64, device="cuda")
    o1, o2 = ring.gather(idx, 1.0 / 255.0)
    s = torch.tensor(1.0 / 255.0, dtype=torch.float32, device="cuda")
    assert torch.equal(o1, model.obs[idx].float() * s) and torch.equal(o2, model.next[idx].float() * s)


@pytest.mark.gpu
@pytest.mark.parametrize("truthful", [False, True])
@pytest.mark.parametrize("C,T,N", [(4, 10, 3), (4, 2, 1), (3, 64, 2)])
def test_memory_efficient_add_sample_keeps_the_first_rows_older_frames(C, T, N, truthful):
    """MemoryEfficientReplayBuffer.add_sample with full stacks.  The default episode_steps (C-1, mid-episode) is right
    for a run without resets; truthful episode_steps with resets.  The first row is mid-episode, so rows 0 .. C-2 need
    frames older than the ring -- they come from the first stack, not from an empty history."""
    from torchrl_b200.replay_buffers.memory_efficient import MemoryEfficientReplayBuffer
    F = 48
    model = FrameModel(N, C, F, T, seed=77 + T, resets=truthful)
    buf = MemoryEfficientReplayBuffer(T * N, env_nums=N, device="cuda", obs_scale=1.0 / 255.0)
    for step in range(1, 2 * T + 3):
        obs, el, nxt = model.step()
        buf.add_sample({"obs": obs.view(N, C, 4, F // 4), "next_obs": nxt.view(N, C, 4, F // 4)},
                       episode_steps=el if truthful else None)
        if step in (1, C - 1, T, 2 * T + 2):
            idx = torch.arange(model.size, dtype=torch.int64, device="cuda")
            out = buf.gather_rows(idx, ["obs", "next_obs"])
            s = torch.tensor(1.0 / 255.0, dtype=torch.float32, device="cuda")
            want = model.obs[idx].float() * s
            got = out["obs"].view(want.shape)
            bad = [int(r) for r in idx if not torch.equal(got[r], want[r])]
            assert not bad, "step %d: rows %s gather the wrong frames" % (step, bad)
            assert torch.equal(out["next_obs"].view(want.shape), model.next[idx].float() * s)


# ================================================================================== D. collector step (collect.cu)
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 7])
def test_step_advance_every_pointer_combination(T):
    """row = (row + 1) % T, size = min(size + 1, T), counter + 1, each only when given; the counters sit in 0xA5
    guards, and two runs of the same sequence give the same bytes"""
    for mask in range(8):
        def run():
            t = guarded_ints(1, torch.int32, T - 1) if mask & 1 else None
            s = guarded_ints(1, torch.int32, T - 1) if mask & 2 else None
            c = guarded_ints(1, torch.int64, 41) if mask & 4 else None
            for k in range(1, T + 2):
                call("trl_step_advance", None if t is None else t.t.data_ptr(), T,
                     None if s is None else s.t.data_ptr(), None if c is None else c.t.data_ptr(), stream())
                if t is not None:
                    assert int(t.check("row").item()) == (T - 1 + k) % T
                if s is not None:
                    assert int(s.check("size").item()) == T, "size must saturate at T"
                if c is not None:
                    assert int(c.check("counter").item()) == 41 + k
            return [g.t for g in (t, s, c) if g is not None]

        twice(run)


class Dev:
    """a device copy of a NumPy array inside GUARD bytes of 0xA5 on each side; `expect` compares the whole buffer,
    guards included, with the array it should now hold"""

    def __init__(self, arr):
        self.arr = np.ascontiguousarray(arr)
        raw = self.arr.reshape(-1).view(np.uint8)
        host = np.full(2 * GUARD + raw.size, SENTINEL, dtype=np.uint8)
        host[GUARD:GUARD + raw.size] = raw
        self.buf = torch.from_numpy(host).cuda()
        self.ptr = self.buf.data_ptr() + GUARD

    def expect(self, want, what):
        got = self.buf.cpu().numpy()
        assert (got[:GUARD] == SENTINEL).all() and (got[-GUARD:] == SENTINEL).all(), \
            "%s: a write landed outside the output" % what
        g = got[GUARD:-GUARD].view(self.arr.dtype).reshape(self.arr.shape)
        w = np.ascontiguousarray(want, dtype=self.arr.dtype).reshape(self.arr.shape)
        bad = (g.reshape(-1).view(np.uint8).reshape(g.size, -1) != w.reshape(-1).view(np.uint8).reshape(g.size, -1)).any(1)
        if bad.any():
            first = np.unravel_index(int(np.flatnonzero(bad)[0]), g.shape)
            raise AssertionError("%s: %d of %d entries differ (first at %s: got %r, want %r)" % (
                what, int(bad.sum()), g.size, tuple(int(i) for i in first), g[first], w[first]))


def mix32b(x):
    x = x ^ (x >> np.uint64(16))
    x = (x * np.uint64(0x85EBCA6B)) & np.uint64(0xFFFFFFFF)
    x = x ^ (x >> np.uint64(13))
    x = (x * np.uint64(0xC2B2AE35)) & np.uint64(0xFFFFFFFF)
    return x ^ (x >> np.uint64(16))


def reset_value_b(seed, episode, j, init_scale):
    """collect.cu's reset_value_b: 32-bit integer hashing (wrapping), 24 bits to a float32 in [0, 1), then one fp64
    affine map rounded to float32"""
    s, e, jj = (np.asarray(v).astype(np.uint64) for v in (seed, episode, j))
    with np.errstate(over="ignore"):                           # wraps mod 2^64, then reduced mod 2^32
        key = (s * np.uint64(0x9E3779B1) + e * np.uint64(0x85EBCA77) + jj * np.uint64(0xC2B2AE3D)
               + np.uint64(0x27D4EB2F)) & np.uint64(0xFFFFFFFF)
    u = (mix32b(key) >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return (init_scale * (2.0 * u.astype(np.float64) - 1.0)).astype(np.float32)


FIN_T, FIN_MAXF, FIN_DISCOUNT, FIN_INIT, FIN_CLIP = 4, 50, 0.99, 5.0, 1.5
# (cur_ob_in aliases cur_ob_out, device env, NormObs mode, any_reset, t = T-1 (else 0), v_next, terminal_includes_surpass,
#  ret_log, b_values); the raw-obs cases set any_reset[t & 1] or clear it, on both parities of t
FIN_CASES = [
    (1, 1, "off", [0, 1], 0, 1, 0, 1, 1),
    (0, 1, "off", [1, 0], 1, 0, 1, 0, 0),
    (1, 1, "norm", [1, 1], 0, 1, 1, 1, 0),
    (0, 1, "norm", [0, 0], 1, 1, 0, 1, 1),
    (1, 1, "raw", [1, 0], 0, 1, 0, 1, 1),
    (0, 1, "raw", [1, 0], 1, 0, 1, 1, 0),
    (1, 1, "raw", [0, 1], 1, 1, 1, 0, 1),
    (0, 1, "raw", [0, 1], 0, 1, 0, 1, 1),
    (1, 1, "raw", None, 1, 1, 0, 1, 1),
    (1, 0, "off", None, 0, 1, 1, 1, 1),
    (0, 0, "norm", [1, 1], 1, 0, 0, 0, 0),
]


def finalize_inputs(N, o, a, rs):
    f32 = lambda *s: rs.randn(*s).astype(np.float32)
    c = dict(cur_ob=f32(N, o), next_norm=f32(N, o), state=2 * f32(N, o), act=f32(N, a), value=f32(N), v_next=f32(N),
             reward=f32(N), done=(rs.rand(N) < 0.3).astype(np.uint8), tl=(rs.rand(N) < 0.3).astype(np.uint8),
             elapsed=rs.randint(0, 100, N).astype(np.int32),
             episode=rs.randint(0, 2 ** 32, N, dtype=np.uint64).astype(np.uint32),
             seeds=rs.randint(0, 2 ** 32, N, dtype=np.uint64).astype(np.uint32),
             step_count=rs.randint(0, FIN_MAXF - 1, N).astype(np.int32), ep_return=10 * rs.randn(N),
             epoch_reward=rs.randn(N), n_done=np.array([5], dtype=np.int32),
             norm_mean=rs.randn(o), norm_var=rs.rand(o) + 0.5, garbage=f32(N, o))
    c["step_count"][rs.rand(N) < 0.3] = FIN_MAXF - 1          # surpass this step, with and without done
    c["episode"][0] = 0xFFFFFFFF                               # a reset wraps the episode counter
    return c


def ref_finalize(c, norm, any_reset, t, v_next, tis, ret_log, values, device):
    """collect.cu's FinalizeParams contract, restated: returns every buffer's expected content"""
    N = c["reward"].shape[0]
    e = {}
    sc = c["step_count"] + 1
    dn = c["done"] != 0
    surpass = sc >= FIN_MAXF
    mask = dn | surpass
    r = c["reward"]
    er = c["ep_return"] + r.astype(np.float64)                 # train_rew: the un-bootstrapped reward
    e["epoch_reward"] = c["epoch_reward"] + r.astype(np.float64)
    e["ret_log"] = np.full((FIN_T, N), np.nan, dtype=np.float32)
    if ret_log:
        e["ret_log"][t, dn] = er[dn].astype(np.float32)
    e["n_done"] = c["n_done"] + np.int32(dn.sum())
    e["ep_return"] = np.where(dn, 0.0, er)
    if v_next:                                                 # fp32: discount * V(next), then + r
        r = np.where(surpass, np.float32(FIN_DISCOUNT) * c["v_next"] + r, r)
    nanrows = lambda *s: np.full((FIN_T, N) + s, np.nan, dtype=np.float32)
    e["b_rewards"] = nanrows()
    e["b_rewards"][t] = r
    e["b_terminals"] = np.full((FIN_T, N), SENTINEL, dtype=np.uint8)
    e["b_terminals"][t] = dn | (bool(tis) & surpass)
    e["b_time_limits"] = np.full((FIN_T, N), SENTINEL, dtype=np.uint8)
    e["b_time_limits"][t] = c["tl"]
    e["b_values"] = nanrows()
    if values:
        e["b_values"][t] = c["value"]
    e["step_count"] = np.where(mask, 0, sc).astype(np.int32)
    e["b_obs"], e["b_next_obs"], e["b_acts"] = nanrows(c["cur_ob"].shape[1]), nanrows(c["cur_ob"].shape[1]), \
        nanrows(c["act"].shape[1])
    e["b_obs"][t], e["b_next_obs"][t], e["b_acts"][t] = c["cur_ob"], c["next_norm"], c["act"]
    e["state"], e["elapsed"], e["episode"] = c["state"], c["elapsed"].copy(), c["episode"].copy()
    if not device:                                             # host env: the bridge resets after the launch
        e["cur_ob_out"] = c["next_norm"]
        return e
    e["elapsed"][mask] = 0
    j = np.arange(c["state"].shape[1])
    rv = reset_value_b(c["seeds"][:, None], c["episode"][:, None], j[None, :], FIN_INIT)
    raw = np.where(mask[:, None], rv, c["state"])
    e["state"] = raw
    hit = any_reset is not None and any_reset[t & 1] != 0
    if norm == "off":
        ob = raw
    elif norm == "raw":
        ob = raw if hit else c["next_norm"]
    else:
        y = (raw.astype(np.float64) - c["norm_mean"]) / (np.sqrt(c["norm_var"]) + 1e-4)
        ob = np.where(mask[:, None], np.fmin(np.fmax(y, -FIN_CLIP), FIN_CLIP).astype(np.float32), c["next_norm"])
    e["cur_ob_out"] = ob
    e["episode"][mask] += np.uint32(1)
    return e


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(FIN_CASES)))
@pytest.mark.parametrize("N", [1, 31, 32, 33, 1000])
def test_collect_finalize_matches_its_contract(N, case):
    """trl_collect_finalize against a NumPy restatement of its contract (csrc/collect.cu, FinalizeParams), byte for
    byte in every buffer it reads or writes, guards included: the row-t stores, the un-bootstrapped episode return and
    ret_log only for done envs, n_done, the fp32 bootstrap on surpass only, terminal_includes_surpass, step_count /
    elapsed / episode bookkeeping, and the next observation -- carried over (host env), or reset from reset_value_b
    (device env) then raw, normalised and clipped in fp64, or raw for all envs after any reset.  N straddles the
    32-env CTAs; every input array is checked unchanged."""
    alias, device, norm, any_reset, t_last, v_next, tis, ret_log, values = FIN_CASES[case]
    o, a = 3, 2
    t = FIN_T - 1 if t_last else 0
    c = finalize_inputs(N, o, a, np.random.RandomState(N * 31 + case))
    want = ref_finalize(c, norm, any_reset, t, v_next, tis, ret_log, values, device)
    nan = lambda *s: np.full(s, np.nan, dtype=np.float32)
    flags = lambda: np.full((FIN_T, N), SENTINEL, dtype=np.uint8)

    def run():
        d = {k: Dev(c[k]) for k in ("next_norm", "act", "value", "v_next", "reward", "done", "tl", "step_count",
                                    "ep_return", "epoch_reward", "n_done", "norm_mean", "norm_var")}
        d["cur_out"] = Dev(c["cur_ob"] if alias else c["garbage"])
        d["cur_in"] = d["cur_out"] if alias else Dev(c["cur_ob"])
        for k in ("state", "elapsed", "episode", "seeds"):
            d[k] = Dev(c[k]) if device else None
        d["any_reset"] = None if any_reset is None else Dev(np.array(any_reset, dtype=np.int32))
        d["ret_log"] = Dev(nan(FIN_T, N)) if ret_log else None
        d["b_obs"], d["b_next_obs"], d["b_acts"] = Dev(nan(FIN_T, N, o)), Dev(nan(FIN_T, N, o)), Dev(nan(FIN_T, N, a))
        d["b_values"], d["b_rewards"] = Dev(nan(FIN_T, N)), Dev(nan(FIN_T, N))
        d["b_terminals"], d["b_time_limits"], d["t"] = Dev(flags()), Dev(flags()), Dev(np.array([t], dtype=np.int32))
        P = lambda k: None if d[k] is None else d[k].ptr
        normed = norm != "off"
        call("trl_collect_finalize", P("cur_in"), P("next_norm"), P("state"), P("act"),
             P("value") if values else None, P("v_next") if v_next else None, P("reward"), P("done"), P("tl"),
             P("elapsed"), P("episode"), P("seeds"), P("step_count"), P("ep_return"), P("epoch_reward"), P("ret_log"),
             P("n_done"), P("any_reset"), P("norm_mean") if normed else None, P("norm_var") if normed else None,
             P("cur_out"), P("b_obs"), P("b_next_obs"), P("b_acts"), P("b_values") if values else None,
             P("b_rewards"), P("b_terminals"), P("b_time_limits"), P("t"), N, o, a, FIN_MAXF, FIN_DISCOUNT,
             FIN_INIT, FIN_CLIP, tis, 1 if norm == "raw" else 0, stream())
        torch.cuda.synchronize()
        run.d = d
        return [x.buf for x in d.values() if x is not None]

    twice(run)
    d = run.d
    for k in ("next_norm", "act", "value", "v_next", "reward", "done", "tl", "norm_mean", "norm_var", "t"):
        d[k].expect(d[k].arr, k + " (input)")
    if d["any_reset"] is not None:
        d["any_reset"].expect(np.array(any_reset, dtype=np.int32), "any_reset (input)")
    if not alias:
        d["cur_in"].expect(c["cur_ob"], "cur_ob_in (input)")
    d["cur_out"].expect(want["cur_ob_out"], "cur_ob_out")
    for k in ("step_count", "ep_return", "epoch_reward", "n_done", "b_obs", "b_next_obs", "b_acts", "b_values",
              "b_rewards", "b_terminals", "b_time_limits"):
        d[k].expect(want[k], k)
    if ret_log:
        d["ret_log"].expect(want["ret_log"], "ret_log")
    if device:
        for k in ("state", "elapsed", "episode"):
            d[k].expect(want[k], k)
        d["seeds"].expect(c["seeds"], "seeds (input)")
    mask = (c["done"] != 0) | (c["step_count"] + 1 >= FIN_MAXF)
    assert mask.any() and (~mask).any() or N < 32, "the case must mix reset and running envs"


def sample_call(mean, ls, ls_stride, eps, noise_scale, seed, ctr, tanh_action, nan=False):
    M, a = mean.shape

    def run():
        act, pre, lp, eo = Guarded(M, a), Guarded(M, a), Guarded(M), Guarded(M, a)
        flag = guarded_ints(1, torch.int32, 0)
        call("trl_tanh_gaussian_sample", mean.data_ptr(), ls.data_ptr(), ls_stride,
             None if eps is None else eps.data_ptr(), noise_scale, seed, None if ctr is None else ctr.data_ptr(), M, a,
             tanh_action, act.t.data_ptr(), pre.t.data_ptr(), lp.t.data_ptr(), eo.t.data_ptr(), flag.t.data_ptr(),
             stream())
        return [act.check("action"), pre.check("pre_tanh"), lp.check("log_prob"), eo.check("eps_out"),
                flag.check("nan_flag")]

    return twice(run)


def check_sample_formula(mean, ls_full, out, tanh_action):
    """action, pre-tanh and log-prob against the formula in fp64 applied to the returned noise e:
      z = mu + exp(ls) e: expf (2 ulp = 4U relative) and the fma (U):           e_z <= 4U |sd e| + U |z|
      a = tanh(z): the z error through tanh' <= 1 and tanhf's 2 ulp (4U):        e_a <= e_z + 4U |a|
      l_j = -e^2/2 - ls - log(2 pi)/2 - log(1 - a^2 + 1e-6) with the kernel's own a (fp32): the square and the three
            additions (4U of the magnitudes), the fp32 constant (U/2), w = 1 - a^2 + 1e-6 off by U a^2 + 2U w, logf's 2
            ulp on log w; the fp32 sum over the columns adds (cols - 1) U sum |l_j|; doubled for second-order terms."""
    act, pre, lp, e = [t.double() for t in out[:4]]
    mu, ls = mean.double(), ls_full.double()
    sd = ls.exp()
    z = mu + sd * e
    ez = 4 * U * (sd * e).abs() + U * z.abs()
    assert torch.all((pre - z).abs() <= ez + 1e-300), "pre-tanh beyond the bound"
    a_ref = torch.tanh(z) if tanh_action else z
    ea = ez + 4 * U * a_ref.abs() if tanh_action else ez
    assert torch.all((act - a_ref).abs() <= ea + 1e-300), "action beyond the bound"
    l = -0.5 * e * e - ls - 0.5 * math.log(2 * math.pi)
    el = 4 * U * (0.5 * e * e + ls.abs() + 1) + 0.5 * U
    if tanh_action:
        w = 1 - act * act + float(np.float32(1e-6))
        L = torch.log(w)
        l = l - L
        el = el + (U * act * act + 2 * U * w) / w + 8 * U * L.abs()
    cols = e.shape[1]
    bound = 2 * (el.sum(1) + (cols - 1) * U * l.abs().sum(1))
    assert torch.all((lp - l.sum(1)).abs() <= bound), "log-prob beyond the bound"


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 127, 128, 129])
@pytest.mark.parametrize("a", [1, 3, 4, 5, 8, 17])
def test_tanh_gaussian_sample_matches_the_formula(a, M):
    torch.manual_seed(a * 1000 + M)
    mean = 0.5 * torch.randn(M, a, device="cuda")
    for ls_stride in (0, a):
        ls = -1.0 + 0.3 * torch.randn(*((a,) if ls_stride == 0 else (M, a)), device="cuda")
        ls_full = ls.expand(M, a)
        for tanh_action in (1, 0):
            eps = torch.randn(M, a, device="cuda")
            out = sample_call(mean, ls, ls_stride, eps, 0.5, 0, None, tanh_action)
            assert same_bits(out[3], eps * 0.5), "eps_out is not the scaled given noise"
            check_sample_formula(mean, ls_full, out, tanh_action)
            assert int(out[4].item()) == 0
            ctr = torch.tensor([3], dtype=torch.int64, device="cuda")
            out = sample_call(mean, ls, ls_stride, None, 1.0, 1234, ctr, tanh_action)     # twice: same counter, same noise
            check_sample_formula(mean, ls_full, out, tanh_action)
            half = sample_call(mean, ls, ls_stride, None, 0.5, 1234, ctr, tanh_action)
            assert same_bits(half[3], out[3] * 0.5), "noise_scale does not scale the Philox noise"
            check_sample_formula(mean, ls_full, half, tanh_action)
            ctr += 1
            nxt = sample_call(mean, ls, ls_stride, None, 1.0, 1234, ctr, tanh_action)
            assert (nxt[3] == out[3]).double().mean().item() < 0.01, "counter + 1 gave the same noise"
            assert int(ctr.item()) == 4


@pytest.mark.gpu
@pytest.mark.parametrize("a", [5, 8, 17])
def test_tanh_gaussian_sample_philox_blocks_do_not_overlap(a):
    """M = 65536: every (row, block of 4 columns) draws its own Philox output -- two equal 4-tuples of normals would
    mean a shared counter or subsequence (chance equality of 4 floats is out of reach; single fp32 normals collide by
    chance thousands of times at this size).  A partial last block (act_dim 5, 17) must be the prefix of the full
    block a wider call draws: the Philox input of (row, block) does not depend on act_dim, so the overlap check of the
    act_dim rounded up to a multiple of 4 covers it."""
    M, full = 65536, -(-a // 4) * 4
    ctr = torch.tensor([7], dtype=torch.int64, device="cuda")
    wide = sample_call(torch.zeros(M, full, device="cuda"), torch.zeros(full, device="cuda"), 0, None, 1.0, 99, ctr, 1)
    quads = wide[3].reshape(M * full // 4, 4)
    assert torch.unique(quads, dim=0).shape[0] == quads.shape[0], "two (row, block) pairs share their noise"
    e = wide[3].double()
    assert abs(e.mean().item()) < 0.01 and abs(e.std().item() - 1) < 0.01
    if a != full:
        out = sample_call(torch.zeros(M, a, device="cuda"), torch.zeros(a, device="cuda"), 0, None, 1.0, 99, ctr, 1)
        assert same_bits(out[3], wide[3][:, :a].contiguous()), "the partial last block draws other noise"


@pytest.mark.gpu
def test_tanh_gaussian_sample_nan_flag_and_empty_batch():
    M, a = 129, 5
    mean, ls = torch.randn(M, a, device="cuda"), torch.zeros(a, device="cuda")
    assert int(sample_call(mean, ls, 0, None, 1.0, 1, None, 1)[4].item()) == 0
    mean[128, 3] = float("nan")
    out = sample_call(mean, ls, 0, None, 1.0, 1, None, 1)
    assert int(out[4].item()) == 1 and torch.isnan(out[0]).sum().item() == 1
    # M = 0 launches nothing, whatever the pointers
    call("trl_tanh_gaussian_sample", None, None, 0, None, 1.0, 0, None, 0, a, 1, None, None, None, None, None, stream())


# ================================================================================== E. pixel widening (atari_env.cu)
@pytest.mark.gpu
@pytest.mark.parametrize("n", [4, 7056 * 4 * 3, 2 * 16 * 132 * 256 * 4 + 148])
def test_u8_to_f32_is_exact(n):
    """float32(byte) * scale is one fp32 rounding on both sides; n = 4.3M takes the grid-stride loop past one lap of
    16 CTAs per SM"""
    x = torch.arange(n, dtype=torch.int64, device="cuda").remainder(256).to(torch.uint8)
    x[::7] = torch.randint(0, 256, x[::7].shape, dtype=torch.uint8, device="cuda")
    buf = torch.zeros(n + 8, dtype=torch.uint8, device="cuda")
    src = buf[4:4 + n]
    src.copy_(x)
    for scale in (1.0 / 255.0, 1.0, 0.5):
        def run():
            o = Guarded(n)
            call("trl_u8_to_f32", src.data_ptr(), o.t.data_ptr(), n, scale, stream())
            return [o.check()]

        (got,) = twice(run)
        assert same_bits(got, x.float() * torch.tensor(scale, dtype=torch.float32, device="cuda"))


# ============================================================================= F. argument validation (no GPU needed)
def _buf16():
    buf = (ctypes.c_uint8 * 256)()
    p = _host_ptr(buf)
    return buf, p + (-p % 16)


def test_row_copy_entry_points_reject_bad_arguments(native_lib):
    buf, p = _buf16()
    L = native_lib
    src, dst, rb = (vp * 9)(*[p] * 9), (vp * 9)(*[p] * 9), i64_table([4] * 9)
    _rejects(L, L.trl_row_gather(9, src, dst, rb, p, None, 1, None), "nkeys 9 not in 1..8")
    _rejects(L, L.trl_row_gather(0, src, dst, rb, p, None, 1, None), "nkeys 0 not in 1..8")
    _rejects(L, L.trl_row_gather(1, src, dst, rb, p, None, -1, None), "negative row count")
    _rejects(L, L.trl_row_gather(1, None, dst, rb, p, None, 1, None), "null key table")
    _rejects(L, L.trl_row_gather(2, (vp * 2)(p, None), dst, rb, p, None, 1, None), "key 1 has a null pointer")
    _rejects(L, L.trl_row_gather(1, src, dst, i64_table([0]), p, None, 1, None), "key 0 has a null pointer or empty row")
    _rejects(L, L.trl_row_gather(1, src, dst, rb, None, None, 1, None), "trl_row_gather: null index pointer")
    _rejects(L, L.trl_ring_write(1, src, dst, rb, None, None), "trl_ring_write: null row pointer")
    _rejects(L, L.trl_ring_write_advance(1, src, dst, rb, p, 0, None, p, None), "null pointer or T < 1")
    _rejects(L, L.trl_ring_write_advance(1, src, dst, rb, p, 4, None, None, None), "null pointer or T < 1")


def test_prioritized_entry_points_reject_bad_arguments(native_lib):
    buf, p = _buf16()
    L = native_lib
    _rejects(L, L.trl_per_sample(p, 0, p, 1, 0.4, p, p, None), "size 0 not in 1..4096")
    _rejects(L, L.trl_per_sample(p, 4097, p, 1, 0.4, p, p, None), "size 4097 not in 1..4096")
    _rejects(L, L.trl_per_sample(p, 8, p, 0, 0.4, p, p, None), "empty batch")
    _rejects(L, L.trl_per_sample(p, 8, None, 1, 0.4, p, p, None), "trl_per_sample: null pointer")
    _rejects(L, L.trl_per_update(p, p, p, 0, 1, 0.6, 1e-6, p, None), "trl_per_update: bad sizes")
    _rejects(L, L.trl_per_update(p, p, p, 1, 0, 0.6, 1e-6, p, None), "trl_per_update: bad sizes")
    _rejects(L, L.trl_per_update(p, p, p, 1, 1, 0.6, 1e-6, None, None), "trl_per_update: null pointer")
    _rejects(L, L.trl_per_insert(p, None, p, None), "trl_per_insert: null pointer")


def test_frame_entry_points_reject_bad_arguments(native_lib):
    buf, p = _buf16()
    L = native_lib
    W = L.trl_frame_ring_write
    _rejects(L, W(p, p, None, None, None, None, p, None, 1, 1, 16, 4, 0, None), "bad sizes N=1 C=1")
    _rejects(L, W(p, p, None, None, None, None, p, None, 1, 4, 24, 4, 3, None), "F=24")
    _rejects(L, W(p, p, None, None, None, None, p, None, 1, 4, 16, 4, 4, None), "frame=4")
    _rejects(L, W(p, p, None, None, None, None, p, None, 0, 4, 16, 4, 3, None), "N=0")
    _rejects(L, W(p, p, None, None, None, None, None, None, 1, 4, 16, 4, 3, None), "trl_frame_ring_write: null pointer")
    _rejects(L, W(p, p, p, None, None, None, p, None, 1, 4, 16, 4, 3, None), "age_ring and elapsed go together")
    _rejects(L, W(p, p, None, None, p, None, p, p, 1, 4, 16, 4, 3, None), "hist, hist_count and size go together")
    _rejects(L, W(p, p, None, None, p, p, p, None, 1, 4, 16, 4, 3, None), "hist, hist_count and size go together")
    _rejects(L, W(p + 4, p, None, None, None, None, p, None, 1, 4, 16, 4, 3, None), "16-byte aligned")
    _rejects(L, L.trl_frame_hist_advance(None, p, 4, None), "trl_frame_hist_advance: bad arguments")
    _rejects(L, L.trl_frame_hist_advance(p, p, 0, None), "trl_frame_hist_advance: bad arguments")
    G = L.trl_frame_stack_gather
    _rejects(L, G(p, p, p, p, p, p, None, 1, p, p, 1, 4, 20, 4, 1.0, p, p, None), "trl_frame_stack_gather: bad sizes")
    _rejects(L, G(p, p, p, p, p, p, None, -1, p, p, 1, 4, 16, 4, 1.0, p, p, None), "trl_frame_stack_gather: bad sizes")
    _rejects(L, G(p, p, p, None, p, p, None, 1, p, p, 1, 4, 16, 4, 1.0, p, p, None), "trl_frame_stack_gather: null")
    _rejects(L, G(p, p, p, p, p, p, None, 1, p, p, 1, 4, 16, 4, 1.0, p + 4, p, None), "16-byte aligned")


def test_collector_entry_points_reject_bad_arguments(native_lib):
    buf, p = _buf16()
    L = native_lib
    S = L.trl_tanh_gaussian_sample
    _rejects(L, S(p, p, 0, None, 1.0, 0, None, -1, 3, 1, p, None, None, None, None, None), "bad sizes")
    _rejects(L, S(p, p, 0, None, 1.0, 0, None, 4, 0, 1, p, None, None, None, None, None), "bad sizes")
    _rejects(L, S(p, p, 0, None, 1.0, 0, None, 4, 3, 1, None, None, None, None, None, None),
             "trl_tanh_gaussian_sample: null pointer")
    _rejects(L, S(p, p, 2, None, 1.0, 0, None, 4, 3, 1, p, None, None, None, None, None), "ls_stride must be 0 or act_dim")
    _rejects(L, L.trl_step_advance(p, 0, None, None, None), "T must be >= 1")
    _rejects(L, L.trl_u8_to_f32(p, p, 6, 1.0, None), "multiple of 4")
    _rejects(L, L.trl_u8_to_f32(p, p + 4, 8, 1.0, None), "null or misaligned pointer")
    _rejects(L, L.trl_u8_to_f32(p + 2, p, 8, 1.0, None), "null or misaligned pointer")
    F = L.trl_collect_finalize
    ptrs = [p] * 29
    _rejects(L, F(*ptrs, -1, 3, 2, 100, 0.99, 1.0, 5.0, 0, 0, None), "trl_collect_finalize: bad sizes")
    _rejects(L, F(*ptrs, 4, 0, 2, 100, 0.99, 1.0, 5.0, 0, 0, None), "trl_collect_finalize: bad sizes")
    _rejects(L, F(*([None] + ptrs[1:]), 4, 3, 2, 100, 0.99, 1.0, 5.0, 0, 0, None), "trl_collect_finalize: null pointer")
    no_state = list(ptrs)
    no_state[2] = None                                           # state missing, elapsed / episode / seeds given
    _rejects(L, F(*no_state, 4, 3, 2, 100, 0.99, 1.0, 5.0, 0, 0, None), "all given")
    no_value = list(ptrs)
    no_value[4] = None                                           # b_values without value
    _rejects(L, F(*no_value, 4, 3, 2, 100, 0.99, 1.0, 5.0, 0, 0, None), "b_values given without value")
