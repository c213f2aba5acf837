"""The loss, optimizer and statistics kernels called straight through the C ABI and compared with float64 restatements
of the same operation: the PPO / A2C actor and critic losses and the Gaussian log-probability (csrc/ppo_loss.cu), the
categorical actor loss (csrc/categorical.cu), the off-policy targets and losses (csrc/offpolicy.cu), the gradient norm
and Adam step (csrc/optim.cu), the vector and row-group statistics (csrc/gather.cu), the observation normaliser
(csrc/obs_norm.cu) and the backward of the reparameterised tanh-Gaussian sample (csrc/collect.cu).

Conventions (those of test_layer_kernels.py, with one change):
  * every output is a view into a larger NaN-filled buffer whose guards must still be NaN after the call;
  * the cross-CTA scratch is exactly as long as its size query says and sits inside a guard region; each case runs
    once with the scratch filled with +1e300 and once with -1e300, and both runs must give identical bits.  NaN would
    not do: the folds' fmax / fmin drop NaN, so an unwritten max / min slot would go unnoticed.  The guard region must
    still hold the sentinel afterwards, and the ticket must be back at zero after every call;
  * the two runs are also the repeat of every call: a fixed reduction order gives identical bits;
  * small-integer cases must match the exact result where the arithmetic is exact;
  * random cases check against float64 with a bound derived next to each check (U = 2^-24, the fp32 unit round-off;
    first-order error analysis, doubled where second-order terms are dropped).
The tests without the `gpu` mark check argument validation; nothing is launched there.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import ref_numpy as rn
from tests.test_layer_kernels import U, Guarded, _host_ptr, _rejects, assert_within, call, lib, rna_tf32_bits, \
    same_bits, stream, twice

GUARD = 64
SENTINELS = (1e300, -1e300)
B_EDGES = [1, 2, 255, 256, 257, 8192, 8193, 70000]
E53 = 2.0 ** -53                # fp64 unit round-off
HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)
F32 = lambda v: float(np.float32(v))      # a constant as the kernels see it (fp32)


# ------------------------------------------------------------------------------------------------------------- helpers
class Scratch:
    """n doubles filled with `fill` inside GUARD doubles of the same value on each side."""

    def __init__(self, n, fill):
        self.n, self.fill = int(n), fill
        self.buf = torch.full((self.n + 2 * GUARD,), fill, dtype=torch.float64, device="cuda")
        self.t = self.buf[GUARD:GUARD + self.n]

    def check(self):
        assert (self.buf[:GUARD] == self.fill).all() and (self.buf[GUARD + self.n:] == self.fill).all(), \
            "scratch: a write landed outside its advertised size"


class Guarded64:
    """a float64 / int32 output inside a guard region of `fill` (NaN for doubles)"""

    def __init__(self, *shape, dtype=torch.float64, fill=float("nan")):
        self.n = math.prod(shape)
        self.fill = fill
        self.buf = torch.full((self.n + 2 * GUARD,), fill, dtype=dtype, device="cuda")
        self.t = self.buf[GUARD:GUARD + self.n].view(shape)

    def check(self, what="output"):
        for g in (self.buf[:GUARD], self.buf[GUARD + self.n:]):
            ok = torch.isnan(g).all() if isinstance(self.fill, float) and math.isnan(self.fill) else (g == self.fill).all()
            assert ok, "%s: a write landed outside the output" % what
        return self.t


def ptr(t):
    return None if t is None else t.data_ptr()


def poisoned(n, run):
    """run(scratch_ptr, ticket_ptr) -> outputs.  Called with the scratch (exactly n doubles) at +1e300, then at -1e300;
    the ticket must be back at zero after each call and both calls must give identical bits."""
    tk = torch.zeros(1, dtype=torch.int32, device="cuda")
    outs = []
    for fill in SENTINELS:
        s = Scratch(n, fill)
        outs.append([t.clone() for t in run(s.t.data_ptr(), tk.data_ptr())])
        s.check()
        assert int(tk.item()) == 0, "ticket not back at zero"
    for i, (a, b) in enumerate(zip(*outs)):
        assert same_bits(a, b), "output %d differs between a +1e300 and a -1e300 scratch: a partial slot that no CTA " \
                                "wrote was folded in" % i
    return outs[0]


def close(got, ref, bound, what):
    """|got - ref| <= bound with got finite (assert_within on any shape, scalars included)"""
    got = torch.as_tensor(got).reshape(-1)
    ref = torch.as_tensor(ref, dtype=torch.float64, device=got.device).reshape(-1)
    assert_within(got, ref, torch.as_tensor(bound, dtype=torch.float64, device=got.device).reshape(-1) + 1e-300, what)


def exact(got, ref, what):
    got = torch.as_tensor(got)
    ref = torch.as_tensor(ref, device=got.device).to(got.dtype)
    assert same_bits(got.reshape(-1), ref.reshape(-1)), "%s: %r != %r (exact)" % (what, got.reshape(-1)[:8].tolist(),
                                                                                 ref.reshape(-1)[:8].tolist())


def gen(seed):
    torch.manual_seed(seed)


def randn(*shape):
    return torch.randn(*shape, device="cuda")


def ints(lo, hi, *shape):
    return torch.randint(lo, hi + 1, shape, device="cuda").float()


def mean_sum_bound(x, depth):
    """fp64 sum of fp32 values along a reduction tree of the given depth: depth * 2^-53 * sum |x|"""
    return depth * E53 * x.double().abs().sum().item()


# ======================================================================================= A. ppo_loss.cu: actor, critic
ACT_DIMS = [1, 2, 6, 17, 26, 27, 32]
CLIP, ENT = 0.25, 2.0 ** -7      # binary fractions: the kernel's 1 -+ clip and ent_coef equal the reference's exactly
LS_CLAMP = (-2.0, -1.0)


def gaussian_terms(mean, ls, acts, tanh):
    """float64 per-dimension pieces of TanhNormal.log_prob and the first-order bound of the kernel's fp32 evaluation
    of each term l_j = -d^2/2 - ls - log(2 pi)/2 [- log(1 - a^2 + 1e-6)], d = (z - mu) / exp(ls):
      z = atanh(a) = log((1+a)/(1-a))/2:  three roundings in the quotient, logf's 2 ulp:   e_z <= 2U (1 + |z|)
      d: subtraction, expf (2 ulp), division:                                             e_d <= e_z / sd + 4U |d|
      l_j: the square (|d| e_d + U d^2), three additions (3U of the magnitudes added), the fp32 constant (U/2), and
           log(w), w = 1 - a^2 + 1e-6 with w off by U a^2 + 2U w and logf's 2 ulp:  (U a^2 + 2U w)/w + 2U |log w|
    and the fp32 sum over a terms adds (a-1) U sum |l_j|."""
    x = acts.double()
    lsb = ls.double().expand(x.shape)
    sd = lsb.exp()
    z = 0.5 * torch.log((1 + x) / (1 - x)) if tanh else x
    d = (z - mean.double()) / sd
    l = -0.5 * d * d - lsb - HALF_LOG_2PI
    e_z = 2 * U * (1 + z.abs()) if tanh else torch.zeros_like(z)
    e_d = e_z / sd + 4 * U * d.abs()
    e_l = d.abs() * e_d + U * d * d + 3 * U * (0.5 * d * d + lsb.abs() + 1)
    if tanh:
        w = 1 - x * x + F32(1e-6)
        L = torch.log(w)
        l = l - L
        e_l = e_l + 3 * U * L.abs() + (U * x * x + 2 * U * w) / w + 2 * U * L.abs()
    a = x.shape[1]
    e_lp = 2 * (e_l.sum(1) + (a - 1) * U * l.abs().sum(1))       # x2: second-order terms
    return dict(lp=l.sum(1), d=d, sd=sd, e_d=2 * e_d, e_lp=e_lp)


def ref_actor(mean, ls_raw, acts, old, advs, st, tanh, clamp):
    """float64 autograd restatement of PPO.update_actor (old given) / A2C's policy gradient (old None) with the Normal
    entropy bonus, the advantage normalisation by a stats row and torch.clamp of the raw log-std"""
    m = mean.double().requires_grad_()
    lr = ls_raw.double().requires_grad_()
    ls = lr.clamp(*clamp) if clamp else lr
    lsb = ls.expand(m.shape)
    x = acts.double()
    z = 0.5 * torch.log((1 + x) / (1 - x)) if tanh else x
    d = (z - m) / lsb.exp()
    l = -0.5 * d * d - lsb - HALF_LOG_2PI
    if tanh:
        l = l - torch.log(1 - x * x + F32(1e-6))
    lp = l.sum(1)
    adv = advs.double() if st is None else (advs.double() - st[0]) / (st[1] + F32(1e-5))
    if old is None:
        ratio = torch.ones_like(lp)
        Lb = -lp * adv
    else:
        ratio = torch.exp(lp - old.double())
        Lb = -torch.min(ratio.clamp(1 - CLIP, 1 + CLIP) * adv, ratio * adv)     # torch splits the gradient on ties
    ent = (0.5 + HALF_LOG_2PI + lsb).sum(1)
    loss = Lb.mean() - ENT * ent.mean()
    g_m, g_ls = torch.autograd.grad(loss, [m, lr])
    return dict(loss=loss.item(), lp=lp.detach(), ratio=ratio.detach(), adv=adv.detach(), Lb=Lb.detach(), g_m=g_m,
                g_ls=g_ls, ls=ls.detach(), ent=ent.mean().item())


def actor_case(B, a, shared, j):
    """inputs of case j: the options rotate over the batch sizes so every combination of (tanh, PPO/A2C, stats row,
    clamp) meets several B"""
    tanh, ppo, stats, clamp = j % 2 == 0, j % 3 != 2, (j // 2) % 2 == 0, (j // 4) % 2 == 1 or j == 7
    mean = 0.5 * randn(B, a)
    ls_raw = -1.5 + 0.6 * randn(*((a,) if shared else (B, a)))
    z = (mean + ls_raw.clamp(*LS_CLAMP).exp() * 1.3 * randn(B, a)).clamp(-4, 4)     # |a| <= tanh(4): not saturated
    acts = torch.tanh(z) if tanh else z
    table = torch.stack([0.3 * randn(3), 0.5 + torch.rand(3, device="cuda"), randn(3), randn(3)], 1) if stats else None
    pos = torch.tensor([2], dtype=torch.int32, device="cuda") if stats else None
    advs = 2 * randn(B) + 0.3
    return dict(tanh=tanh, ppo=ppo, mean=mean, ls_raw=ls_raw, acts=acts, table=table, pos=pos, advs=advs,
                clamp=LS_CLAMP if clamp else None)


def run_actor(c, old, B, a, shared):
    lo, hi = c["clamp"] if c["clamp"] else (1.0, -1.0)        # ls_min > ls_max: no clamp

    def run(scratch, ticket):
        gm, gl, lpo, info = Guarded(B, a), Guarded(*c["ls_raw"].shape), Guarded(B), Guarded(16)
        call("trl_ppo_actor_loss", c["mean"].data_ptr(), c["ls_raw"].data_ptr(), 0 if shared else a,
             c["acts"].data_ptr(), ptr(old), c["advs"].data_ptr(), ptr(c["table"]), ptr(c["pos"]), B, a, int(c["tanh"]),
             CLIP, ENT, lo, hi, gm.t.data_ptr(), gl.t.data_ptr(), lpo.t.data_ptr(), info.t.data_ptr(), scratch, ticket,
             stream())
        return [gm.check("g_mean"), gl.check("g_log_std"), lpo.check("logp_out"), info.check("info")[:13]]
    return poisoned(lib().trl_ppo_actor_scratch_doubles(B, a), run)


@pytest.mark.gpu
@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("a", ACT_DIMS)
def test_ppo_actor_loss_matches_fp64(a, shared):
    """All 13 info slots, both gradients and logp_out against float64 autograd, at every CTA / fold edge of B.  With a
    shared log-std and a >= 27 the per-CTA max / min partials were once left unwritten (the sum slots took their
    threads): the sentinel comparison and logprob/max, ratio max / min catch it."""
    for j, B in enumerate(B_EDGES):
        gen(1000 * a + 10 * j + shared)
        c = actor_case(B, a, shared, j)
        what = "a=%d shared=%d B=%d tanh=%d ppo=%d stats=%d clamp=%d" % (a, shared, B, c["tanh"], c["ppo"],
                                                                         c["table"] is not None, bool(c["clamp"]))
        ls = c["ls_raw"].clamp(*c["clamp"]) if c["clamp"] else c["ls_raw"]
        gt = gaussian_terms(c["mean"], ls, c["acts"], c["tanh"])
        st = None if c["table"] is None else c["table"][2].double()
        old = None
        if c["ppo"]:
            old = (gt["lp"] + 0.3 * randn(B).double()).float()
            old[::7] = gt["lp"][::7].float()                       # ratio ~ 1: in range, both surrogates tie
            ratio = torch.exp(gt["lp"] - old.double())
            e_r = 2 * ratio * (gt["e_lp"] + U * (gt["lp"] - old.double()).abs() + 2 * U)   # expf: 2 ulp, + the argument
            # rows whose ratio is within its error of a clip edge may take the other branch in fp32: zero advantage
            risky = ((ratio - (1 - CLIP)).abs() <= 2 * e_r) | ((ratio - (1 + CLIP)).abs() <= 2 * e_r)
            c["advs"][risky] = 0.0 if st is None else c["table"][2, 0]
        r = ref_actor(c["mean"], c["ls_raw"], c["acts"], old, c["advs"], st, c["tanh"], c["clamp"])
        g_m, g_ls, lpo, info = run_actor(c, old, B, a, shared)

        e_lp = gt["e_lp"]
        close(lpo, r["lp"], e_lp, "logp_out " + what)
        adv, lp = r["adv"], r["lp"]
        e_a = 4 * U * adv.abs() if st is not None else torch.zeros_like(adv)   # (adv - m) / (s + 1e-5): 3 roundings
        if c["ppo"]:
            ratio = r["ratio"]
            e_r = 2 * ratio * (e_lp + U * (lp - old.double()).abs() + 2 * U)
            e_L = adv.abs() * e_r + (ratio + e_r) * e_a + U * r["Lb"].abs()
            cabs = adv.abs() * ratio / B                           # |dL/dlogp_b|
            e_c = (adv.abs() * e_r + ratio * e_a) / B + 3 * U * cabs
        else:
            e_r = torch.zeros_like(lp)
            e_L = adv.abs() * e_lp + lp.abs() * e_a + U * r["Lb"].abs()
            cabs = adv.abs() / B
            e_c = e_a / B + 2 * U * cabs
        info = info.double()
        # [0] loss: mean of the per-row errors, the fp32 constant in the entropy (a U / 2), the cast
        close(info[0], r["loss"], e_L.mean() + ENT * a * U + 2 * U * abs(r["loss"]), "policy loss " + what)
        close(info[1], lp.mean(), e_lp.mean() + U * lp.abs().mean(), "logprob/mean " + what)
        if B == 1:
            assert info[2].item() == 0.0, "logprob/std at B = 1 is pinned to 0 (torch gives nan)"
        else:
            # std is sqrt(n/(n-1)) * an L2 norm: moves by at most sqrt(B/(B-1)) max|e|; plus fp64 cancellation and the
            # cast
            sd = lp.std().item()
            close(info[2], sd, math.sqrt(B / (B - 1)) * e_lp.max().item() + 2 * U * sd +
                  600 * E53 * (lp * lp).mean().item() / max(sd, 1e-30), "logprob/std " + what)
        close(info[3], lp.max(), e_lp.max(), "logprob/max " + what)
        close(info[4], lp.min(), e_lp.max(), "logprob/min " + what)
        if c["ppo"]:
            close(info[5], r["ratio"].max(), e_r.max(), "ratio max " + what)
            close(info[6], r["ratio"].min(), e_r.max(), "ratio min " + what)
            close(info[12], (old.double() - lp).mean(), e_lp.mean() + U * (old.double() - lp).abs().mean(),
                  "approx kl " + what)
        else:
            assert info[5].item() == 1.0 and info[6].item() == 1.0 and info[12].item() == 0.0, what
        lsd = r["ls"]
        if shared:
            # the log-std statistics come straight from the a parameters in fp64: the cast only
            close(info[7], lsd.mean(), U * lsd.abs().max(), "ls mean " + what)
            if a == 1:
                assert math.isnan(info[8].item()), "ls std of one shared entry is nan, as torch.std"
            else:
                close(info[8], lsd.std(), 2 * U * lsd.std() + 1e-12, "ls std " + what)
            ent = a * (0.5 + HALF_LOG_2PI) + lsd.sum().item()
            e_ent = a * U + U * abs(ent)
        else:
            # per-row ls sums are fp32 over the a dims of a row: a U sum |ls|, (a + 1) U sum ls^2
            cnt = B * a
            e_s = a * U * lsd.abs().sum().item()
            e_q = (a + 1) * U * (lsd * lsd).sum().item()
            mu = lsd.mean().item()
            close(info[7], mu, e_s / cnt + U * abs(mu), "ls mean " + what)
            if cnt == 1:
                assert info[8].item() == 0.0, "ls std of a single entry is pinned to 0"
            else:
                sd = lsd.std().item()
                dv = (e_q + 2 * abs(mu) * e_s) / (cnt - 1)
                close(info[8], sd, min(dv / max(2 * sd, 1e-300), math.sqrt(dv)) + 2 * U * sd, "ls std " + what)
            ent = a * (0.5 + HALF_LOG_2PI) + lsd.sum().item() / B
            e_ent = a * U + e_s / B + U * abs(ent)
        exact(info[9], lsd.max().float(), "ls max " + what)
        exact(info[10], lsd.min().float(), "ls min " + what)
        close(info[11], r["ent"], e_ent, "entropy " + what)
        # gradients: g_mean = c d / sd, g_ls = c (d^2 - 1) - ent_coef / B per row
        d, sdv, e_d = gt["d"], gt["sd"], gt["e_d"]
        cabs, e_c = cabs[:, None], e_c[:, None]
        e_gm = (d / sdv).abs() * e_c + cabs * (e_d / sdv + 4 * U * d.abs() / sdv)
        close(g_m, r["g_m"], 2 * e_gm + U * r["g_m"].abs(), "g_mean " + what)
        e_gl = (d * d - 1).abs() * e_c + cabs * (2 * d.abs() * e_d + 2 * U * (d * d + 1))
        if shared:
            close(g_ls, r["g_ls"], 2 * e_gl.sum(0) + 2 * U * r["g_ls"].abs() + 2 * U * ENT, "g_log_std " + what)
        else:
            close(g_ls, r["g_ls"], 2 * e_gl + 2 * U * r["g_ls"].abs() + 2 * U * ENT / B, "g_log_std " + what)
        if c["clamp"]:
            raw = c["ls_raw"]
            assert (g_ls[(raw < LS_CLAMP[0]) | (raw > LS_CLAMP[1])] == 0).all(), "clamped entries pass no gradient"


@pytest.mark.gpu
@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("a", ACT_DIMS)
def test_gaussian_log_prob_matches_fp64(a, shared):
    for j, B in enumerate([1, 257, 8193]):
        gen(7 * a + j + 100 * shared)
        tanh = (j + a) % 2 == 0
        c = actor_case(B, a, shared, 0)
        ls = c["ls_raw"]

        def run():
            out = Guarded(B)
            call("trl_gaussian_log_prob", c["mean"].data_ptr(), ls.data_ptr(), 0 if shared else a, c["acts"].data_ptr()
                 if tanh else c["acts"].atanh().data_ptr(), B, a, int(tanh), out.t.data_ptr(), stream())
            return [out.check("logp")]
        lp = twice(run)[0]
        gt = gaussian_terms(c["mean"], ls, c["acts"] if tanh else c["acts"].atanh(), tanh)
        close(lp, gt["lp"], gt["e_lp"], "gaussian_log_prob a=%d shared=%d B=%d tanh=%d" % (a, shared, B, tanh))


def ref_critic(v, ret, old, clipped, clip):
    vd = v.double().requires_grad_()
    if clipped:          # ppo.py:100-107; torch.max splits the gradient on ties, clamp passes it at the edges
        vc = old.double() + (vd - old.double()).clamp(-clip, clip)
        loss = 0.5 * torch.max((vd - ret.double()) ** 2, (vc - ret.double()) ** 2).mean()
    else:
        loss = ((vd - ret.double()) ** 2).mean()
    g, = torch.autograd.grad(loss, vd)
    return loss, g


def run_critic(v, ret, old, clipped, clip):
    B = v.numel()

    def run(scratch, ticket):
        g, info = Guarded(B), Guarded(1)
        call("trl_ppo_critic_loss", v.data_ptr(), ret.data_ptr(), ptr(old), B, int(clipped), clip, g.t.data_ptr(),
             info.t.data_ptr(), scratch, ticket, stream())
        return [g.check("g_values"), info.check("vf_loss")]
    return poisoned(-(-B // 256), run)


def inv_b(B):
    return torch.tensor(1.0) / torch.tensor(float(B))          # the kernels' 1.0f / B (fp32, correctly rounded)


@pytest.mark.gpu
@pytest.mark.parametrize("clipped", [False, True])
@pytest.mark.parametrize("B", B_EDGES)
def test_ppo_critic_loss_matches_fp64(B, clipped):
    gen(B + clipped)
    # integer-exact: every difference, square and fp64 sum is exact; the loss is one fp64 division then the cast, and
    # the gradient one fp32 product with the kernel's 1/B
    v, ret, old = ints(-6, 6, B), ints(-6, 6, B), ints(-6, 6, B)
    clip = 2.0
    g, info = run_critic(v, ret, old, clipped, clip)
    loss, gref = ref_critic(v, ret, old, clipped, clip)
    d1 = v.double() - ret.double()
    if clipped:
        dv = v.double() - old.double()
        d2 = old.double() + dv.clamp(-clip, clip) - ret.double()
        lsum = (0.5 * torch.max(d1 * d1, d2 * d2)).sum()
        gsel = gref * B                                             # the unscaled selected gradient (exact halves)
        if B > 100:
            assert ((d1 * d1 == d2 * d2) & (d1 != d2)).any(), "ties with different gradients must be present"
    else:
        lsum = (d1 * d1).sum()
        gsel = 2 * d1
    exact(info, torch.tensor([lsum.item() / B]).float(), "integer vf_loss B=%d" % B)
    exact(g, (gsel.float().cpu() * inv_b(B)).cuda(), "integer g_values B=%d" % B)
    # random: d1 one rounding, the square one more (and the fp32 halving / max exact): 3U relative on each row's loss
    # and gradient; the fp64 sum adds nothing at this scale, the cast U
    v, ret = randn(B), randn(B)
    old = v + 0.4 * randn(B)
    g, info = run_critic(v, ret, old, clipped, 0.25)
    loss, gref = ref_critic(v, ret, old, clipped, 0.25)
    d1 = (v.double() - ret.double())
    close(info, loss.item(), 3 * U * loss.item() + U * loss.item(), "random vf_loss B=%d" % B)
    keep = torch.ones(B, dtype=torch.bool, device="cuda")
    if clipped:       # rows within round-off of a branch edge may take the other branch: their gradient is not compared
        dv = v.double() - old.double()
        d2 = old.double() + dv.clamp(-0.25, 0.25) - ret.double()
        keep = ((d1 * d1 - d2 * d2).abs() > 8 * U * (d1 * d1 + d2 * d2)) & ((dv.abs() - 0.25).abs() > 4 * U *
                                                                           (v.double().abs() + old.double().abs()))
    close(g[keep], gref[keep], 4 * U * gref[keep].abs(), "random g_values B=%d" % B)


# ====================================================================================== B. categorical.cu: actor loss
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["ppo", "a2c"])
@pytest.mark.parametrize("B,A", [(1, 32), (1, 6), (257, 32), (8193, 32), (8193, 5), (70000, 18)])
def test_categorical_actor_loss_edges(B, A, mode):
    """The edges test_categorical_kernels.py does not reach: B = 1, B >= 8193 (the lane-strided fold loops more than
    once), A = 32, with the sentinel scratch, ticket and guards.  The reference is that file's float32 torch autograd of
    Categorical(softmax(x)), at its tolerance (2e-4, the float32 reference's own accuracy at these magnitudes)."""
    from tests.test_categorical_kernels import _logits, _torch_ref
    rs = np.random.RandomState(B + A)
    x = _logits(B, A, B * A)
    acts = rs.randint(0, A, B)
    advs = rs.randn(B).astype(np.float32)
    table = np.array([[0.1, 1.3, 0, 0], [-0.2, 0.7, 0, 0]], dtype=np.float32)
    with torch.no_grad():
        lp_now = torch.distributions.Categorical(torch.softmax(torch.tensor(x), -1)).log_prob(
            torch.as_tensor(acts)).numpy()
    old = None
    if mode == "ppo":
        old = (lp_now + rs.randn(B) * 0.3).astype(np.float32)
        old[::7] = lp_now[::7]
    xd, ad, advd = torch.tensor(x, device="cuda"), torch.tensor(acts, dtype=torch.float32, device="cuda"), \
        torch.tensor(advs, device="cuda")
    od = None if old is None else torch.tensor(old, device="cuda")
    tbl, pos = torch.tensor(table, device="cuda"), torch.tensor([1], dtype=torch.int32, device="cuda")

    def run(scratch, ticket):
        g, lpo, info = Guarded(B, A), Guarded(B), Guarded(16)
        call("trl_ppo_categorical_actor_loss", xd.data_ptr(), ad.data_ptr(), ptr(od), advd.data_ptr(), tbl.data_ptr(),
             pos.data_ptr(), B, A, 0.2, 0.01, g.t.data_ptr(), lpo.t.data_ptr(), info.t.data_ptr(), scratch, ticket,
             stream())
        return [g.check("g_logits"), lpo.check("logp"), info.check("info")[:13]]
    g, lpo, info = poisoned(lib().trl_ppo_categorical_actor_scratch_doubles(B), run)
    ref = _torch_ref(x, acts, old, advs, (float(table[1, 0]), float(table[1, 1])), 0.2, 0.01)
    info = info.cpu().numpy()
    assert np.isfinite(info).all()
    np.testing.assert_allclose(lpo.cpu().numpy(), ref["lp"], atol=2e-4)
    np.testing.assert_allclose(info[0], ref["loss"], atol=2e-4, rtol=2e-4)
    np.testing.assert_allclose(info[1], ref["lp"].mean(), atol=2e-4)
    if B == 1:
        assert info[2] == 0.0, "logprob/std at B = 1 is pinned to 0 (torch gives nan)"
    else:
        np.testing.assert_allclose(info[2], ref["lp"].astype(np.float64).std(ddof=1), atol=2e-4, rtol=1e-3)
    np.testing.assert_allclose(info[3:5], [ref["lp"].max(), ref["lp"].min()], atol=2e-4)
    np.testing.assert_allclose(info[5:7], [ref["ratio"].max(), ref["ratio"].min()], atol=2e-4, rtol=2e-4)
    assert (info[7:11] == 0).all()
    np.testing.assert_allclose(info[11], ref["ent"], atol=2e-4)
    np.testing.assert_allclose(g.cpu().numpy() * B, ref["g"] * B, atol=2e-4, rtol=2e-3)


# ===================================================================================== C. offpolicy.cu
def off_scratch(B):
    return lib().trl_offpolicy_scratch_doubles(B)


def run_td_target(r, d, q1, q2, lp, la, alpha, gamma):
    B = r.numel()

    def run(scratch, ticket):
        y, info = Guarded(B), Guarded(1)
        call("trl_td_target", r.data_ptr(), d.data_ptr(), q1.data_ptr(), ptr(q2), ptr(lp), ptr(la), alpha, gamma, B,
             y.t.data_ptr(), info.t.data_ptr(), scratch, ticket, stream())
        return [y.check("y"), info.check("reward mean")]
    return poisoned(off_scratch(B), run)


TD_FORMS = ["sac_device_alpha", "sac_fixed_alpha", "td3_twin", "single_critic"]


@pytest.mark.gpu
@pytest.mark.parametrize("form", TD_FORMS)
@pytest.mark.parametrize("B", [1, 255, 257, 8193, 70000])
def test_td_target_matches_oracle(B, form):
    gen(B)
    twin, soft = form != "single_critic", form.startswith("sac")
    dev_alpha = form == "sac_device_alpha"
    # integer-exact: small integers, gamma = alpha = 1/2 (log_alpha = -ln 2 is not exact in fp32: fixed alpha only)
    r, q1, q2, lp = ints(-8, 8, B), ints(-8, 8, B), ints(-8, 8, B), ints(-8, 8, B)
    d = (torch.rand(B, device="cuda") < 0.3).to(torch.uint8)
    if not dev_alpha:
        y, info = run_td_target(r, d, q1, q2 if twin else None, lp if soft else None, None, 0.5, 0.5)
        q = torch.minimum(q1, q2) if twin else q1
        ref = rn.sac_q_target(*[t.double().cpu().numpy() for t in (r, d, q, q, lp if soft else 0 * lp)], 0.5, 0.5)
        exact(y, torch.from_numpy(ref).float(), "integer y " + form)
        exact(info, torch.tensor([r.double().sum().item() / B]).float(), "integer reward mean " + form)
    # random, against the oracle with the kernel's fp32 gamma / alpha: fminf exact, then alpha logp, the subtraction,
    # gamma v and the addition round once each (4U of the magnitudes), and expf's 2 ulp on a device alpha
    r, q1, q2, lp = randn(B), randn(B), randn(B), randn(B)
    la = torch.tensor([-0.7], device="cuda")
    alpha = math.exp(F32(-0.7)) if dev_alpha else F32(0.2)
    gamma = F32(0.99)
    y, info = run_td_target(r, d, q1, q2 if twin else None, lp if soft else None, la if dev_alpha else None, 0.2, 0.99)
    q = (torch.minimum(q1, q2) if twin else q1).double()
    lpd = lp.double() if soft else torch.zeros_like(q)
    ref = torch.from_numpy(rn.sac_q_target(*[t.double().cpu().numpy() for t in (r, d, q, q, lpd)], alpha, gamma))
    bnd = 4 * U * (r.double().abs() + gamma * (q.abs() + alpha * lpd.abs())) + \
        (2 * U * gamma * alpha * lpd.abs() if dev_alpha else 0)
    close(y, ref, bnd, "random y B=%d %s" % (B, form))
    close(info, r.double().mean(), U * r.double().abs().mean() + mean_sum_bound(r, 300) / B, "reward mean")


@pytest.mark.gpu
def test_sac_alpha_step_five_steps_match_fp64_adam():
    """5 consecutive steps of the fused alpha loss + one-parameter Adam against a float64 Adam (the kernel's fp32
    constants).  Each step's update lr m / (sqrt(v) / sqrt(bc2) + eps) / bc1 is evaluated with about ten fp32 roundings
    (12 U of it), log_alpha itself is rounded once per step (U |log_alpha|); the errors add over the steps."""
    B = 8193
    gen(3)
    lr, b1, b2, eps, target = F32(3e-4), F32(0.9), F32(0.999), F32(1e-8), -6.0
    la = torch.zeros(1, device="cuda")
    st = torch.zeros(3, device="cuda")
    la64, m64, v64 = 0.0, 0.0, 0.0
    e_la = 0.0
    for t in range(1, 6):
        lp = randn(B) + 0.5 * t
        la_prev, st_prev = la.clone(), st.clone()

        def run(scratch, ticket):
            la.copy_(la_prev)
            st.copy_(st_prev)
            info = Guarded(2)
            call("trl_sac_alpha_step", lp.data_ptr(), target, la.data_ptr(), st.data_ptr(), 3e-4, 0.9, 0.999, 1e-8, B,
                 info.t.data_ptr(), scratch, ticket, stream())
            return [info.check("info"), la, st]
        info, la_k, st_k = poisoned(off_scratch(B), run)
        mt = (lp.double() + target).mean().item()
        loss = -la64 * mt
        g = -mt
        m64 = b1 * m64 + (1 - b1) * g
        v64 = b2 * v64 + (1 - b2) * g * g
        upd = (lr / (1 - b1 ** t)) * m64 / (math.sqrt(v64) / math.sqrt(1 - b2 ** t) + eps)
        la64 -= upd
        e_la += 12 * U * abs(upd) + U * abs(la64)
        close(la_k, la64, e_la, "log_alpha after step %d" % t)
        assert st_k[2].item() == t, "step count"
        close(st_k[0], m64, 4 * U * abs(m64) * t, "exp_avg step %d" % t)
        close(st_k[1], v64, 6 * U * v64 * t, "exp_avg_sq step %d" % t)
        close(info[0], math.exp(la64), math.exp(la64) * (e_la + 2 * U), "alpha step %d" % t)
        close(info[1], loss, abs(mt) * (e_la - 12 * U * abs(upd) - U * abs(la64)) + 2 * U * abs(loss) + 1e-30,
              "alpha loss step %d" % t)


def run_sac_policy(lp, q1, q2, la, alpha):
    B = lp.numel()

    def run(scratch, ticket):
        g_lp, g1, g2, info = Guarded(B), Guarded(B), Guarded(B), Guarded(5)
        call("trl_sac_policy_loss", lp.data_ptr(), q1.data_ptr(), q2.data_ptr(), ptr(la), alpha, B, g_lp.t.data_ptr(),
             g1.t.data_ptr(), g2.t.data_ptr(), info.t.data_ptr(), scratch, ticket, stream())
        return [g_lp.check("g_logp"), g1.check("g_q1"), g2.check("g_q2"), info.check("info")]
    return poisoned(off_scratch(B), run)


@pytest.mark.gpu
@pytest.mark.parametrize("dev_alpha", [False, True])
@pytest.mark.parametrize("B", [1, 2, 257, 8193, 70000])
def test_sac_policy_loss_matches_fp64(B, dev_alpha):
    gen(B + dev_alpha)
    lp, q1, q2 = ints(-8, 8, B), ints(-8, 8, B), ints(-8, 8, B)
    q2[::3] = q1[::3]                                           # ties: torch.min splits the gradient evenly
    la = torch.tensor([0.0], device="cuda")                     # alpha = exp(0) = 1 exactly
    alpha = 1.0 if dev_alpha else 0.5
    g_lp, g1, g2, info = run_sac_policy(lp, q1, q2, la if dev_alpha else None, 0.5)
    L = alpha * lp.double() - torch.minimum(q1, q2).double()
    ib = inv_b(B).item()
    exact(info[0], torch.tensor([L.sum().item() / B]).float(), "integer policy loss")
    exact(g_lp, torch.full((B,), F32(alpha * ib), device="cuda"), "integer g_logp")
    half = F32(-0.5 * ib)
    exact(g1, torch.where(q1 < q2, -ib, torch.where(q1 > q2, 0.0, half)).float(), "integer g_q1 (ties split)")
    exact(g2, torch.where(q2 < q1, -ib, torch.where(q2 > q1, 0.0, half)).float(), "integer g_q2 (ties split)")
    exact(info[3], lp.max(), "logp max")
    exact(info[4], lp.min(), "logp min")
    if B == 1:
        assert info[2].item() == 0.0, "logp std at B = 1 is pinned to 0 (torch gives nan)"
    # random: alpha logp - min(q): expf (2 ulp), product and difference round once each
    lp, q1, q2 = randn(B), randn(B), randn(B)
    q2[::5] = q1[::5]
    la = torch.tensor([-0.7], device="cuda")
    alpha = math.exp(F32(-0.7)) if dev_alpha else F32(0.5)
    g_lp, g1, g2, info = run_sac_policy(lp, q1, q2, la if dev_alpha else None, 0.5)
    L = alpha * lp.double() - torch.minimum(q1, q2).double()
    close(info[0], L.mean(), (4 * U * (alpha * lp.double().abs() + torch.minimum(q1, q2).double().abs())).mean() +
          U * L.abs().mean(), "random policy loss")
    close(info[1], lp.double().mean(), U * lp.double().abs().mean() + mean_sum_bound(lp, 300) / B, "logp mean")
    if B > 1:
        close(info[2], lp.double().std(), 2 * U * lp.double().std() + 1e-12, "logp std")
    close(g_lp, torch.full((B,), alpha / B, device="cuda"), 4 * U * alpha / B, "random g_logp")
    close(g1, torch.where(q1 < q2, -1.0 / B, torch.where(q1 > q2, 0.0, -0.5 / B)), U / B, "random g_q1")


@pytest.mark.gpu
@pytest.mark.parametrize("twin", [False, True])
@pytest.mark.parametrize("B", [1, 256, 257, 8193, 70000])
def test_twin_mse_loss_matches_fp64(B, twin):
    gen(B + twin)
    for integer in (True, False):
        q1, q2, y = (ints(-9, 9, B) for _ in range(3)) if integer else (randn(B) for _ in range(3))

        def run(scratch, ticket):
            g1, g2, info = Guarded(B), Guarded(B), Guarded(2)
            call("trl_twin_mse_loss", q1.data_ptr(), ptr(q2 if twin else None), y.data_ptr(), B, g1.t.data_ptr(),
                 g2.t.data_ptr() if twin else None, info.t.data_ptr(), scratch, ticket, stream())
            return [g1.check("g1"), g2.check("g2 (untouched without q2)"), info.check("info")]
        g1, g2, info = poisoned(off_scratch(B), run)
        for k, (q, g) in enumerate([(q1, g1), (q2, g2)]):
            if k == 1 and not twin:
                assert torch.isnan(g).all(), "g2 written without q2"
                assert info[1].item() == 0.0
                continue
            dd = q.double() - y.double()
            if integer:       # exact: the difference, square and fp64 sum; one fp64 division; fp32 (2d) * (1/B)
                exact(info[k], torch.tensor([(dd * dd).sum().item() / B]).float(), "integer loss %d" % k)
                exact(g, ((2 * dd).float().cpu() * inv_b(B)).cuda(), "integer grad %d" % k)
            else:             # two roundings in d^2, the cast; 2 d / B: the difference, the 1/B and the product
                close(info[k], (dd * dd).mean(), 3 * U * (dd * dd).mean(), "random loss %d B=%d" % (k, B))
                close(g, 2 * dd / B, 3 * U * (2 * dd / B).abs(), "random grad %d B=%d" % (k, B))


def ref_qr(pred, nxt, acts, r, d, w, gamma, Q, mse):
    """float64 restatement of QRDQN.update's loss (qrdqn.py:36-60; test_offpolicy._ref_qr) and of DQN's (mse), weighted
    per sample by the importance weights w: loss = mean_b w_b l_b.  The greedy action is numpy's argmax of the
    target means: the first maximum, as torch.max."""
    B = pred.shape[0]
    pred = pred.double().requires_grad_()
    nq = nxt.double().view(B, -1, Q)
    a_star = torch.from_numpy(np.argmax(nq.mean(2).cpu().numpy(), axis=1)).to(pred.device)
    picked = nq[torch.arange(B, device=pred.device), a_star]                      # (B, Q)
    tgt = r.double()[:, None] + gamma * (1 - d.double()[:, None]) * picked
    q_s_a = pred.view(B, -1, Q)[torch.arange(B, device=pred.device), acts.long()]  # (B, Q)
    if mse:
        per = ((q_s_a - tgt) ** 2)[:, 0]
        td = (q_s_a - tgt).abs()[:, 0]
    else:
        tau = torch.tensor((2 * np.arange(Q) + 1) / (2.0 * Q), device=pred.device).view(1, 1, -1)
        diff = tgt.unsqueeze(-1) - q_s_a.unsqueeze(1)                                 # (B, Q_target j, Q_source i)
        hub = torch.where(diff.abs() < 1.0, 0.5 * diff ** 2, diff.abs() - 0.5)
        per = (hub * (tau - (diff.detach() < 0).double()).abs()).mean((1, 2))
        td = per
    loss = (per * w.double()).mean()
    g, = torch.autograd.grad(loss, pred)
    return loss.item(), g, td.detach(), q_s_a.detach(), tgt.detach(), a_star


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("A", [1, 18])
@pytest.mark.parametrize("Q", [1, 5, 200, 257])
def test_qr_dqn_loss_matches_fp64(Q, A, weighted):
    """Q = 1 is DQN's squared error (mse); Q = 257 > 256 threads takes the strided quantile loop.  Target quantiles
    are integers with tied action means (a reversed copy of another action's quantiles, +12 so they are the maximum):
    the first maximum wins, and with Q > 1 the two tied actions give different targets."""
    mse = Q == 1
    for B in (1, 300):
        gen(Q * 100 + A + B + weighted)
        pred = randn(B, A * Q)
        nxt = ints(-4, 4, B, A, Q)
        if A > 1:
            nxt[:, 3] = nxt[:, 1].flip(-1)
            nxt[:, 1] += 12
            nxt[:, 3] += 12
        nxt = nxt.view(B, A * Q)
        acts = torch.randint(0, A, (B,), device="cuda").float()
        r = randn(B)
        d = (torch.rand(B, device="cuda") < 0.2).to(torch.uint8)
        w = (torch.rand(B, device="cuda") + 0.25) if weighted else torch.ones(B, device="cuda")
        gamma = F32(0.99)

        def run(scratch, ticket):
            g, td, info = Guarded(B, A * Q), Guarded(B), Guarded(3)
            call("trl_qr_dqn_loss", pred.data_ptr(), nxt.data_ptr(), acts.data_ptr(), r.data_ptr(), d.data_ptr(),
                 ptr(w if weighted else None), B, A, Q, 0.99, 1.0, int(mse), g.t.data_ptr(), td.t.data_ptr(),
                 info.t.data_ptr(), scratch, ticket, stream())
            return [g.check("grad"), td.check("td_out"), info.check("info")]
        g, td, info = poisoned(off_scratch(B), run)
        loss, gref, tdref, q_s_a, tgt, a_star = ref_qr(pred, nxt, acts, r, d, w, gamma, Q, mse)
        if A > 1:
            assert (a_star == 1).all(), "tied maxima: the first one wins"
        what = "Q=%d A=%d B=%d weighted=%d" % (Q, A, B, weighted)
        # y_j = r + gamma (1-d) n_j: two roundings (e_y); each term of the fp32 sum over j moves by at most
        # max(|u|, kappa) e_u through the 1-Lipschitz-per-|u| Huber (e_u = e_y + U |u|), its weight |tau - 1[u<0]| by U,
        # and the sum of Q terms adds Q U sum |terms|
        e_y = 2 * U * (2 * r.double().abs()[:, None] + tgt.abs())             # gamma |n_j| <= |y_j| + |r|
        if mse:
            dd = (q_s_a - tgt)[:, 0]
            e_dd = e_y[:, 0] + U * dd.abs()
            per_err = 2 * dd.abs() * e_dd + U * dd * dd
            close(td, dd.abs(), e_dd + 2 * U * dd.abs(), "td_out " + what)
            e_g = (2 * e_dd * w.double() + 4 * U * (2 * dd * w.double()).abs()) / B
        else:
            u = tgt.unsqueeze(-1) - q_s_a.unsqueeze(1)
            e_u = e_y.unsqueeze(-1) + U * u.abs()
            hub = torch.where(u.abs() < 1.0, 0.5 * u * u, u.abs() - 0.5)
            term_err = torch.maximum(u.abs(), torch.ones_like(u)) * e_u + 4 * U * hub
            per_err = (term_err.sum(1) + Q * U * hub.sum(1)).sum(1) / (Q * Q)
            close(td, tdref, per_err + U * tdref, "td_out " + what)
            dh = torch.where(u.abs() < 1.0, u, u.sign())
            # dh moves by e_u, and where u changes sign the weight jumps by 1 at |dh| = |u| <= e_u: 2 e_u per term
            e_gi = (2 * e_u + 2 * U * dh.abs()).sum(1) + Q * U * dh.abs().sum(1)   # + the fp32 sum over j
            e_g = (e_gi * w.double()[:, None] / (B * Q * Q) + 0) * (1 + 8 * U)
        close(info[0], loss, (per_err * w.double()).mean() + 2 * U * abs(loss), "loss " + what)
        close(info[1], q_s_a.mean(), U * q_s_a.abs().mean(), "mean q_s_a " + what)
        close(info[2], r.double().mean(), U * r.double().abs().mean(), "mean reward " + what)
        gsel = g.view(B, A, Q)[torch.arange(B, device="cuda"), acts.long()]
        grsel = gref.view(B, A, Q)[torch.arange(B, device="cuda"), acts.long()]
        close(gsel, grsel, (e_g if not mse else e_g[:, None]) + 4 * U * grsel.abs(), "grad " + what)
        mask = torch.ones(B, A, Q, dtype=torch.bool, device="cuda")
        mask[torch.arange(B, device="cuda"), acts.long()] = False
        assert (g.view(B, A, Q)[mask] == 0).all(), "grad outside the taken action must be zero"


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 5, 1023, 4097, 70001])
def test_td3_smooth_action_is_exact(n):
    """a' = clamp(a + clamp(sigma eps, +-c), +-1) with supplied eps: the same fp32 operations in torch give the same
    bits, and the result is within U of the oracle's float64 value.  The Philox path keeps to [-1, 1] and its guards."""
    gen(n)
    act, eps = torch.tanh(randn(n)), 2 * randn(n)

    def run(eps_t):
        out = Guarded(n)
        call("trl_td3_smooth_action", act.data_ptr(), ptr(eps_t), 0.2, 0.5, 77, None, n, out.t.data_ptr(), stream())
        return [out.check("a'")]
    out = twice(lambda: run(eps))[0]
    exact(out, torch.clamp(act + torch.clamp(F32(0.2) * eps, -0.5, 0.5), -1, 1), "smoothed action n=%d" % n)
    ref = rn.td3_smooth_action(act.double().cpu().numpy(), F32(0.2) * eps.double().cpu().numpy(), 0.5)
    close(out, torch.from_numpy(ref), 2 * U, "oracle n=%d" % n)
    ph = twice(lambda: run(None))[0]
    assert ph.abs().max().item() <= 1.0 and ((ph - act).abs() <= 0.5 + 2 * U).all()


# ========================================================================================================== D. optim.cu
def seg_table(sizes):
    b = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return (ctypes.c_int64 * len(b))(*b.tolist()), b


OPT_CASES = [
    # sizes, active mask, max_norm per segment (<= 0: no clip), eps per segment, grad_scale, zero_grad, planes
    ([200003], 0b1, [0.5], [1e-5], 1.0, 1, False),
    ([1, 0, 140001], 0b111, [-1.0, 0.5, 1e9], [1e-8, 1e-5, 1e-3], 0.5, 0, True),
    ([5, 257, 1023, 0, 4099, 65537, 3, 70001], 0b10110101, [0.5, 0.0, 2.0, 1.0, 0.1, 1.0, -1.0, 0.3],
     [1e-8, 1e-5, 1e-8, 1e-5, 1e-3, 1e-8, 1e-5, 1e-8], 1.0, 1, True),
    ([3, 1021], 0b10, [0.5, 0.5], [1e-5, 1e-5], 0.5, 1, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(OPT_CASES)))
def test_grad_sumsq_and_adam_step_match_fp64(case):
    """trl_grad_sumsq then trl_adam_step for 5 steps against float64 clip_grad_norm_ + torch.optim.Adam restated, each
    step from the kernel's own state (so every step is checked at one step's error).  Inactive segments must keep
    every bit (weights, gradient, moments, planes, step count)."""
    sizes, mask, max_norm, eps, gscale, zero_grad, planes = OPT_CASES[case]
    nseg = len(sizes)
    tbl, b = seg_table(sizes)
    n = int(b[-1])
    gen(case)
    w, m, v = randn(n), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    hi, lo = (torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")) if planes else (None, None)
    steps = torch.zeros(nseg, dtype=torch.int32, device="cuda")
    lr = torch.tensor([F32(1e-3 * (k + 1)) for k in range(nseg)], device="cuda")
    b1, b2 = F32(0.9), F32(0.999)
    mn = (ctypes.c_float * nseg)(*max_norm)
    ep = (ctypes.c_float * nseg)(*eps)
    active = [(mask >> k) & 1 == 1 for k in range(nseg)]
    seg_of = torch.from_numpy(np.repeat(np.arange(nseg), sizes)).cuda()
    act_el = torch.tensor(active, device="cuda")[seg_of] if n else torch.zeros(0, dtype=torch.bool)
    for t in range(1, 6):
        g = randn(n) * (10.0 if t % 2 else 0.01)               # alternately clipped and not
        if t == 3:
            g[: min(n, 7)] = 0.0
        g0, w0, m0, v0, s0 = g.clone(), w.clone(), m.clone(), v.clone(), steps.clone()
        h0, l0 = (hi.clone(), lo.clone()) if planes else (None, None)

        def run_sumsq(scratch, ticket):
            steps.copy_(s0)
            out = Guarded64(3 * nseg)
            call("trl_grad_sumsq", g.data_ptr(), tbl, nseg, mask, out.t.data_ptr(), steps.data_ptr(), b1, b2, scratch,
                 ticket, stream())
            return [out.check("sumsq3"), steps]
        sq, steps_k = poisoned(lib().trl_grad_sumsq_blocks(nseg), run_sumsq)
        steps.copy_(steps_k)
        g64 = g.double()
        for k in range(nseg):
            if not active[k]:
                assert steps[k].item() == s0[k].item(), "inactive segment %d: step count moved" % k
                continue
            gk = g64[b[k]:b[k + 1]].cpu().numpy()
            ref = math.fsum(gk * gk)
            # non-negative terms: error <= (longest addition chain) 2^-53 sum; the chain is ceil(n_k / 4096) strided
            # adds per thread, 5 + 3 shuffle levels and 16 partials (< 1e-12 relative at these sizes)
            depth = -(-len(gk) // 4096) + 24
            assert abs(sq[k].item() - ref) <= depth * E53 * ref, (k, sq[k].item(), ref)
            assert depth * E53 < 1e-12
            tk = steps[k].item()
            assert tk == t, "step count"
            # 1 - beta^t by repeated squaring: a few ulp on beta^t, absolute
            close(sq[nseg + 2 * k], 1 - b1 ** tk, 4 * tk * E53, "bias correction 1")
            close(sq[nseg + 2 * k + 1], math.sqrt(1 - b2 ** tk), 4 * tk * E53 / math.sqrt(1 - b2 ** tk) + E53,
                  "bias correction 2")

        def run_adam():
            g.copy_(g0); w.copy_(w0); m.copy_(m0); v.copy_(v0)
            if planes:
                hi.copy_(h0); lo.copy_(l0)
            call("trl_adam_step", w.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), tbl, nseg, mask,
                 sq.data_ptr(), lr.data_ptr(), mn, ep, b1, b2, gscale, zero_grad, ptr(hi), ptr(lo), stream())
            return [w, g, m, v] + ([hi, lo] if planes else [])
        outs = twice(run_adam)
        for o, cur in zip(outs, [w, g, m, v] + ([hi, lo] if planes else [])):
            cur.copy_(o)
        # float64 restatement of clip_grad_norm_ (per segment) + Adam from the kernel's state before this step
        G = g0.double() * gscale
        norm = torch.zeros(n, dtype=torch.float64, device="cuda")
        coef = torch.ones(n, dtype=torch.float64, device="cuda")
        for k in range(nseg):
            nk = math.sqrt(sq[k].item()) * abs(gscale) if active[k] else 0.0
            norm[b[k]:b[k + 1]] = nk
            if active[k] and max_norm[k] > 0:
                coef[b[k]:b[k + 1]] = min(1.0, F32(max_norm[k]) / (nk + F32(1e-6)))
        Gc = G * coef
        M = b1 * m0.double() + (1 - b1) * Gc
        V = b2 * v0.double() + (1 - b2) * Gc * Gc
        tt = steps[seg_of].double() if n else torch.zeros(0)
        bc1, bc2s = 1 - b1 ** tt, torch.sqrt(1 - b2 ** tt)
        epsv = torch.tensor([F32(e) for e in eps], dtype=torch.float64, device="cuda")[seg_of]
        den = V.sqrt() / bc2s + epsv
        upd = lr.double()[seg_of] / bc1 * M / den
        W = w0.double() - upd
        # g * scale * coef: coef from the norm's cast, the sum and the division (4U), the products (2U)
        e_G = 6 * U * Gc.abs()
        e_M = 2 * U * (b1 * m0.double().abs() + (1 - b1) * Gc.abs()) + (1 - b1) * e_G
        e_V = 3 * U * (b2 * v0.double() + (1 - b2) * Gc * Gc) + (1 - b2) * 2 * Gc.abs() * e_G
        e_sqrt = torch.minimum(e_V / (2 * V.sqrt()).clamp_min(1e-300), e_V.sqrt()) + U * V.sqrt()
        e_den = e_sqrt / bc2s + 3 * U * den                 # the division, bc2's cast, + eps
        e_upd = lr.double()[seg_of] / bc1 * (e_M / den + M.abs() * e_den / (den * den)) + 4 * U * upd.abs()
        A = act_el
        close(m[A], M[A], 2 * e_M[A], "exp_avg step %d" % t)
        close(v[A], V[A], 2 * e_V[A], "exp_avg_sq step %d" % t)
        close(w[A], W[A], 2 * e_upd[A] + U * W[A].abs(), "weights step %d" % t)
        if zero_grad:
            assert (g[A] == 0).all(), "zero_grad: active gradient not zeroed"
        else:
            assert same_bits(g[A], g0[A]), "zero_grad = 0: gradient changed"
        for name, now, before in [("weights", w, w0), ("grad", g, g0), ("exp_avg", m, m0), ("exp_avg_sq", v, v0)] + \
                ([("hi", hi, h0), ("lo", lo, l0)] if planes else []):
            assert same_bits(now[~A], before[~A]), "inactive segment: %s changed" % name
        if planes:
            ref_hi = torch.from_numpy(rna_tf32_bits(w[A].cpu().numpy()).view(np.float32)).cuda()
            assert same_bits(hi[A], ref_hi), "hi plane is not rna(w)"
            assert torch.equal(lo[A].double(), w[A].double() - ref_hi.double()), "lo plane is not w - hi"


# ====================================================================================== E. gather.cu statistics
def stats64(x):
    x = x.double()
    return [x.mean().item(), x.std().item() if x.numel() > 1 else float("nan"), x.max().item(), x.min().item()]


def check_stats(st, x, depth, what):
    """mean, unbiased std, max, min from fp64 raw moments: the sums err by depth 2^-53 sum|x| (sum of squares alike),
    the one-pass variance turns that into an error of 2 depth 2^-53 sum x^2 / (n - 1) on var; then the casts (U)"""
    mu, sd, mx, mn = stats64(x)
    n = x.numel()
    xd = x.double()
    close(st[0], mu, U * abs(mu) + depth * E53 * xd.abs().sum().item() / n, "mean " + what)
    if n == 1:
        assert math.isnan(st[1].item()), "std of one value is nan, as torch.std (pinned)"
    else:
        dv = 4 * depth * E53 * (xd * xd).sum().item() / (n - 1)
        close(st[1], sd, U * sd + min(dv / max(2 * sd, 1e-300), math.sqrt(dv)), "std " + what)
    exact(st[2], torch.tensor([mx]).float(), "max " + what)
    exact(st[3], torch.tensor([mn]).float(), "min " + what)


def vec_moments(x):
    out = Guarded64(4)
    call("trl_vec_moments", x.data_ptr(), x.numel(), out.t.data_ptr(), stream())
    return out.check("moments")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 1023, 1024, 1025, (1 << 20) + 3])
def test_vec_stats_and_moments_match_fp64(n):
    gen(n)
    depth = -(-n // 1024) + 10          # strided per-thread adds, then two shuffle trees
    for integer in (True, False):
        x = ints(-50, 50, n) if integer else 3.0 + 2.0 * randn(n)

        def run():
            st = Guarded(4)
            call("trl_vec_stats", x.data_ptr(), n, st.t.data_ptr(), stream())
            return [st.check("stats"), vec_moments(x)]
        st, mo = twice(run)
        xd = x.double()
        if integer:     # every partial sum is an integer below 2^53: exact
            exact(mo, torch.tensor([xd.sum().item(), (xd * xd).sum().item(), xd.max().item(), -xd.min().item()],
                                   dtype=torch.float64), "integer moments n=%d" % n)
        else:
            close(mo[0], xd.sum(), mean_sum_bound(x, depth), "sum")
            close(mo[1], (xd * xd).sum(), depth * E53 * (xd * xd).sum().item(), "sum of squares")
            exact(mo[2:], torch.tensor([xd.max().item(), -xd.min().item()]), "max, -min")
        check_stats(st, x, depth, "vec_stats n=%d integer=%d" % (n, integer))
        sf = Guarded(4)
        call("trl_vec_stats_from_moments", mo.data_ptr(), 1, float(n), sf.t.data_ptr(), stream())
        check_stats(sf.check(), x, depth, "vec_stats_from_moments n=%d" % n)


@pytest.mark.gpu
def test_vec_stats_from_three_ranks():
    gen(5)
    xs = [randn(n) * s + o for n, s, o in ((1000, 1.0, 0.0), (4097, 3.0, 2.0), (1, 1.0, -9.0))]
    g = torch.stack([vec_moments(x) for x in xs])
    st = Guarded(4)
    call("trl_vec_stats_from_moments", g.data_ptr(), 3, float(sum(x.numel() for x in xs)), st.t.data_ptr(), stream())
    check_stats(st.check(), torch.cat(xs), 20, "three ranks")


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [1, 7])
@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("row_elems", [1, 1000, 2049])
def test_row_group_moments_and_group_stats_match_fp64(groups, b, row_elems):
    """raw moments of the rows idx[u b .. (u+1) b) (a permutation) of x, for world 1 and for three different tables
    stacked (3, groups, 4), then mean / unbiased std / max / min per group"""
    gen(groups * 10 + b + row_elems)
    rows = groups * b + 5
    W = 3
    xs = [ints(-20, 20, rows, row_elems) if k == 0 else randn(rows, row_elems) * (k + 1) + k for k in range(W)]
    idx = torch.randperm(rows, device="cuda")[: groups * b].contiguous()
    tables = []
    for k, x in enumerate(xs):
        def run():
            out = Guarded64(groups, 4)
            call("trl_row_group_moments", x.data_ptr(), idx.data_ptr(), groups, b, row_elems, out.t.data_ptr(),
                 stream())
            return [out.check("moments")]
        mo = twice(run)[0]
        sel = x[idx].view(groups, b * row_elems).double()
        if k == 0:      # integers: exact
            exact(mo, torch.stack([sel.sum(1), (sel * sel).sum(1), sel.max(1).values, -sel.min(1).values], 1),
                  "integer group moments")
        depth = b * -(-row_elems // 1024) + 10
        for u in range(groups):
            close(mo[u, 0], sel[u].sum(), depth * E53 * sel[u].abs().sum().item(), "group sum")
            close(mo[u, 1], (sel[u] ** 2).sum(), depth * E53 * (sel[u] ** 2).sum().item(), "group sum of squares")
        tables.append(mo)
        st = Guarded(groups, 4)
        call("trl_group_stats_from_moments", mo.data_ptr(), 1, groups, float(b * row_elems), st.t.data_ptr(), stream())
        st = st.check()
        for u in range(groups):
            check_stats(st[u], sel[u], depth, "world 1 group %d" % u)
    g = torch.stack(tables).contiguous()                      # (W, groups, 4)
    st = Guarded(groups, 4)
    call("trl_group_stats_from_moments", g.data_ptr(), W, groups, float(W * b * row_elems), st.t.data_ptr(), stream())
    st = st.check()
    for u in range(groups):
        allx = torch.cat([x[idx].view(groups, -1)[u] for x in xs])
        check_stats(st[u], allx, b * -(-row_elems // 1024) + 12, "world 3 group %d" % u)


# ====================================================================================== F. obs_norm.cu, collect.cu
@pytest.mark.gpu
@pytest.mark.parametrize("o", [1, 17, 376, 1024])
@pytest.mark.parametrize("N", [1, 3, 4096])
def test_obs_norm_matches_running_norm(o, N):
    """moments -> merge (Chan, starting from count 1e-4) -> filter, over four batches, against ref_numpy.RunningNorm.
    Column 0 has a large offset (1000) and a small spread (0.01).  The batch variance is the one-pass q/n - mean^2 in
    fp64: with the sums off by depth 2^-53 of their magnitudes it errs by about (2 depth + 4) 2^-53 q/n, i.e. relative
    (2 depth + 4) 2^-53 (1 + mean^2 / var): 1e-5 for column 0 at N = 4096 -- acceptable for a normaliser, which only
    divides by sqrt(var) + 1e-4."""
    gen(o * 7 + N)
    mean = torch.zeros(o, dtype=torch.float64, device="cuda")
    var = torch.ones(o, dtype=torch.float64, device="cuda")
    count = torch.tensor([1e-4], dtype=torch.float64, device="cuda")
    ref = rn.RunningNorm(o)
    depth = -(-N // 256) + 10
    e_mean = np.zeros(o)
    e_var = np.zeros(o)
    for step in range(4):
        x = randn(N, o) * (1 + step)
        x[:, 0] = 1000.0 + 0.01 * randn(N)

        def run():
            sums = Guarded64(2 * o)
            call("trl_obs_norm_moments", x.data_ptr(), N, o, sums.t.data_ptr(), stream())
            return [sums.check("sums")]
        sums = twice(run)[0]
        xd = x.double()
        close(sums[:o], xd.sum(0), depth * E53 * xd.abs().sum(0), "column sums")
        close(sums[o:], (xd * xd).sum(0), depth * E53 * (xd * xd).sum(0), "column sums of squares")
        call("trl_obs_norm_merge", sums.data_ptr(), float(N), o, mean.data_ptr(), var.data_ptr(), count.data_ptr(),
             stream())
        ref.update(xd.cpu().numpy())
        q_n = (xd * xd).mean(0).cpu().numpy()
        e_mean += depth * E53 * np.abs(xd.cpu().numpy()).mean(0) + 4 * E53 * np.abs(ref.mean)
        e_var += (2 * depth + 8) * E53 * (q_n + ref.var)
        assert count.item() == ref.count, "count"
        close(mean, torch.from_numpy(ref.mean).cuda(), torch.from_numpy(e_mean).cuda(), "mean after merge %d" % step)
        close(var, torch.from_numpy(ref.var).cuda(), torch.from_numpy(e_var).cuda(), "var after merge %d" % step)
    # filter: fp64 on the kernel's own state, then the cast; far values hit the clip exactly
    raw = torch.cat([randn(N, o) * 2, torch.full((2, o), 1e6, device="cuda"), torch.full((2, o), -1e6,
                                                                                           device="cuda")])
    raw[-4, :] *= -1.0
    for clip in (10.0, 2.5):
        def run():
            out = Guarded(N + 4, o)
            call("trl_obs_norm_filt", raw.data_ptr(), mean.data_ptr(), var.data_ptr(), N + 4, o, clip,
                 out.t.data_ptr(), stream())
            return [out.check("filtered")]
        y = twice(run)[0]
        yr = ((raw.double() - mean) / (var.sqrt() + 1e-4)).clamp(-clip, clip)
        close(y, yr, U * yr.abs() + 1e-12, "filt clip=%g" % clip)
        assert (y[-2:] == -clip).all() and (y[-4:-2].abs() == clip).all(), "values past the clip sit at +-clip"
        assert (y.abs() <= clip).all()


class _TanhAtStored(torch.autograd.Function):
    """tanh whose value is the stored fp32 action y: backward is torch's tanh backward g (1 - y^2) at that y.  Where
    the fp32 action saturates to +-1 (|z| > 9) this is the derivative of what the forward computed (zero through the
    action), as in the float32 reference; the exact float64 tanh would still pass ~1e-7 there."""

    @staticmethod
    def forward(ctx, z, y):
        ctx.save_for_backward(y)
        return y.clone()

    @staticmethod
    def backward(ctx, g):
        y, = ctx.saved_tensors
        return g * (1 - y * y), None


@pytest.mark.gpu
@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("grads", ["both", "action_only", "logp_only"])
@pytest.mark.parametrize("tanh", [True, False])
def test_tanh_gaussian_sample_bwd_matches_fp64(shared, grads, tanh):
    """d(action, log_prob)/d(mean, log_std) of z = mu + exp(ls) eps, a = tanh(z), TanhNormal.log_prob, by float64
    autograd; rows with |z| > 9 (saturated fp32 actions) included."""
    gen(int(shared) + 2 * len(grads) + 7 * tanh)
    M, a = 4099, 6
    mu = randn(M, a)
    ls = -1.0 + 0.5 * randn(*((a,) if shared else (M, a)))
    e = randn(M, a)
    mu[::50] = 12.0 * mu[::50].sign()                           # |z| > 9: the fp32 action is exactly +-1
    z32 = mu + ls.exp() * e
    act = torch.tanh(z32) if tanh else z32
    if tanh:
        assert (act[::50].abs() == 1).all()
    g_a = randn(M, a) if grads != "logp_only" else None
    g_l = randn(M) if grads != "action_only" else None

    def run():
        gm, gl = Guarded(M, a), Guarded(M, a)
        call("trl_tanh_gaussian_sample_bwd", act.data_ptr(), e.data_ptr(), ls.data_ptr(), 0 if shared else a,
             ptr(g_a), ptr(g_l), M, a, int(tanh), gm.t.data_ptr(), gl.t.data_ptr(), stream())
        return [gm.check("g_mean"), gl.check("g_log_std")]
    gm, gl = twice(run)
    m64 = mu.double().requires_grad_()
    l64 = ls.double().requires_grad_()
    lsb = l64.expand(M, a)
    z = m64 + lsb.exp() * e.double()
    y = act.double()
    if tanh:
        assert ((y - torch.tanh(z32.double())).abs() <= 2 * U).all(), "stored action is tanh(z) to 2 ulp"
        av = _TanhAtStored.apply(z, y)
    else:
        av = z
    # Normal(mu, sd).log_prob(z) - log(1 - a^2 + 1e-6), summed over the action dims
    lp = (-((z - m64) ** 2) / (2 * lsb.exp() ** 2) - lsb - HALF_LOG_2PI)
    if tanh:
        lp = lp - torch.log(1 - av * av + F32(1e-6))
    lp = lp.sum(1)
    obj = (av * g_a.double()).sum() if g_a is not None else 0
    if g_l is not None:
        obj = obj + (lp * g_l.double()).sum()
    rg_m, rg_ls_raw = torch.autograd.grad(obj, [m64, l64])
    # per-row log-std gradient (the caller reduces a shared log-std): d obj / d ls_j of row m
    sd, ed = lsb.detach().exp(), e.double()
    ga = g_a.double() if g_a is not None else torch.zeros(M, a, dtype=torch.float64, device="cuda")
    glr = g_l.double()[:, None] if g_l is not None else torch.zeros(M, 1, dtype=torch.float64, device="cuda")
    # first-order bound of the fp32 evaluation: dadz = 1 - a^2 (U a^2 + U dadz), w = 1 - a^2 + 1e-6 (U a^2 + 2U w),
    # dldz = 2 a dadz / w (three more roundings), gz = ga dadz + gl dldz (two), g_ls = gz sd eps - gl (expf 2 ulp,
    # two products, one difference); x2 for second-order terms
    if tanh:
        dadz = 1 - y * y
        w = dadz + F32(1e-6)
        dldz = 2 * y * dadz / w
        e_dadz = U * (y * y + dadz)
        e_w = U * (y * y + 2 * w)
        e_dldz = 2 * y.abs() * (e_dadz / w + dadz * e_w / (w * w)) + 3 * U * dldz.abs()
    else:
        dadz, dldz = torch.ones_like(y), torch.zeros_like(y)
        e_dadz = e_dldz = torch.zeros_like(y)
    gz = ga * dadz + glr * dldz
    e_gz = ga.abs() * e_dadz + glr.abs() * e_dldz + 2 * U * (ga * dadz).abs() + 2 * U * (glr * dldz).abs()
    close(gm, rg_m, 2 * e_gz + U * rg_m.abs(), "g_mean shared=%d %s tanh=%d" % (shared, grads, tanh))
    gls_row = gz * sd * ed - glr
    e_gls = 2 * ((sd * ed).abs() * e_gz + 4 * U * (gz * sd * ed).abs()) + U * gls_row.abs()
    close(gl, gls_row, e_gls, "g_log_std shared=%d %s tanh=%d" % (shared, grads, tanh))
    close(gl.double().sum(0) if shared else gl, rg_ls_raw, (e_gls.sum(0) + 1e-12 * gls_row.abs().sum(0)) if shared
          else e_gls, "g_log_std vs autograd")


# ============================================================================= G. argument validation (no GPU needed)
def _p(native_lib):
    buf = (ctypes.c_float * 256)()
    p = _host_ptr(buf)
    return buf, p + (-p % 16)


def test_loss_kernels_reject_bad_sizes(native_lib):
    _buf, p = _p(native_lib)
    L = native_lib
    for a in (0, 33):
        _rejects(L, L.trl_ppo_actor_loss(p, p, 0, p, p, p, None, None, 8, a, 1, 0.2, 0.0, 1.0, -1.0, p, p, None, p, p, p,
                                         None), "bad sizes")
        _rejects(L, L.trl_ppo_categorical_actor_loss(p, p, p, p, None, None, 8, a, 0.2, 0.0, p, None, p, p, p, None),
                 "bad sizes")
        _rejects(L, L.trl_categorical_sample(p, p, 0, None, 8, a, p, None, None, None), "bad sizes")
        _rejects(L, L.trl_categorical_log_prob(p, p, 8, a, p, None), "bad sizes")
    _rejects(L, L.trl_gaussian_log_prob(p, p, 0, p, 8, 0, 1, p, None), "bad sizes")
    for stride in (1, 5, 7):
        _rejects(L, L.trl_ppo_actor_loss(p, p, stride, p, p, p, None, None, 8, 6, 1, 0.2, 0.0, 1.0, -1.0, p, p, None, p,
                                         p, p, None), "ls_stride")
        _rejects(L, L.trl_gaussian_log_prob(p, p, stride, p, 8, 6, 1, p, None), "ls_stride")
        _rejects(L, L.trl_tanh_gaussian_sample(p, p, stride, p, 1.0, 0, None, 8, 6, 1, p, None, None, None, None, None),
                 "ls_stride")
        _rejects(L, L.trl_tanh_gaussian_sample_bwd(p, p, p, stride, p, p, 8, 6, 1, p, p, None), "ls_stride")
    # B = 0 for every loss kernel
    _rejects(L, L.trl_ppo_actor_loss(p, p, 0, p, p, p, None, None, 0, 6, 1, 0.2, 0.0, 1.0, -1.0, p, p, None, p, p, p,
                                     None), "bad sizes")
    _rejects(L, L.trl_ppo_critic_loss(p, p, p, 0, 1, 0.2, p, p, p, p, None), "empty batch")
    _rejects(L, L.trl_ppo_categorical_actor_loss(p, p, p, p, None, None, 0, 6, 0.2, 0.0, p, None, p, p, p, None),
             "bad sizes")
    _rejects(L, L.trl_td_target(p, p, p, p, p, p, 0.2, 0.99, 0, p, p, p, p, None), "empty batch")
    _rejects(L, L.trl_sac_alpha_step(p, -6.0, p, p, 3e-4, 0.9, 0.999, 1e-8, 0, p, p, p, None), "empty batch")
    _rejects(L, L.trl_sac_policy_loss(p, p, p, p, 0.2, 0, p, p, p, p, p, p, None), "empty batch")
    _rejects(L, L.trl_twin_mse_loss(p, p, p, 0, p, p, p, p, p, None), "empty batch")
    _rejects(L, L.trl_qr_dqn_loss(p, p, p, p, p, None, 0, 6, 5, 0.99, 1.0, 0, p, None, p, p, p, None), "bad sizes")
    # the DQN form is Q = 1 only; q2 needs g2
    _rejects(L, L.trl_qr_dqn_loss(p, p, p, p, p, None, 8, 6, 5, 0.99, 1.0, 1, p, None, p, p, p, None),
             "n_quantiles == 1")
    _rejects(L, L.trl_twin_mse_loss(p, p, p, 8, p, None, p, p, p, None), "without g2")


def test_optimizer_and_normaliser_reject_bad_tables(native_lib):
    _buf, p = _p(native_lib)
    L = native_lib
    mn = (ctypes.c_float * 9)(*[1.0] * 9)
    for nseg in (0, 9):
        tbl = (ctypes.c_int64 * 10)(*range(10))
        _rejects(L, L.trl_grad_sumsq(p, tbl, nseg, 1, p, p, 0.9, 0.999, p, p, None), "bad segment table")
        _rejects(L, L.trl_adam_step(p, p, p, p, tbl, nseg, 1, p, p, mn, mn, 0.9, 0.999, 1.0, 1, None, None, None),
                 "bad segment table")
    dec = (ctypes.c_int64 * 4)(0, 10, 5, 20)
    _rejects(L, L.trl_grad_sumsq(p, dec, 3, 7, p, p, 0.9, 0.999, p, p, None), "bad segment table")
    _rejects(L, L.trl_adam_step(p, p, p, p, dec, 3, 7, p, p, mn, mn, 0.9, 0.999, 1.0, 1, None, None, None),
             "bad segment table")
    _rejects(L, L.trl_obs_norm_merge(p, 4.0, 1025, p, p, p, None), "1..1024")
    _rejects(L, L.trl_obs_norm_merge(p, 4.0, 0, p, p, p, None), "1..1024")
