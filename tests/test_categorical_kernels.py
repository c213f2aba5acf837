"""Categorical distribution kernels (csrc/categorical.cu) against torch's Categorical(softmax(x)) -- the recorded
reference data of oracle/make_golden_categorical.py and torch autograd of the same expressions -- and against a NumPy
restatement of inverse-CDF sampling.  Tolerance 2e-4 throughout; saturated rows (logit gaps above 16, where the
probability clamp of probs_to_logits is active) are part of every comparison."""
import os

import numpy as np
import pytest

from oracle import make_golden_categorical as gold

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "categorical_reference.npz")


def _logits(M, A, seed, sat_every=3):
    rs = np.random.RandomState(seed)
    x = rs.randn(M, A).astype(np.float32) * 2.0
    sat = np.arange(M) % sat_every == 0
    x[sat] = (rs.randn(int(sat.sum()), A) * 12.0).astype(np.float32)
    x[sat, rs.randint(0, A, int(sat.sum()))] += 20.0
    return x


def _torch_ref(x, acts, old_logp, advs, adv_stats, clip, ent_coef):
    """The reference's actor loss (ppo.py:41-68 with old_logp, a2c.py:62-70 without) in torch autograd on the CPU, in
    float32 like the reference (the probability clamp's eps is float32's)."""
    import torch
    xt = torch.tensor(x, dtype=torch.float32, requires_grad=True)
    dis = torch.distributions.Categorical(torch.softmax(xt, dim=-1))
    lp = dis.log_prob(torch.as_tensor(acts, dtype=torch.int64))
    ent = dis.entropy()
    adv = (torch.as_tensor(advs, dtype=torch.float32) - adv_stats[0]) / (adv_stats[1] + 1e-5)
    if old_logp is None:
        loss = (-lp * adv).mean() - ent_coef * ent.mean()
        ratio = torch.ones_like(lp)
    else:
        ratio = torch.exp(lp - torch.as_tensor(old_logp, dtype=torch.float32))
        s1 = ratio * adv
        s2 = torch.clamp(ratio, 1 - clip, 1 + clip) * adv
        loss = -torch.mean(torch.min(s2, s1)) - ent_coef * ent.mean()
    g, = torch.autograd.grad(loss, xt)
    lpn = lp.detach().numpy()
    return dict(loss=float(loss.detach()), g=g.numpy(), lp=lpn, ent=float(ent.detach().mean()),
                ratio=ratio.detach().numpy())


def test_log_prob_entropy_and_gradients_match_reference():
    import torch
    from torchrl_b200 import ops
    r = gold.load(GOLDEN)["dist"]["out"]
    x, acts, w1, w2 = gold.dist_inputs()
    M, A = x.shape
    p = torch.softmax(torch.tensor(x, dtype=torch.float64), -1).numpy()
    assert (p.min(axis=1) < np.finfo(np.float32).eps).sum() > M // 4, "the saturated rows must engage the clamp"
    xd = torch.tensor(x, device="cuda")
    ad = torch.tensor(acts, dtype=torch.float32, device="cuda")
    lp = ops.categorical_log_prob(xd, ad).cpu().numpy()
    np.testing.assert_allclose(lp, r["log_prob"], atol=2e-4, rtol=0)
    # gradient of sum(w1 * logp): the loss kernel with A2C mode, unit advantages scaled by -w1 * B, no entropy
    B = M
    scratch = ops.LossScratch(B, A, "cuda", categorical=True)
    stats = torch.tensor([0.0, 1.0 - 1e-5, 0.0, 0.0], device="cuda")
    g, info = ops.ppo_categorical_actor_loss(xd, ad, None, torch.tensor(-w1 * B, device="cuda"), stats, 0.0, 0.0,
                                             scratch)
    np.testing.assert_allclose(g.cpu().numpy(), r["grad_log_prob"], atol=2e-4, rtol=0)
    np.testing.assert_allclose(info[11].item(), r["entropy"].mean(), atol=2e-4)
    # gradient of sum(w2 * ent) per row is not a loss the kernel computes (its entropy term is a batch mean); check the
    # entropy gradient through ent_coef with zero advantages: d(-c * mean(ent)) = -c/B * d ent
    g, _ = ops.ppo_categorical_actor_loss(xd, ad, None, torch.zeros(B, device="cuda"), stats, 0.0, 1.0, scratch)
    ref = _torch_ref(x, acts, None, np.zeros(B), (0.0, 1.0 - 1e-5), 0.0, 1.0)
    np.testing.assert_allclose(g.cpu().numpy(), ref["g"], atol=2e-4 / B, rtol=2e-4)
    # the recorded weighted entropy gradient equals the unweighted one row by row times w2
    xt = torch.tensor(x, requires_grad=True)
    ent = torch.distributions.Categorical(torch.softmax(xt, -1)).entropy()
    g2, = torch.autograd.grad((ent * torch.as_tensor(w2)).sum(), xt)
    np.testing.assert_allclose(g2.numpy(), r["grad_entropy"], atol=1e-5)
    gk = -g.cpu().numpy() * B * w2[:, None]
    np.testing.assert_allclose(gk, r["grad_entropy"], atol=2e-4)


@pytest.mark.parametrize("mode", ["ppo", "a2c"])
@pytest.mark.parametrize("B,A", [(1000, 6), (300, 18), (257, 1), (64, 32)])
def test_actor_loss_matches_torch_autograd(mode, B, A):
    import torch
    from torchrl_b200 import ops
    rs = np.random.RandomState(B + A)
    x = _logits(B, A, B * A)
    acts = rs.randint(0, A, B)
    advs = rs.randn(B).astype(np.float32)
    U = 3
    table = np.stack([rs.randn(U) * 0.3, 0.5 + rs.rand(U), np.zeros(U), np.zeros(U)], 1).astype(np.float32)
    clip, ent_coef = 0.2, 0.01
    with torch.no_grad():
        lp_now = torch.distributions.Categorical(torch.softmax(torch.tensor(x), -1)).log_prob(
            torch.as_tensor(acts)).numpy()
    old = None
    if mode == "ppo":
        old = (lp_now + rs.randn(B) * 0.3).astype(np.float32)
        old[::7] = lp_now[::7]                            # ratio 1: both surrogate terms equal (torch's tie rule)
    scratch = ops.LossScratch(B, A, "cuda", categorical=True)
    xd = torch.tensor(x, device="cuda")
    ad = torch.tensor(acts, dtype=torch.float32, device="cuda")
    advd = torch.tensor(advs, device="cuda")
    od = None if old is None else torch.tensor(old, device="cuda")
    tbl = torch.tensor(table, device="cuda")
    for u in range(U):
        pos = torch.tensor([u], dtype=torch.int32, device="cuda")
        outs = []
        for _ in range(2):
            lpo = torch.empty(B, device="cuda")
            g, info = ops.ppo_categorical_actor_loss(xd, ad, od, advd, tbl, clip, ent_coef, scratch, stats_pos=pos,
                                                     logp_out=lpo)
            outs.append((g.clone(), info.clone(), lpo))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "not deterministic"
        g, info, lpo = outs[0]
        ref = _torch_ref(x, acts, old, advs,
                         (float(table[u, 0]), float(table[u, 1])), clip, ent_coef)
        info = info.cpu().numpy()
        np.testing.assert_allclose(lpo.cpu().numpy(), ref["lp"], atol=2e-4)
        np.testing.assert_allclose(info[0], ref["loss"], atol=2e-4, rtol=2e-4)
        np.testing.assert_allclose(info[1], ref["lp"].mean(), atol=2e-4)
        np.testing.assert_allclose(info[2], ref["lp"].astype(np.float64).std(ddof=1), atol=2e-4, rtol=1e-3)
        np.testing.assert_allclose(info[3:5], [ref["lp"].max(), ref["lp"].min()], atol=2e-4)
        np.testing.assert_allclose(info[5:7], [ref["ratio"].max(), ref["ratio"].min()], atol=2e-4, rtol=2e-4)
        np.testing.assert_allclose(info[11], ref["ent"], atol=2e-4)
        # dL/dlogits is O(1/B): compare at the scale of the batch-summed loss
        np.testing.assert_allclose(g.cpu().numpy() * B, ref["g"] * B, atol=2e-4, rtol=2e-3)


def _np_inverse_cdf(x, u):
    z = x.astype(np.float64)
    p = np.exp(z - z.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    c = np.cumsum(p, 1)
    a = (u[:, None] >= c).sum(1)
    near = (np.abs(c - u[:, None]) < 1e-6).any(1)
    return np.minimum(a, x.shape[1] - 1), near


def test_sampling_with_supplied_uniforms_is_the_inverse_cdf():
    import torch
    from torchrl_b200 import ops
    M, A = 20000, 18
    x = _logits(M, A, 5)
    rs = np.random.RandomState(6)
    u = rs.rand(M).astype(np.float32)
    want, near = _np_inverse_cdf(x, u.astype(np.float64))
    act, lp = ops.categorical_sample(torch.tensor(x, device="cuda"), u=torch.tensor(u, device="cuda"),
                                     want_log_prob=True)
    got = act.cpu().numpy()
    assert np.all(got == np.round(got)) and got.min() >= 0 and got.max() < A
    ok = ~near
    assert near.sum() < M // 100, near.sum()
    np.testing.assert_array_equal(got[ok].astype(np.int64), want[ok])
    ref_lp = ops.categorical_log_prob(torch.tensor(x, device="cuda"), act).cpu().numpy()
    np.testing.assert_array_equal(lp.cpu().numpy(), ref_lp)


def test_philox_sampling_reproducible_advancing_and_distributed():
    import torch
    from scipy import stats
    from torchrl_b200 import ops
    from torchrl_b200.policies.continuous_policy import _DeviceRng
    rng = _DeviceRng().ensure("cuda")
    A = 6
    row = np.array([0.3, -1.0, 2.0, 0.0, 1.2, -3.0], dtype=np.float32)
    M = 1 << 20
    x = torch.tensor(np.tile(row, (M, 1)), device="cuda")
    a1 = ops.categorical_sample(x, rng=rng).clone()
    a2 = ops.categorical_sample(x, rng=rng).clone()
    assert torch.equal(a1, a2)
    ops.counter_advance(rng.counter)
    a3 = ops.categorical_sample(x, rng=rng)
    assert not torch.equal(a1, a3)
    p = np.exp(row - row.max()).astype(np.float64)
    p /= p.sum()
    counts = np.bincount(a1.cpu().numpy().astype(np.int64), minlength=A)
    chi2, pval = stats.chisquare(counts, p * M)
    assert pval > 1e-4, (counts, p * M, pval)


def test_non_finite_logits_set_the_nan_flag():
    import torch
    from torchrl_b200 import ops
    from torchrl_b200.policies.continuous_policy import _DeviceRng
    x = torch.zeros(64, 6, device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.categorical_sample(x, rng=_DeviceRng().ensure("cuda"), nan_flag=flag)
    assert int(flag) == 0
    x[17, 2] = float("nan")
    ops.categorical_sample(x, rng=_DeviceRng().ensure("cuda"), nan_flag=flag)
    assert int(flag) == 1
