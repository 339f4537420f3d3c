"""The generic kernel-matrix pipeline (raw r -> within_subject_column in place -> SYRK), the parts that need no GPU: the
reference of its normaliser with its error bound, and the reference's precomputed-kernel fixtures above 64 epochs
(tests/golden/make_golden_precomputed_wide.py) against the oracle's fp32 restatement on the regenerated inputs.

Normaliser bound (``wsc_ref``).  ``within_subject_column`` (fcma_b200.cu) restates fcma_extension.cc:52-84 in IEEE fp32:
Fisher ``0.5 logf(fl(fl(1 + r) / fl(1 - r)))`` (clamps 1e-4 where ``1 +- r <= 0``), sequential sums of z and z^2 over
the subject's eps epochs, ``var = sq/eps - mean^2``, ``inv = 1 / sqrt(var)`` (both correctly rounded), then
``(z - mean) inv``.  With u = 2^-24, for a kernel that reads r + dr, |dr| <= rho:
* Fisher: the three roundings of the quotient move ``ln q`` by at most 3u, ``logf`` (at most 1 ulp) adds 2u |ln q|,
  halving is exact: ``eF = rho / (1 - (|r| + rho)^2) + 2u (1 + |F|)`` (the first term: the mean value theorem on
  atanh, whose derivative is 1 / (1 - r^2)).
* z-score: the sums err by at most (eps - 1) u sum |F| and eps u sum F^2, the divisions, the square and the
  difference by one rounding each, so ``|dvar| <= (3 eps + 4) u (var + m^2)``; inv adds 2 roundings to half of that,
  ``(z - mean) inv`` two more; |m| / sigma <= 1 + m^2/var.  Collecting,
  ``|dz| <= (4 eps + 8) u (1 + m^2/var) max(1, |z|) + (2 + |z| zmax) max_subject(eF) / sigma``,
  the second term the propagation of an input error eF (the mean moves by eF, the variance by 2 sigma zmax eF).
* Trailing epochs (e >= (E / eps) eps) keep r: ``|dz| <= rho``.
* Ill-conditioned subjects, where no first-order bound exists, are left out by the rule of ``zref`` in
  test_gpu_norm_syrk.py ((3 eps + 1) u (1 + m^2/var) >= 1/16, or the Fisher term (2 + zmax^2) eF / sigma reaching 1/16),
  plus the limit of that rule, a subject whose fp64 variance is 0 at a mean != 0 (equal r in every epoch, e.g. the self
  column of a one-mask block clamped at r >= 1): the fp32 variance is then rounding noise and z is arbitrary, in the
  reference's fp32 as in the kernel.  With one mask this leaves out the self column where its r is clamped.

Kernel bound between two fp32 implementations x, y of the pipeline (``side_bound``): with z_c a centre (the oracle's
fp32 z) and |z_x - z_c| <= D_x, an fp32 chain of n2 products (any order, ssyrk or k_syrk_simt) gives
``|K_x - Z_c Z_c^T| <= F(D_x) + n2 u (S_c + F(D_x))``, F(D) = sum_j (D_aj |z_bj| + |z_aj| D_bj + D_aj D_bj), S_c =
sum_j |z_aj z_bj|; ``|K_x - K_y|`` is the sum of both sides.  The decimal shrink multiplies both by the same
float32(10^(2 - nd)) (the digit counts must agree unless K[0, 0] lies within the bound of a power of ten) and rounds
once more: ``p (bound + u (|K_x| + |K_y|))``.  r: an fp32 chain over T samples errs by at most T u sum |x y|.
"""
import math
import os

import numpy as np
import pytest
import torch

from brainiak_b200.fcma import synthetic
from oracle import fcma_oracle as orc

U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ------------------------------------------------------------------------------- the normaliser's reference and bound
def wsc_ref(r, eps, rho=None):
    """fp64 reference of within_subject_column on r (float64 tensor [rows, E, n2], any device) and the bound of
    |z_kernel - z| for a kernel that reads r + dr, |dr| <= rho.  Returns (z, delta, ill)."""
    rows, E, n2 = r.shape
    rho = torch.zeros_like(r) if rho is None else rho
    ill = torch.zeros(r.shape, dtype=torch.bool, device=r.device)
    z = r.clone()
    delta = rho.clone()
    S = (E // eps) * eps
    if S:
        v = r[:, :S]
        num = torch.where(1 + v <= 0, torch.full_like(v, 1e-4), 1 + v)
        den = torch.where(1 - v <= 0, torch.full_like(v, 1e-4), 1 - v)
        F = 0.5 * torch.log(num / den)
        rs = rho[:, :S]
        ef = rs / (1 - (v.abs() + rs).clamp(max=1 - 1e-12) ** 2) + 2 * U * (1 + F.abs())
        g = F.reshape(rows, S // eps, eps, n2)
        m = g.mean(2, keepdim=True)
        var = ((g - m) ** 2).mean(2, keepdim=True)
        pos = var > 0
        sd = torch.sqrt(torch.where(pos, var, torch.ones_like(var)))
        zz = torch.where(pos, (g - m) / sd, torch.zeros_like(g))
        cond = 1 + m * m / torch.where(pos, var, torch.ones_like(var))
        zmax = zz.abs().amax(2, keepdim=True)
        efm = ef.reshape(g.shape).amax(2, keepdim=True) / sd
        d = (4 * eps + 8) * U * cond * zz.abs().clamp(min=1) + (2 + zz.abs() * zmax) * efm
        # zref's rule, and its limit: an fp64 variance of 0 (or below rounding) at a mean != 0
        bad = pos & (((3 * eps + 1) * U * cond >= 1.0 / 16) | ((2 + zmax * zmax) * efm >= 1.0 / 16))
        bad = bad | (~pos & (m != 0))
        d = torch.where(pos & ~bad, d, torch.zeros_like(d))
        z[:, :S] = zz.reshape(rows, S, n2)
        delta[:, :S] = d.reshape(rows, S, n2)
        ill[:, :S] = bad.expand(g.shape).reshape(rows, S, n2)
    return z, delta, ill


def side_bound(zc, D, n2):
    """|K_x - Z_c Z_c^T| <= F(D) + n2 u (S_c + F(D)) for an fp32 chain over z_x, |z_x - z_c| <= D ([rows, E, n2])."""
    a = zc.abs()
    DA = torch.einsum("iaj,ibj->iab", D, a)
    F = DA + DA.transpose(1, 2) + torch.einsum("iaj,ibj->iab", D, D)
    S = torch.einsum("iaj,ibj->iab", a, a)
    return F + n2 * U * (S + F)


def digits(k00):
    return len(str(int(k00)))


def near_power_of_ten(k, bound):
    """k within bound of +-10^j for some j >= 1 (where the digit count of int(k) may go either way)."""
    a = abs(float(k))
    if a < 5:
        return False
    j = round(math.log10(a))
    return abs(a - 10.0 ** j) <= float(bound)


# ------------------------------------------------------------------------------- the fixtures' inputs
def fixture_inputs(name):
    """(raw, raw2, eps) of tests/golden/vs_pre_<name>.npz, regenerated from their seeds."""
    if name == "w1":
        return synthetic.make_dyadic_epochs(48, 20, 140, seed=4242, informative=8)[0], None, 20
    d1, d2, _ = synthetic.make_two_masks(24, 40, 16, 100, seed=6262)
    return d1, d2, 12


def corr_terms(raw, raw2, v):
    """For row voxel v: the oracle's fp32 r, sum_t |x y| and |x| |y| (fp64), each [1, E, V2], and the epoch length T."""
    r = orc.corr_block(raw, raw2, v, 1)
    cols = raw if raw2 is None else raw2
    P = orc.corr_block([np.abs(m) for m in raw], [np.abs(m) for m in cols], v, 1, f64=True)
    nx = np.stack([np.sqrt((m[:, v].astype(np.float64) ** 2).sum()) for m in raw])
    ny = np.stack([np.sqrt((m.astype(np.float64) ** 2).sum(0)) for m in cols])
    N = (nx[:, None] * ny)[None]
    return r, P, N, max(m.shape[0] for m in raw)


def kernel_pair_bound(raw, raw2, v, eps, rho_x, rho_y=None):
    """(z_c, bound of |K_x - K_y| unshrunk) for row voxel v, z_c the oracle's fp32 z; rho_x(P, N, T), rho_y(...): each
    side's bound of its r error against the oracle's r (None: the side is the oracle itself, D = 0)."""
    r, P, N, T = corr_terms(raw, raw2, v)
    n2 = r.shape[2]
    rt = torch.from_numpy(r).double()
    zc = torch.from_numpy(orc.within_subject_norm(r.copy(), eps)).double()
    _, d0, ill = wsc_ref(rt, eps)                # the oracle's own normaliser rounding
    assert not ill.any(), "ill-conditioned subject in a fixture voxel"
    total = 0.0
    for rho in (rho_x, rho_y):
        if rho is None:
            total = total + side_bound(zc, torch.zeros_like(zc), n2)
            continue
        _, dx, ill = wsc_ref(rt, eps, torch.from_numpy(rho(P, N, T)))
        assert not ill.any(), "ill-conditioned subject in a fixture voxel"
        total = total + side_bound(zc, dx + d0, n2)
    return zc, total


def ref_rho(P, N, T):
    """|r_reference - r_oracle|: two fp32 chains over T samples."""
    return 2 * T * U * P


def oracle_shrunk(raw, raw2, v, eps):
    """The oracle's fp32 pipeline for row voxel v: (unshrunk K [E, E] float32, digit count, shrunk K)."""
    _, _, K = orc.voxel_block(raw, raw2, v, 1, eps, shrink=False)
    Ks = K[0].copy()
    nd = orc.shrink_(Ks)
    return K[0], nd, Ks


def compare_shrunk(K_got_shrunk, nd_got, K_ref_shrunk, K_unshrunk_centre, bound, what):
    """The fixture's shrunk kernel against another implementation's, both within ``bound`` (unshrunk) of each other.
    Returns the fraction of the bound used."""
    nd_ref = digits(K_unshrunk_centre[0, 0])
    near = near_power_of_ten(K_unshrunk_centre[0, 0], bound[0, 0])
    if not near:
        assert nd_got == nd_ref, "%s: digit count %d, the reference's %d" % (what, nd_got, nd_ref)
    p = float(np.float32(10.0 ** (2 - nd_got))) if nd_got > 2 else 1.0
    a = np.asarray(K_got_shrunk, np.float64)
    b = np.asarray(K_ref_shrunk, np.float64)
    lim = p * bound.numpy() + U * (np.abs(a) + np.abs(b))
    err = np.abs(a - b)
    assert np.all(err <= lim), "%s: %d entries outside the bound, worst excess %.3g" % (
        what, int((err > lim).sum()), float((err - lim).max()))
    return float((err / lim).max())


# ------------------------------------------------------------------------------- tests
def test_wsc_ref_matches_oracle_fp32():
    """The fp64 reference of within_subject_column against the oracle's fp32 restatement of fcma_extension.cc (the
    same arithmetic), inside the bound with rho = 0, at eps 3, 5, 12, 13 and 20 with trailing epochs, a dead column and a
    column of equal r (r = 1, clamped) that the rule leaves out."""
    rng = np.random.RandomState(8)
    for E, eps in ((9, 3), (33, 5), (100, 12), (65, 13), (140, 20)):
        r = np.tanh(rng.randn(2, E, 60) * 0.5).astype(np.float32)
        r[0, :, 4] = 0.0
        r[1, :, 7] = 1.0
        want = orc.within_subject_norm(r.copy(), eps).astype(np.float64)
        z, d, ill = wsc_ref(torch.from_numpy(r).double(), eps)
        S = (E // eps) * eps
        assert bool(ill[1, :S, 7].all()) and not bool(ill[0].any())
        ok = ~ill.numpy()
        err = np.abs(want - z.numpy())
        assert np.all(err[ok] <= d.numpy()[ok]), (E, eps, float((err - d.numpy())[ok].max()))
        assert np.array_equal(want[:, S:], r[:, S:].astype(np.float64))
        assert np.all(want[0, :, 4] == 0)


@pytest.mark.parametrize("name", ["w1", "w2"])
def test_precomputed_fixture_kernels_match_oracle(golden, name):
    """The reference's shrunk kernels of the sampled voxels (planted ones included) against the oracle's fp32 pipeline
    on the regenerated inputs, within both fp32 chains' bound; the input probes match."""
    g = golden("vs_pre_" + name)
    raw, raw2, eps = fixture_inputs(name)
    assert int(g["eps"]) == eps
    assert np.array_equal(np.stack([raw[e][:4, ::997][:, :16] for e in (0, len(raw) - 1)]), g["probe"])
    if raw2 is not None:
        assert np.array_equal(np.stack([raw2[e][:4, ::997][:, :16] for e in (0, len(raw2) - 1)]), g["probe2"])
    for v, K_ref in zip(g["sample_vids"], g["sample_kernels"]):
        v = int(v)
        K_orc, nd, K_orc_s = oracle_shrunk(raw, raw2, v, eps)
        _, bound = kernel_pair_bound(raw, raw2, v, eps, ref_rho)
        frac = compare_shrunk(K_orc_s, nd, K_ref, K_orc, bound[0], "%s voxel %d" % (name, v))
        print("%s voxel %d: %.3g of the bound" % (name, v, frac))
