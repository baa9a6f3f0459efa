"""The float64 sampler oracle (oracle/sampling.py) against transformers' own warpers, on the CPU.

``kept`` must be the set HF's TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper leaves finite wherever no tie
group straddles the top-p cut (there the library keeps the group whole and HF's sort may split it) and the cut is not within
a hair of a token boundary (where fp32 and fp64 cumulative sums may disagree).  ``check_draws`` is pinned on rows whose
masses are small integers, where the inverse CDF can be written down by hand."""
import math

import pytest
import torch

from oracle import sampling as osm

MARGIN = 1e-4     # HF sums its softmax in fp32: a cut this close to a token boundary may fall either way


def hf_finite(x, T, k, p):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = TemperatureLogitsWarper(T)(None, x.float().clone())
    if k:
        s = TopKLogitsWarper(k)(None, s)
    if p < 1.0:
        s = TopPLogitsWarper(p)(None, s)
    return torch.isfinite(s)


def test_kept_matches_transformers_warpers():
    V = 1000
    g = torch.Generator().manual_seed(0)
    rows = torch.cat([torch.randn(3, V, generator=g) * s for s in (0.5, 2.0, 5.0)])
    rows[1, ::7] = -math.inf
    rows[4, 900:] = -math.inf
    checked = skipped = 0
    for T in (0.6, 1.0, 1.7):
        for k in (0, 1, 50, V - 1, V, V + 7):
            for p in (0.0, 0.5, 0.9, 0.99, 1.0):
                want = hf_finite(rows, T, k, p)
                lo = osm.kept(rows, T, k, p, margin=MARGIN)
                hi = osm.kept(rows, T, k, p, margin=-MARGIN)
                for r in range(rows.shape[0]):
                    if not torch.equal(lo[r], hi[r]):
                        skipped += 1
                        continue
                    assert torch.equal(lo[r], want[r]), (T, k, p, r)
                    assert torch.equal(osm.kept(rows[r:r + 1], T, k, p)[0], want[r]), (T, k, p, r)
                    checked += 1
    # flat rows put ~1e-3 of the mass on each token, so some cuts land within MARGIN of a boundary: 688 of 810 are clear
    assert checked >= 0.8 * (checked + skipped), (checked, skipped)


def test_kept_signed_zero_is_one_value():
    """HF's top-k keeps `scores >= kth`, so a k-th value of +0.0 keeps every -0.0 too; the oracle agrees."""
    x = torch.full((1, 64), -3.0)
    x[0, :5] = torch.tensor([4.0, 3.0, 2.0, 1.0, 0.5])
    x[0, [10, 20, 30]] = 0.0
    x[0, [15, 25]] = -0.0
    for k in (6, 8, 10):
        want = hf_finite(x, 1.0, k, 1.0)
        assert torch.equal(osm.kept(x, 1.0, k), want), k
        assert int(want.sum()) == 10
    # a top-p cut inside the zero group keeps the whole group (5 + 5 zeros; the cut falls between their members)
    z = torch.full((1, 16), -math.inf)
    z[0, 0] = 1.0
    z[0, 1:6] = 0.0
    z[0, 6:11] = -0.0
    got = osm.kept(z, 1.0, 0, 0.5)
    assert got[0, :11].all() and not got[0, 11:].any()


def test_check_draws_on_integer_masses():
    """Five tokens at the maximum among -inf entries: mass 1 each, Z = 5, so the pick for u is kept[floor(fl32(5 u))]."""
    x = torch.full((50,), -math.inf)
    support = [0, 9, 10, 31, 49]
    x[support] = 2.5
    keep = osm.kept(x.view(1, -1), 1.0)[0]
    assert keep.nonzero().view(-1).tolist() == support
    u = torch.tensor([0.0, 0.1999, 0.2, 0.39999998, 0.4, 0.6, 0.8, 0.99999994, 0.9999], dtype=torch.float32)
    want = [0, 0, 9, 9, 10, 31, 49, 49, 49]
    r = osm.check_draws(x, 1.0, keep, u, torch.tensor(want), delta=0.0)
    assert r["expected"].tolist() == want and bool(r["inside"].all())
    wrong = torch.tensor([9, 9, 31, 49, 0, 0, 0, 10, 10])
    assert not bool(osm.check_draws(x, 1.0, keep, u, wrong, delta=0.0)["inside"].any())
    # a pick on a -inf entry is never inside, however wide the window
    assert not bool(osm.check_draws(x, 1.0, keep, u[:1], torch.tensor([48]), delta=10.0)["inside"].any())


@pytest.mark.parametrize("T", [0.25, 1.0, 1.8])
def test_error_bound_covers_fp32_sums(T):
    """The window is at least the gap between a plain fp32 left-to-right CDF (rounded masses included) and the float64
    one, on the widest row kind the GPU suite uses."""
    V = 128256
    x = torch.randn(V, generator=torch.Generator().manual_seed(1)) * 3
    keep = osm.kept(x.view(1, -1), T)[0]
    p, _ = osm.masses(x.view(1, -1), T, keep.view(1, -1))
    m32 = torch.exp(osm.kernel_arg(x, T).float())
    c32 = m32.cumsum(0)                                     # fp32 cumsum: one rounding per add, like the walk
    gap = float((c32.double() - p.view(-1).cumsum(0)).abs().max())
    assert gap < osm.error_bound(x.view(1, -1), T, keep.view(1, -1))
