"""The sampling cut-offs' float64 oracle (``kept`` / ``cutoffs`` / ``cutoff_margin`` below, on top of oracle/sampling.py's
top-k / top-p ``kept``) against transformers' MinP / Typical / Epsilon / EtaLogitsWarper after Temperature / TopK / TopP in
HF's order, its margins against fp32 evaluations of the same rules, and the host side of the new ABI entries (no device
needed).  tests/test_sampling_cutoffs_gpu.py checks the kernels against the same oracle."""
import math
import pathlib
import re

import pytest
import torch
from transformers.generation import logits_process as lp

from oracle import sampling as osm

ROOT = pathlib.Path(__file__).resolve().parents[1]


# ------------------------------------------------------------------------------------------------------------------------
# the oracle: HF's four cut-offs in float64 after oracle/sampling.py's top-k / top-p set
def kept(x: torch.Tensor, temperature: float, top_k: int = 0, top_p: float = 1.0, margin: float = 0.0, *, min_p: float = 0.0,
         typical_p: float = 1.0, epsilon: float = 0.0, eta: float = 0.0, cut_margin: float = 0.0) -> torch.Tensor:
    """``osm.kept`` (top-k, then top-p moved by ``margin``), then the cut-offs (``cutoffs``; all off by default), each moved
    by ``cut_margin``: x [R, V] fp32 -> bool [R, V], the finite entries a draw may pick."""
    keep = osm.kept(x, temperature, top_k, top_p, margin)
    if osm.f32(min_p) > 0.0 or osm.f32(typical_p) < 1.0 or osm.f32(epsilon) > 0.0 or osm.f32(eta) > 0.0:
        keep = cutoffs(x.double(), temperature, keep, min_p, typical_p, epsilon, eta, cut_margin)
    return keep & torch.isfinite(x)


def cutoffs(xd: torch.Tensor, temperature: float, keep: torch.Tensor, min_p: float = 0.0, typical_p: float = 1.0,
            epsilon: float = 0.0, eta: float = 0.0, cut_margin: float = 0.0) -> torch.Tensor:
    """HF's MinP -> Typical -> Epsilon -> Eta warpers (min_tokens_to_keep = 1) in float64 on the set ``keep`` [R, V] of rows
    xd [R, V] float64, each on the survivors of the one before; settings as the fp32 values the kernel reads, off as
    (0, 1, 0, 0).  m = exp((x - max) / T) with max the row maximum (always kept by top-k / top-p), p = m / Z over the current
    survivors, H = -sum p log p.  ``cut_margin`` c > 0 moves every cut towards fewer tokens, c < 0 towards more:
    min_p keeps m >= min_p + c; typical keeps d <= D - c and the tie group at D, D the d at which the cumulative p (d
    ascending) first reaches typical_p - c; epsilon / eta keep p >= threshold + c (and the largest survivor's tie group).
    A tie group has one m and one d, so each cut keeps or drops it whole."""
    T = osm.f32(temperature)
    mp, tp, ep, et = osm.f32(min_p), osm.f32(typical_p), osm.f32(epsilon), osm.f32(eta)
    a = (xd - xd.max(-1, keepdim=True).values) / T
    keep = keep.clone()
    for r in range(xd.shape[0]):
        k, ar = keep[r] & torch.isfinite(xd[r]), a[r]

        def probs(kk):
            m = torch.where(kk, torch.exp(ar), torch.zeros_like(ar))
            return m, m / m.sum()

        def entropy(p):
            q = p[p > 0]
            return float(-(q * q.log()).sum())

        if mp > 0.0:
            m, _ = probs(k)
            k = k & (m >= mp + cut_margin)
        if tp < 1.0:
            _, p = probs(k)
            H = entropy(p)
            d = torch.where(k & (p > 0), (-p.log() - H).abs(), torch.full_like(p, math.inf))
            ds, order = d.sort()
            cum = p[order].cumsum(0)
            n = int((k & (p > 0)).sum())
            last = min(int((cum < tp - cut_margin).sum()), n - 1)
            D = float(ds[last])
            k = k & ((d <= D - cut_margin) | (d == D))           # the tie group at D is the cut's own: kept whole
        for thr_of in ([lambda p: ep] if ep > 0.0 else []) + ([lambda p: min(et, math.sqrt(et) * math.exp(-entropy(p)))]
                                                              if et > 0.0 else []):
            _, p = probs(k)
            top = xd[r][k].max()
            k = k & ((p >= thr_of(p) + cut_margin) | (xd[r] == top))
        keep[r] = k
    return keep


def cutoff_margin(x: torch.Tensor, temperature: float, top_k: int = 0, top_p: float = 1.0) -> float:
    """A bound on how far each of the kernel's cut-off decisions can sit from the float64 one, in the units ``cutoffs``
    moves them by (a probability, a mass relative to the maximum, or a deviation d), for one row x [1, V].  With err_i the
    per-entry bound of ``osm.masses`` over the top-k / top-p survivors (a superset of every later stage's), Z their mass and
    E = sum err + n 2^-41 + 2^-40 the error of the fixed-point total (as in ``osm.top_p_margin``):
    * min_p compares the fp32 mass with min_p: off by at most max err (the __expf bound).
    * epsilon / eta compare the fp32 mass with fl32(threshold * Z_fixed): the probability moves by at most
      (max err + 2 E) / Z + 2^-23 (rounding of the threshold); eta's threshold also carries exp(-H)'s error, bounded by the
      entropy error below (|d exp(-H)| <= exp(-H) |dH| <= |dH|).
    * typical compares fp32 deviations |a - c| with c = S / Z (S = sum m a in float64): |dc| <= (sum err |a| + sum p |a32 - a|) / Z
      + |c| E / Z + 2^-24 |c|; each d also carries |a32 - a| and one fp32 rounding; its mass target carries 2 E / Z.
    The entropy error |dH| <= |dc| + E / Z.  The sum of these is returned: every decision the kernel makes lies within it of
    the float64 decision, so kept(cut_margin=+m) <= kernel <= kept(cut_margin=-m) when each earlier stage is unambiguous."""
    keep = osm.kept(x, temperature, top_k, top_p)
    p, err = osm.masses(x, temperature, keep)
    z = float(p.sum())
    e_tot = float(err.sum()) + int(keep.sum()) * 2.0 ** -41 + 2.0 ** -40
    a = ((x.double() - x.double().max(-1, keepdim=True).values) / osm.f32(temperature))
    a32 = osm.kernel_arg(x, temperature)
    fin = keep & torch.isfinite(a)
    aa = torch.where(fin, a, torch.zeros_like(a))
    da = torch.where(fin, (a32 - a).abs(), torch.zeros_like(a))
    c = float((p * aa).sum()) / z
    dc = (float((err * aa.abs()).sum()) + float((p * da).sum())) / z + abs(c) * e_tot / z + osm.EPS32 * abs(c)
    amax = float(aa.abs().max())
    d_err = 2.0 * (dc + float(da.max()) + 2.0 * osm.EPS32 * (amax + abs(c)))
    prob = (float(err.max()) + 2.0 * e_tot) / z + 2.0 ** -23 + dc + e_tot / z
    return float(err.max()) + prob + d_err + 2.0 ** -40


CASES = {
    "min_p": dict(min_p=0.05),
    "typical": dict(typical_p=0.8),
    "epsilon": dict(epsilon=3e-3),
    "eta": dict(eta=2e-3),
    "all": dict(min_p=0.02, typical_p=0.95, epsilon=1e-3, eta=1e-3),
}


def hf_scores(x, T, k, p, min_p=0.0, typical_p=1.0, epsilon=0.0, eta=0.0):
    """x [R, V] fp32 through HF's warpers (as _get_logits_processor adds them when sampling with num_beams = 1)."""
    procs = [lp.TemperatureLogitsWarper(T)]
    if 0 < k < x.shape[-1]:
        procs.append(lp.TopKLogitsWarper(k))
    if p < 1.0:
        procs.append(lp.TopPLogitsWarper(p))
    if min_p > 0:
        procs.append(lp.MinPLogitsWarper(min_p))
    if typical_p < 1.0:
        procs.append(lp.TypicalLogitsWarper(typical_p))
    if 0 < epsilon < 1:
        procs.append(lp.EpsilonLogitsWarper(epsilon))
    if 0 < eta < 1:
        procs.append(lp.EtaLogitsWarper(eta))
    s = x.clone()
    ids = torch.zeros(x.shape[0], 1, dtype=torch.long)
    for proc in procs:
        s = proc(ids, s)
    return s


def llama_like(g, V, R=1):
    """Peaked rows: a normal background and a few large logits, as an LM head gives."""
    x = torch.randn(R, V, generator=g) * 2.0
    top = torch.randint(0, V, (R, 8), generator=g)
    x.scatter_(1, top, 8.0 + 3.0 * torch.rand(R, 8, generator=g))
    return x.float()


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_equals_hf(name):
    kw = CASES[name]
    g = torch.Generator().manual_seed(len(name))
    checked = 0
    for trial in range(40):
        V = (300, 1000, 4096)[trial % 3]
        T = (0.7, 1.0, 1.5)[trial % 3]
        k, p = ((0, 1.0), (50, 0.9), (200, 1.0), (0, 0.95))[trial % 4]
        x = llama_like(g, V)
        m = cutoff_margin(x, T, k, p)
        tight = kept(x, T, k, p, **kw, cut_margin=m)
        loose = kept(x, T, k, p, **kw, cut_margin=-m)
        if not torch.equal(tight, loose):
            continue                                     # the cut sits within the margin: ambiguous by construction
        if p < 1.0:
            pm = osm.top_p_margin(x, T, k)
            if not torch.equal(osm.kept(x, T, k, p, margin=pm), osm.kept(x, T, k, p, margin=-pm)):
                continue
        want = torch.isfinite(hf_scores(x, T, k, p, **kw))
        assert torch.equal(kept(x, T, k, p, **kw), want), (name, trial)
        checked += 1
    assert checked >= 25, checked


def test_typical_can_drop_the_maximum():
    x = torch.full((1, 200), 4.0)
    x[0, 7] = 5.0
    x[0, 100:] = -2.0
    x = x.float()
    hf = torch.isfinite(hf_scores(x, 1.0, 0, 1.0, typical_p=0.5))
    ours = kept(x, 1.0, typical_p=0.5)
    assert torch.equal(ours, hf) and not bool(ours[0, 7]) and bool(ours[0, :7].all())


def test_signed_zeros_are_one_value():
    """-0.0 and +0.0 share one m and one d: every cut keeps or drops the two together."""
    g = torch.Generator().manual_seed(5)
    for kw in CASES.values():
        for _ in range(10):
            x = (torch.randint(-12, 3, (1, 400), generator=g).float() * 0.5)
            x[0, ::7] = 0.0
            x[0, 3::7] = -0.0
            keep = kept(x, 1.0, 0, 1.0, **kw)
            z = x[0] == 0
            assert bool(keep[0][z].all()) or not bool(keep[0][z].any())


@pytest.mark.parametrize("name", list(CASES))
def test_margins_bracket_fp32_rules(name):
    """The same rules evaluated in fp32 (torch softmax, fp32 entropy and cumsum, as HF runs them) land between the float64
    oracle moved by -margin and by +margin."""
    kw = CASES[name]
    g = torch.Generator().manual_seed(100 + len(name))
    for trial in range(20):
        V, T = (1000, 4096)[trial % 2], (0.8, 1.0, 1.3)[trial % 3]
        x = llama_like(g, V)
        m = cutoff_margin(x, T)
        tight, loose = kept(x, T, **kw, cut_margin=m), kept(x, T, **kw, cut_margin=-m)
        if not torch.equal(kept(x, T, **{k: v for k, v in kw.items() if k == "min_p"}, cut_margin=m),
                           kept(x, T, **{k: v for k, v in kw.items() if k == "min_p"}, cut_margin=-m)):
            continue
        got = torch.isfinite(hf_scores(x, T, 0, 1.0, **kw))
        assert bool((tight <= got).all() and (got <= loose).all()), (name, trial)


def test_abi_symbols_bound():
    from ultravox_b200 import _lib
    header = (ROOT / "include" / "uvx.h").read_text()
    names = sorted(set(re.findall(r"\b(uvx_\w*_cutoffs)\s*\(", header)))
    assert names == ["uvx_record_scores_cutoffs", "uvx_record_scores_rows_cutoffs", "uvx_sample_cutoffs",
                     "uvx_sample_rows_cutoffs", "uvx_sample_slots_cutoffs"]
    for name in names:
        assert name in _lib.SIGNATURES, name
    assert [f for f, _ in _lib.Cutoffs._fields_] == ["min_p", "typical_p", "epsilon", "eta"]


def test_argument_checks():
    from ultravox_b200 import ops
    assert ops.sampling_cutoffs() == ops.CUTOFFS_OFF
    assert ops.sampling_cutoffs(0.05, 0.9, 3e-4, 2e-4) == (0.05, 0.9, 3e-4, 2e-4)
    assert ops.sampling_cutoffs(typical_p=1.5, epsilon_cutoff=1.0, eta_cutoff=-0.1) == ops.CUTOFFS_OFF   # HF's gating: off
    assert ops.sampling_cutoffs(epsilon_cutoff=0.0, eta_cutoff=0.0) == ops.CUTOFFS_OFF
    for bad in (dict(min_p=-0.1), dict(min_p=1.5), dict(min_p=math.nan), dict(typical_p=0.0), dict(typical_p=-1.0),
                dict(typical_p=math.nan)):
        with pytest.raises(ValueError):
            ops.sampling_cutoffs(**bad)
    assert not ops.cutoffs_on(None) and not ops.cutoffs_on(ops.CUTOFFS_OFF) and ops.cutoffs_on((0.0, 0.99, 0.0, 0.0))
