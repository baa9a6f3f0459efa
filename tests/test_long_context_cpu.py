"""The reference helpers and score patterns of test_long_context_gpu, checked on the CPU: both attention references against a
float64 softmax per q head (GQA grouping, left / right / causal mask bounds), the vectorized tile walk against the literal
64-key walk, keys outside the bounds never read, the needle's scaled gap underflowing fp32 exp2 for every other key, and the
sink / band and page-table constructors."""
import pytest
import torch

from test_long_context_gpu import (BF, HD, LOG2E, NEEDLE_GAP, PAGE, attention_refs, bf16_ulp, flat, needle_gap, needle_q,
                                   paged_table, plant_needle, sink_recency, tie_positions)

CPU = "cpu"


def softmax_f64(q, k, v, begin, end, shift=None):
    """Each q head h against KV head h // G in float64: q [Sq, Hq, D], k / v [S, Hkv, D] -> [Sq, Hq * D]."""
    Sq, Hq, D = q.shape
    G = Hq // k.shape[1]
    out = torch.zeros(Sq, Hq, D, dtype=torch.float64)
    for h in range(Hq):
        for i in range(Sq):
            hi = end if shift is None else min(end, i + shift + 1)
            if hi <= begin:
                continue
            kk, vv = k[begin:hi, h // G].double(), v[begin:hi, h // G].double()
            p = torch.softmax(kk @ q[i, h].double() * D ** -0.5, 0)
            out[i, h] = p @ vv
    return out.view(Sq, Hq * D)


def walk_literal(q, k, v, begin, end, shift=None):
    """The kernels' walk one 64-key tile at a time (running max, per-tile rescale, P rounded to bf16 before P.V)."""
    Sq, Hq, D = q.shape
    G = Hq // k.shape[1]
    sl2 = float(torch.tensor(D ** -0.5, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32))
    kk = k.float().repeat_interleave(G, 1).transpose(0, 1)                # [Hq, S, D]
    vv = v.float().repeat_interleave(G, 1).transpose(0, 1)
    s = q.float().transpose(0, 1) @ kk.transpose(1, 2)                    # [Hq, Sq, S]
    j = torch.arange(k.shape[0])
    ok = (j >= begin) & (j < end)
    ok = ok[None].expand(Sq, -1)
    if shift is not None:
        ok = ok & (j[None] <= torch.arange(Sq)[:, None] + shift)
    s = s.masked_fill(~ok, float("-inf"))
    vv = vv.masked_fill(~ok[-1][None, :, None], 0.0)
    m = torch.full((Hq, Sq), float("-inf"))
    l = torch.zeros(Hq, Sq)
    o = torch.zeros(Hq, Sq, D)
    for t0 in range(begin // PAGE * PAGE, end, PAGE):
        st = s[..., t0:t0 + PAGE]
        m_new = torch.maximum(m, st.amax(-1))
        mref = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
        corr = torch.exp2((m - mref) * sl2)
        m = m_new
        p = torch.exp2((st - mref[..., None]) * sl2)
        l = l * corr + p.sum(-1)
        o = o * corr[..., None] + p.to(BF).float() @ vv[:, t0:t0 + PAGE]
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    return (o * inv[..., None]).to(BF).transpose(0, 1).reshape(Sq, Hq * D)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


# begin, end, shift over S = 300 keys: whole cache, right pad, left pad inside a tile, causal chunk after a past, all masked
BOUNDS = [(0, 300, None), (0, 129, None), (70, 300, None), (5, 64, None), (0, 300, 300 - 5), (70, 250, 200), (40, 40, None)]


@pytest.mark.parametrize("Sq", [1, 5])
@pytest.mark.parametrize("begin,end,shift", BOUNDS)
def test_refs_against_float64_and_literal_walk(Sq, begin, end, shift):
    Hq, Hkv, D, S = 8, 2, 64, 300
    q = flat(Sq, Hq, D, seed=1, device=CPU)
    k, v = flat(S, Hkv, D, seed=2, device=CPU, scale=2.0), flat(S, Hkv, D, seed=3, device=CPU)
    ref, matched = attention_refs(q, k, v, begin, end, shift)
    want = softmax_f64(q, k, v, begin, end, shift)
    if end <= begin:
        assert int(torch.count_nonzero(ref)) == 0 and int(torch.count_nonzero(matched)) == 0
        return
    assert rel(ref, want) < 1e-5, rel(ref, want)
    assert rel(matched, want) < 3e-3, rel(matched, want)
    # the vectorized walk is the literal one up to fp32 summation order: within one bf16 ulp everywhere
    lit = walk_literal(q, k, v, begin, end, shift)
    assert (matched.double() - lit.double()).abs().le(bf16_ulp(lit.double()) + 1e-30).all()
    # keys outside [begin, end) and any key no query sees: NaN / +-Inf there change no bit
    kp, vp = k.clone(), v.clone()
    out = torch.ones(S, dtype=torch.bool)
    out[begin:end if shift is None else min(end, Sq - 1 + shift + 1)] = False
    kp[out] = float("nan")
    vp[out] = torch.tensor([float("inf"), float("-inf")]).to(BF).repeat(S)[:S][out][:, None, None]
    r2, m2 = attention_refs(q, kp, vp, begin, end, shift)
    assert torch.equal(r2, ref) and torch.equal(m2, matched)


def test_refs_gqa_grouping():
    """A q head reads KV head h // G only: changing KV head 1 moves exactly q heads G..2G-1."""
    Hq, Hkv, D, S = 8, 2, 64, 200
    G = Hq // Hkv
    q = flat(3, Hq, D, seed=4, device=CPU)
    k, v = flat(S, Hkv, D, seed=5, device=CPU), flat(S, Hkv, D, seed=6, device=CPU)
    ref, matched = attention_refs(q, k, v, 0, S)
    v2 = v.clone()
    v2[:, 1] = flat(S, D, seed=7, device=CPU)
    r2, m2 = attention_refs(q, k, v2, 0, S)
    for t, t2 in ((ref, r2), (matched, m2)):
        t, t2 = t.view(3, Hq, D), t2.view(3, Hq, D)
        assert torch.equal(t[:, :G], t2[:, :G]) and not torch.equal(t[:, G:], t2[:, G:])
    assert rel(r2, softmax_f64(q, k, v2, 0, S)) < 1e-5


@pytest.mark.parametrize("p", [0, 63, 64, 70001, 131071])
def test_needle_gap_underflows_fp32_exp2(p):
    """At D = 128 over 131072 randn keys the needle's scaled log2 gap to every other key is > 160, so exp2 of every other key's
    (s_j - s_p) * scale * log2 e is exactly 0 in fp32, and both references return the needle's V row bit for bit."""
    Hkv, D, S, G = 2, HD, 131072, 4
    k, v = flat(S, Hkv, D, seed=8, device=CPU), flat(S, Hkv, D, seed=9, device=CPU)
    plant_needle(k, p)
    gap = needle_gap(k, p, 0, S)
    assert gap > NEEDLE_GAP, gap
    q = needle_q(1, G * Hkv, D, CPU)
    s = (k.float().transpose(0, 1) @ q.view(G * Hkv, D)[::G].float()[:, :, None])[..., 0]    # [Hkv, S] fp32
    sl2 = float(torch.tensor(D ** -0.5, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32))
    e = torch.exp2((s - s[:, p:p + 1]) * sl2)
    assert torch.equal(e[:, p], torch.ones(Hkv)) and int(torch.count_nonzero(e)) == Hkv
    ref, matched = attention_refs(q.view(1, G * Hkv, D), k, v, 0, S)
    want = v[p].repeat_interleave(G, 0).reshape(1, -1)
    assert torch.equal(matched, want) and torch.equal(ref.to(BF), want)


def test_sink_band_sets_the_max_early_and_corrects_it_late():
    """The sink scores above every flat key of the first tiles, and the band's largest score is above the sink's."""
    Hq, Hkv, D, S = 4, 1, HD, 131072
    q = flat(1, Hq * D, seed=10, device=CPU)
    k = flat(S, Hkv, D, seed=11, device=CPU)
    sink_recency(q, k, 0, S, Hq, D)
    s = (q.view(Hq, D).float() @ k[:, 0].float().T)                   # [Hq, S]
    sink, flat_max, band_max = s[:, 0], s[:, 1:S - 256].amax(-1), s[:, S - 256:].amax(-1)
    assert bool((sink > flat_max).all()) and bool((band_max > sink).all()), (sink, flat_max, band_max)


def test_tie_positions_and_paged_table():
    pos = tie_positions(70001, 131071)
    assert all(70001 <= p < 131071 for p in pos) and len({p // PAGE for p in pos}) == len(pos) > 20
    lens, n_pages, hot = [131072, 100001], 17411, [0, 1, 1500, 2047]
    t = paged_table(lens, n_pages, hot, seed=3)
    assert t.shape == (2, 2048)
    live = t[t >= 0]
    assert len(set(live.tolist())) == live.numel() and int(live.max()) < n_pages
    assert bool((t[1, -(-lens[1] // PAGE):] == -1).all()) and bool((t[0] >= 0).all())
    assert sorted(t[:, hot][t[:, hot] >= 0].tolist()) == list(range(n_pages - 2 * len(hot), n_pages - 1))
