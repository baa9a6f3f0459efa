"""Per-op parity of the token sampler (generate.cu ``keep_threshold`` + ``sample_row``, behind ``uvx_sample``,
``uvx_sample_top_p``, ``uvx_sample_slots`` and ``uvx_sample_rows``) and of the set ``uvx_record_scores`` leaves finite,
against the float64 oracle in oracle/sampling.py: each draw maps a given uniform to a token, and that token is compared with
the one an inverse CDF over the oracle's kept set picks.

Two tiers.
* Exact rows: every kept token sits at the row maximum (mass __expf(0) = 1) and every other entry is -inf, cut by top-k, cut
  by top-p far from the boundary, or so far below the maximum that __expf flushes it to 0.  The kernel's sums are then
  small integers and each draw must be ``kept[floor(fl32(u * m))]`` exactly.  The kept tokens sit where the kernel's
  bookkeeping changes: chunk edges t*c - 1 / t*c (c = ceil(V / 1024)), index 0 and V - 1, next to threads with empty chunks.
* General rows: each pick must have positive float64 mass and a CDF interval that, widened by the proven fp32 error bound
  delta (``oracle.sampling.error_bound``), contains the target; where that window holds one token, it must be the oracle's.

Uniforms: a midpoint grid, every chunk boundary and kept-token boundary of the float64 CDF with the floats around it, and
the top of [0, 1).  Rows are tiled (at most 256 copies per launch) and a [steps, rows] uniform table is stepped through with
``step_idx``, as the decode step does."""
import math

import pytest
import torch

from oracle import sampling as osm

pytestmark = pytest.mark.gpu

V_LLAMA = 128256
LLAMA_EOS = (128001, 128008, 128009)
TILE_BYTES = 1 << 30


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------------------------------
# helpers

def around(u, k):
    """fp32 uniforms u and the k floats on either side of each, kept inside [0, 1)."""
    u = u.float().clamp(0.0, osm.U_MAX)
    out, up, dn = [u], u, u
    for _ in range(k):
        up, dn = torch.nextafter(up, torch.ones_like(up)), torch.nextafter(dn, torch.zeros_like(dn))
        out += [up, dn]
    return torch.cat(out).clamp(0.0, osm.U_MAX)


def top_of_unit(n=64):
    return torch.tensor([1.0 - j * 2.0 ** -24 for j in range(n)], dtype=torch.float32)


def grid(n):
    return ((torch.arange(n, dtype=torch.float64) + 0.5) / n).float()


def draw(ops, rows, T, k, p, us):
    """rows [R, V] cuda, us: R uniform lists -> R pick lists (ops.sample: uvx_sample for p >= 1, else uvx_sample_top_p)."""
    R, V = rows.shape
    copies = max(1, min(256 // R, TILE_BYTES // (R * V * 4)))
    L = max(u.numel() for u in us)
    steps = -(-L // copies)
    tab = torch.full((R, steps * copies), 0.5, dtype=torch.float32)
    for r, u in enumerate(us):
        tab[r, :u.numel()] = u
    utab = tab.view(R, steps, copies).permute(1, 2, 0).reshape(steps, copies * R).contiguous().cuda()
    big = rows.repeat(copies, 1)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.empty(steps, copies * R, dtype=torch.int64, device="cuda")
    for s in range(steps):
        step.fill_(s)
        ops.sample(big, T, k, utab, step, out=out[s], top_p=p)
    picks = out.view(steps, copies, R).permute(2, 0, 1).reshape(R, steps * copies)
    return [picks[r, :u.numel()] for r, u in enumerate(us)]


def recorded(ops, rows, T, k, p):
    """uvx_record_scores of rows [R, V] -> scores [R, V] fp32 (the step buffer's only step)."""
    R, V = rows.shape
    sc = torch.empty(1, R, V, device="cuda")
    ops.record_scores(rows, T, k, p, torch.zeros(1, dtype=torch.int32, device="cuda"), scores=sc)
    return sc[0]


def check_recorded(rows, T, k, p, scores, tag):
    """The finite set of uvx_record_scores is the oracle's kept set (bracketed by the top-p margin when the cut may fall
    either way) and its values are x / T, IEEE, bit for bit.  Returns the kernel's kept mask and the ambiguous rows."""
    got = torch.isfinite(scores)
    want_div = rows.cpu() / torch.tensor(T, dtype=torch.float32)
    assert torch.equal(scores.cpu()[got.cpu()], want_div[got.cpu()]), tag
    amb = []
    for r in range(rows.shape[0]):
        x = rows[r:r + 1]
        m = osm.top_p_margin(x, T, k) if osm.f32(p) < 1.0 else 0.0
        lo, hi = osm.kept(x, T, k, p, margin=m)[0], osm.kept(x, T, k, p, margin=-m)[0]
        g = got[r]
        assert bool((lo <= g).all() and (g <= hi).all()), (tag, r, int(lo.sum()), int(g.sum()), int(hi.sum()))
        if not torch.equal(lo, hi):
            amb.append(r)
    return got, amb


def chunk_and_token_uniforms(x, T, keep, chunk_k=4, token_k=4, max_tokens=1024, seed=0):
    """u = C / Z at every chunk end and at the end of (up to max_tokens, seeded choice of) kept tokens, with the floats
    around each."""
    V = x.numel()
    c = (V + 1023) // 1024
    p, _ = osm.masses(x.view(1, -1), T, keep.view(1, -1))
    cum = p.view(-1).cumsum(0)
    z = float(cum[-1])
    ends = torch.arange(c - 1, V, c, device=x.device)
    toks = keep.nonzero().view(-1)
    if toks.numel() > max_tokens:
        g = torch.Generator(device="cpu").manual_seed(seed)
        toks = toks[torch.randperm(toks.numel(), generator=g)[:max_tokens].to(toks.device)]
    return torch.cat([around((cum[ends] / z).cpu(), chunk_k), around((cum[toks] / z).cpu(), token_k)])


# ------------------------------------------------------------------------------------------------------------------------
# exact tier

EXACT_V = [1, 2, 1000, 1023, 1024, 1025, 32000, V_LLAMA, 1 << 20]
TOP = 3.5


def exact_support(V):
    c = -(-V // 1024)
    s = {0, V - 1}
    for t in (1, 2, 31, 32, 33, 100, 511, 512, 513, 1000, 1022, 1023):
        s.update(i for i in (t * c - 1, t * c) if 0 <= i < V)
    return sorted(s)


def exact_rows(V, variants):
    """(name, row, top_k, top_p) with the support at TOP; the rest as the variant says."""
    S = exact_support(V)
    m = len(S)
    g = torch.Generator().manual_seed(V)
    out = []
    for name in variants:
        if name == "ninf":
            x, k, p = torch.full((V,), -math.inf), 0, 1.0
        elif name == "k_over":                                   # top_k beyond the finite entries: -inf keys are kept
            if m + 10 >= V:
                continue
            x, k, p = torch.full((V,), -math.inf), m + 10, 1.0
        elif name == "topk":                                     # finite background cut by top-k
            if m >= V:
                continue
            x, k, p = torch.rand(V, generator=g) * 7.0 - 4.0, m, 1.0
        elif name == "topp":                                     # background mass < 1e-6, cut at 0.5
            if m >= V:
                continue
            x, k, p = TOP - 60.0 - 10.0 * torch.rand(V, generator=g), 0, 0.5
        elif name == "deep":                                     # __expf of <= -104 flushes to 0 (the one assumption)
            if m >= V:
                continue
            x, k, p = TOP - 200.0 - torch.rand(V, generator=g), 0, 1.0
        x[S] = TOP
        out.append((name, x, k, p))
    return S, out


def exact_uniforms(m):
    j = torch.arange(m + 1, dtype=torch.float64)
    return torch.cat([around((j / m).float(), 2), torch.zeros(1), top_of_unit(), grid(4096)])


@pytest.mark.parametrize("V", EXACT_V)
def test_exact_rows_every_draw(ops, V):
    S, rows = exact_rows(V, ("ninf", "k_over", "topk", "topp", "deep"))
    u = exact_uniforms(len(S))
    for name, x, k, p in rows:
        xc = x.cuda()
        keep = torch.zeros(V, dtype=torch.bool, device="cuda")
        keep[S] = True
        for T in (0.25, 1.0, 1.8):
            if name != "deep":                                   # deep entries keep a float64 mass the kernel flushes
                assert torch.equal(osm.kept(xc.view(1, -1), T, k, p)[0], keep), (V, name, T)
            pick = draw(ops, xc.view(1, -1), T, k, p, [u])[0]
            want = osm.check_draws(xc, T, keep, u.cuda(), pick, delta=0.0)["expected"]
            bad = (pick != want).nonzero().view(-1)
            assert bad.numel() == 0, (V, name, T, [(float(u[i]), int(pick[i]), int(want[i])) for i in bad[:8].tolist()])


def test_exact_row_at_the_documented_maximum(ops):
    """V = 2^24 (the largest V the sampler accepts): c = 16384-entry chunks."""
    V = 1 << 24
    S, rows = exact_rows(V, ("ninf", "topk"))
    u = exact_uniforms(len(S))
    keep = torch.zeros(V, dtype=torch.bool, device="cuda")
    keep[S] = True
    for name, x, k, p in rows:
        xc = x.cuda()
        pick = draw(ops, xc.view(1, -1), 1.0, k, p, [u])[0]
        want = osm.check_draws(xc, 1.0, keep, u.cuda(), pick, delta=0.0)["expected"]
        assert torch.equal(pick, want), name
        del xc


# ------------------------------------------------------------------------------------------------------------------------
# general tier

def general_rows(V=V_LLAMA):
    g = torch.Generator().manual_seed(11)
    c = (V + 1023) // 1024
    rows, names = [], []

    def add(name, x):
        rows.append(x)
        names.append(name)

    for s in (0.5, 1.0, 3.0, 8.0):
        add(f"flat x{s}", torch.randn(V, generator=g) * s)
    x = torch.randn(V, generator=g) * 1.5
    x[torch.randperm(V, generator=g)[:40]] = 9.0 + 0.8 * torch.randn(40, generator=g)
    add("peaked", x)
    x = torch.randn(V, generator=g) * 3.0
    ids = torch.randperm(V, generator=g)[:300]
    x[ids] = torch.where(x[ids] < 0, x[ids] * 1.3, x[ids] / 1.3)        # HF's repetition penalty 1.3
    add("penalty", x)
    for s in (1.0, 3.0):
        x = torch.randn(V, generator=g) * s
        x[c - 1::c] = -math.inf                                         # every chunk ends in a banned token
        add(f"chunk-end -inf x{s}", x)
    x = torch.randn(V, generator=g) * 2.0
    x[128002:] = -math.inf                                              # Llama-3's reserved ids suppressed
    add("reserved tail -inf", x)
    x = torch.randn(V, generator=g) * 2.0
    x[torch.tensor([i for i in LLAMA_EOS if i < V], dtype=torch.long)] = -math.inf   # min_new_tokens: EOS ids banned
    add("eos -inf", x)
    return torch.stack(rows).cuda(), names


def general_settings(V):
    s = []
    for T in (0.25, 0.7, 1.0, 1.8):
        s += [(T, 0, 1.0), (T, 0, 0.9), (T, 50, 1.0), (T, 50, 0.99), (T, V - 1, 0.5), (T, V, 1.0)]
    s += [(1.0, 1, 1.0), (1.0, 0, 0.0), (1.0, V + 7, 0.99), (0.7, 50, 0.5)]
    return s


# Share of draws whose window holds more than one token (over all settings; about 0.03 above what these seeded rows give).
# delta is ~2.5e-5 of the mass at V = 128256 and flat rows put ~1e-5 on each token, and every targeted uniform sits on a
# boundary by design, so flat rows have many; the bound keeps the unique-window equality check meaningful.
MULTI_SHARE_MAX = {"flat x0.5": 0.64, "flat x1.0": 0.55, "flat x3.0": 0.30, "flat x8.0": 0.15, "peaked": 0.35, "penalty": 0.30,
                   "chunk-end -inf x1.0": 0.64, "chunk-end -inf x3.0": 0.43, "reserved tail -inf": 0.41, "eos -inf": 0.41}


def run_general(ops, rows, names, T, k, p, n_grid, stats):
    R, V = rows.shape
    scores = recorded(ops, rows, T, k, p)
    keep, _ = check_recorded(rows, T, k, p, scores, (T, k, p))
    us = []
    for r in range(R):
        wide = 16 if names[r].startswith("chunk-end") else 4
        us.append(torch.cat([grid(n_grid), top_of_unit(),
                             chunk_and_token_uniforms(rows[r], T, keep[r], chunk_k=wide, seed=r)]))
    picks = draw(ops, rows, T, k, p, us)
    for r in range(R):
        tag = (names[r], T, k, p)
        res = osm.check_draws(rows[r], T, keep[r], us[r].cuda(), picks[r])
        bad = (~res["inside"]).nonzero().view(-1)
        assert bad.numel() == 0, (tag, res["delta"], [(float(us[r][i]), int(picks[r][i]), float(rows[r][picks[r][i]]),
                                                        int(res["expected"][i])) for i in bad[:8].tolist()])
        one = res["width"] == 1
        assert torch.equal(picks[r][one], res["expected"][one]), tag
        assert bool(torch.isfinite(scores[r][picks[r]]).all()), tag           # a sampled token has a finite score
        multi = int((res["width"] > 1).sum())
        stats.setdefault(names[r], [0, 0])
        stats[names[r]][0] += multi
        stats[names[r]][1] += res["width"].numel()


def test_general_rows_inside_the_proven_window(ops):
    rows, names = general_rows()
    stats = {}
    for T, k, p in general_settings(V_LLAMA):
        run_general(ops, rows, names, T, k, p, 1 << 16, stats)
    for name, (multi, n) in stats.items():
        print(f"{name}: {multi} of {n} draws have a multi-token window")
        assert multi <= MULTI_SHARE_MAX[name] * n, (name, multi, n)


def test_few_finite_entries(ops):
    """1-30 finite entries among -inf at V = 128256, with top_k = #finite + 10 (beyond the finite entries), 0 and V."""
    V = V_LLAMA
    g = torch.Generator().manual_seed(12)
    for n_fin in (1, 2, 7, 30):
        x = torch.full((V,), -math.inf)
        x[torch.randperm(V, generator=g)[:n_fin]] = torch.randn(n_fin, generator=g) * 2.0
        x = x.cuda().view(1, -1)
        for T in (0.25, 1.0, 1.8):
            for k, p in ((n_fin + 10, 1.0), (0, 1.0), (V, 0.9), (n_fin + 10, 0.99)):
                scores = recorded(ops, x, T, k, p)
                keep, _ = check_recorded(x, T, k, p, scores, (n_fin, T, k, p))
                u = torch.cat([grid(1 << 12), top_of_unit(), chunk_and_token_uniforms(x[0], T, keep[0], 4, 8)])
                pick = draw(ops, x, T, k, p, [u])[0]
                res = osm.check_draws(x[0], T, keep[0], u.cuda(), pick)
                assert bool(res["inside"].all()), (n_fin, T, k, p)
                one = res["width"] == 1
                assert torch.equal(pick[one], res["expected"][one]), (n_fin, T, k, p)


# ------------------------------------------------------------------------------------------------------------------------
# radix-select edges and signed zeros

def radix_rows(V=32000):
    g = torch.Generator().manual_seed(13)
    out = []
    # ladders of keys that agree in their top 24, 16 and 8 bits, at scattered positions over a low background
    x = torch.randn(V, generator=g) - 6.0
    pos = torch.randperm(V, generator=g)
    j = torch.arange(300, dtype=torch.float64)
    x[pos[:300]] = (1.0 + j * 2.0 ** -23).float()
    x[pos[300:340]] = (2.0 + j[:40] * 2.0 ** -15).float()
    x[pos[340:360]] = (4.0 + j[:20] * 2.0 ** -7).float()
    out.append(("ladders", x, [(k, 1.0) for k in (1, 5, 20, 21, 40, 60, 61, 100, 104, 105, 300, 360, 361)] + [(300, 0.9)]))
    # a k-th value tied across 500 ranks
    x = torch.randn(V, generator=g) - 4.0
    pos = torch.randperm(V, generator=g)
    x[pos[:500]] = 2.0
    x[pos[500:520]] = 3.0
    out.append(("tied k-th", x, [(k, 1.0) for k in (20, 21, 100, 520, 521)] + [(300, 0.5)]))
    # mixed signs with ten +0.0 and ten -0.0: top-k cuts at and just past the zeros
    x = torch.randn(V, generator=g) * 2.0
    x[x.abs() < 1e-3] = 0.5
    pos = torch.randperm(V, generator=g)
    x[pos[:10]] = 0.0
    x[pos[10:20]] = -0.0
    n_pos = int((x > 0).sum())
    out.append(("signed zeros at the top-k cut", x, [(k, 1.0) for k in (n_pos + 1, n_pos + 5, n_pos + 20, n_pos + 21)]))
    # a top-p cut inside a tie group of ten +0.0 and ten -0.0 (interleaved) under a single maximum
    x = torch.full((V,), -math.inf)
    x[torch.randperm(V, generator=g)[:100]] = -8.0
    zi = torch.randperm(V - 10, generator=g)[:20] + 10
    x[3] = 1.0
    x[zi[0::2]] = 0.0
    x[zi[1::2]] = -0.0
    out.append(("signed zeros in a top-p group", x, [(0, 0.5), (0, 0.3), (0, 0.1), (50, 0.5)]))
    return out


def test_radix_select_edges_and_signed_zeros(ops):
    for name, x, settings in radix_rows():
        xc = x.cuda().view(1, -1)
        for k, p in settings:
            for T in (0.7, 1.0):
                tag = (name, T, k, p)
                want = osm.kept(xc, T, k, p)[0]
                m = osm.top_p_margin(xc, T, k) if p < 1.0 else 0.0
                assert torch.equal(osm.kept(xc, T, k, p, margin=m)[0], osm.kept(xc, T, k, p, margin=-m)[0]), tag
                scores = recorded(ops, xc, T, k, p)
                got = torch.isfinite(scores[0])
                assert torch.equal(got, want), (tag, int(got.sum()), int(want.sum()))
                u = torch.cat([grid(1 << 12), top_of_unit(), chunk_and_token_uniforms(xc[0], T, want, 4, 4)])
                pick = draw(ops, xc, T, k, p, [u])[0]
                res = osm.check_draws(xc[0], T, want, u.cuda(), pick)
                assert bool(res["inside"].all()), tag
                one = res["width"] == 1
                assert torch.equal(pick[one], res["expected"][one]), tag
                assert set(pick.unique().tolist()) <= set(want.nonzero().view(-1).tolist()), tag


def test_token_logprobs_cut_between_signed_zeros(ops):
    """n = 5 over three positives and four zeros (-0.0 at 5 and 9, +0.0 at 7 and 12): value desc, index asc takes 5 and 7."""
    V = 1000
    x = torch.linspace(-9.0, -1.0, V)
    x[[40, 41, 42]] = torch.tensor([3.0, 2.0, 1.0])
    x[[5, 9]] = -0.0
    x[[7, 12]] = 0.0
    x = x.cuda().view(1, -1)
    for n in (4, 5, 6, 7):
        out_lp = torch.empty(1, 1, device="cuda")
        ids = torch.full((1, 1, n), -1, dtype=torch.int64, device="cuda")
        top = torch.empty(1, 1, n, device="cuda")
        one = torch.ones(1, dtype=torch.int32, device="cuda")
        ops.token_logprobs(x, torch.tensor([40], device="cuda"), one * n, one * 0, out_lp, ids, top)
        want = [40, 41, 42, 5, 7, 9, 12][:n]
        assert ids.view(-1).tolist() == want, (n, ids.view(-1).tolist())


# ------------------------------------------------------------------------------------------------------------------------
# slots and rows forms against the oracle

def slot_settings(B, V):
    T = [0.7, 1.0, 0.0, 1.8, -1.0, 0.25, 1.0, 0.7]
    K = [0, 50, 0, V + 7, 0, 1, 0, 50]
    P = [1.0, 0.999, 1.0, 0.9, 0.5, 1.0, 0.999, 0.5]
    rep = -(-B // 8)
    return (torch.tensor((T * rep)[:B], dtype=torch.float32), torch.tensor((K * rep)[:B], dtype=torch.int32),
            torch.tensor((P * rep)[:B], dtype=torch.float32))


def check_row_picks(ops, x, T, k, p, u, picks, tag):
    """Draws of one row with its own settings (T <= 0: the first maximal index)."""
    if not T > 0:
        assert bool((picks == int(x.argmax())).all()), tag
        return
    scores = recorded(ops, x.view(1, -1), T, k, p)
    keep, _ = check_recorded(x.view(1, -1), T, k, p, scores, tag)
    res = osm.check_draws(x, T, keep[0], u, picks)
    assert bool(res["inside"].all()), tag
    one = res["width"] == 1
    assert torch.equal(picks[one], res["expected"][one]), tag


@pytest.mark.parametrize("B,V", [(8, V_LLAMA), (32, 32000)])
def test_sample_slots_against_oracle(ops, B, V):
    rows, _ = general_rows(V)
    lg = rows[torch.arange(B) % rows.shape[0]].contiguous()
    temp, top_k, top_p = (t.cuda() for t in slot_settings(B, V))
    active = torch.ones(B, dtype=torch.int32)
    active[5::7] = 0
    active = active.cuda()
    W = 24
    u_full = torch.rand(B, W + 8, generator=torch.Generator().manual_seed(B)).cuda()
    u = u_full[:, :W]                                               # u_stride = W + 8
    picks = torch.empty(B, W, dtype=torch.int64, device="cuda")
    used = torch.empty(B, W, device="cuda")
    ar = torch.arange(B, device="cuda")
    for step in range(W):
        n_new = ((ar * 5 + step) % W).int()
        out = torch.full((B,), -7, dtype=torch.int64, device="cuda")
        ops.sample_slots(lg, temp, top_k, top_p, u, n_new, active, out)
        picks[:, step] = out
        used[:, step] = u[ar, n_new.long()]
    for b in range(B):
        if not active[b]:
            assert bool((picks[b] == -7).all()), b
            continue
        check_row_picks(ops, lg[b], float(temp[b]), int(top_k[b]), float(top_p[b]), used[b], picks[b], ("slots", B, b))


def test_sample_rows_against_oracle(ops):
    V, slots, per = 32000, 4, 5
    rows, _ = general_rows(V)
    R = slots * per
    lg = rows[torch.arange(R) % rows.shape[0]].contiguous()
    temp, top_k, top_p = (t.cuda() for t in slot_settings(slots, V))
    active = torch.tensor([1, 1, 0, 1], dtype=torch.int32, device="cuda")
    row_slot = (torch.arange(R) // per).int().cuda()
    W = 16
    u = torch.rand(slots, W + 3, generator=torch.Generator().manual_seed(3)).cuda()[:, :W]
    got = {r: ([], []) for r in range(R)}
    for step in range(W):
        row_idx = ((torch.arange(R) * 3 + step) % (W + 2) - 2).int().cuda()   # some rows < 0: left alone
        out = torch.full((R,), -7, dtype=torch.int64, device="cuda")
        ops.sample_rows(lg, temp, top_k, top_p, u, active, row_slot, row_idx, out)
        for r in range(R):
            s, i = int(row_slot[r]), int(row_idx[r])
            if i < 0 or not active[s]:
                assert int(out[r]) == -7, (step, r)
                continue
            got[r][0].append(float(u[s, i]))
            got[r][1].append(int(out[r]))
    checked = 0
    for r, (us, ps) in got.items():
        if not ps:
            continue
        s = int(row_slot[r])
        check_row_picks(ops, lg[r], float(temp[s]), int(top_k[s]), float(top_p[s]), torch.tensor(us, device="cuda"),
                        torch.tensor(ps, device="cuda"), ("rows", r))
        checked += len(ps)
    assert checked > 100


def test_record_scores_rows_against_oracle(ops):
    V = 32000
    rows, _ = general_rows(V)
    B, steps = rows.shape[0], 8
    idx = torch.tensor([0, 3, -1, 5, 9, 2, 1, 4, 12, 8], dtype=torch.int32, device="cuda")   # -1, 9, 12, 8: outside [0, 8)
    for T, k, p in ((0.7, 50, 0.9), (1.0, 0, 0.99), (1.8, V - 1, 1.0)):
        sc = torch.full((steps, V), 123.0, device="cuda")
        ops.record_scores_rows(rows, T, k, p, idx, scores=sc)
        written = set()
        for b in range(B):
            s = int(idx[b])
            if 0 <= s < steps:
                check_recorded(rows[b:b + 1], T, k, p, sc[s:s + 1], ("record rows", T, k, p, b))
                written.add(s)
        assert written == set(range(6)), written
        for s in set(range(steps)) - written:
            assert bool((sc[s] == 123.0).all()), s


# ------------------------------------------------------------------------------------------------------------------------
# all -inf rows and reproducibility

def test_all_minus_inf_row_samples_index_zero(ops):
    for V in (1000, V_LLAMA):
        x = torch.full((3, V), -math.inf, device="cuda")
        u = torch.tensor([0.0, 0.5, osm.U_MAX], device="cuda")
        for k, p in ((0, 1.0), (50, 1.0), (0, 0.9), (V + 7, 0.5)):
            assert ops.sample(x, 1.0, k, u, top_p=p).tolist() == [0, 0, 0], (V, k, p)
        out = torch.full((3,), -7, dtype=torch.int64, device="cuda")
        ones = torch.ones(3, dtype=torch.int32, device="cuda")
        ops.sample_slots(x, torch.tensor([1.0, 0.7, 0.0], device="cuda"), torch.tensor([0, 50, 0], dtype=torch.int32,
                         device="cuda"), torch.tensor([1.0, 0.9, 1.0], device="cuda"), u.view(3, 1).contiguous(),
                         torch.zeros(3, dtype=torch.int32, device="cuda"), ones, out)
        assert out.tolist() == [0, 0, 0], V


def test_picks_reproducible_and_independent_of_batch(ops):
    V = V_LLAMA
    rows, _ = general_rows(V)
    R = rows.shape[0]
    u = torch.rand(R, generator=torch.Generator().manual_seed(4)).cuda()
    for T, k, p in ((1.0, 0, 1.0), (0.7, 50, 0.9), (1.8, 0, 0.99)):
        a = ops.sample(rows, T, k, u, top_p=p)
        assert torch.equal(a, ops.sample(rows, T, k, u, top_p=p))
        perm = torch.randperm(R, generator=torch.Generator().manual_seed(5)).cuda()
        assert torch.equal(ops.sample(rows[perm].contiguous(), T, k, u[perm].contiguous(), top_p=p), a[perm])
        other = torch.randn(R, V, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6)) * 5
        for r in (0, R // 2, R - 1):
            mixed = other.clone()
            mixed[r] = rows[r]
            assert int(ops.sample(mixed, T, k, u, top_p=p)[r]) == int(a[r]), (T, k, p, r)
