"""Sampling cut-offs (min_p, typical_p, epsilon, eta) in the sampler (generate.cu ``cutoff_band``, behind
``uvx_sample_cutoffs``, ``uvx_record_scores(_rows)_cutoffs``, ``uvx_sample_slots_cutoffs`` and ``uvx_sample_rows_cutoffs``),
in ``generate()`` and in the slots, against the float64 oracle (tests/test_sampling_cutoffs_cpu.py on top of oracle/sampling.py) and transformers' warpers.

Kernel rows are checked where the oracle's cut is unambiguous (``cutoff_margin``): the recorded finite set equals the
oracle's kept set with x / T bit for bit (and equals HF's warpers), and every draw lies inside the proven inverse-CDF window
over that set.  Exact rows (unit masses, the rest flushed or cut) must give ``kept[floor(fl32(u * m))]`` exactly."""
import math

import pytest
import torch

from oracle import sampling as osm
from test_sampling_cutoffs_cpu import CASES, cutoff_margin, hf_scores, kept, llama_like
from test_sampling_parity_gpu import around, exact_support, grid, top_of_unit

pytestmark = pytest.mark.gpu

V_LLAMA = 128256
OFF = (0.0, 1.0, 0.0, 0.0)


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def cut(kw):
    return (kw.get("min_p", 0.0), kw.get("typical_p", 1.0), kw.get("epsilon", 0.0), kw.get("eta", 0.0))


def draw(ops, row, T, k, p, cf, us):
    """One row [V] cuda, uniforms us [n] -> picks [n]: the row tiled over the batch, one uniform per copy."""
    n = us.numel()
    big = row.view(1, -1).repeat(n, 1)
    return ops.sample(big, T, k, us.cuda(), None, top_p=p, cutoffs=cf)


def recorded(ops, rows, T, k, p, cf):
    R, V = rows.shape
    sc = torch.empty(1, R, V, device="cuda")
    ops.record_scores(rows, T, k, p, torch.zeros(1, dtype=torch.int32, device="cuda"), scores=sc, cutoffs=cf)
    return sc[0]


def unambiguous(x, T, k, p, kw):
    m = cutoff_margin(x, T, k, p)
    tight, loose = kept(x, T, k, p, **kw, cut_margin=m), kept(x, T, k, p, **kw, cut_margin=-m)
    if p < 1.0:
        pm = osm.top_p_margin(x, T, k)
        if not torch.equal(osm.kept(x, T, k, p, margin=pm), osm.kept(x, T, k, p, margin=-pm)):
            return None
    return tight[0] if torch.equal(tight, loose) else None


# ------------------------------------------------------------------------------------------------------------------------
# kernel: general rows
@pytest.mark.parametrize("V", [1000, V_LLAMA])
@pytest.mark.parametrize("name", list(CASES))
def test_general_rows(ops, V, name):
    kw = CASES[name]
    cf = cut(kw)
    g = torch.Generator().manual_seed(V + len(name))
    checked = 0
    for trial in range(12):
        T = (0.7, 1.0, 1.5)[trial % 3]
        k, p = ((0, 1.0), (50, 0.9), (50, 1.0), (0, 0.95))[trial % 4]
        x = llama_like(g, V)
        keep = unambiguous(x, T, k, p, kw)
        if keep is None:
            continue
        xc = x.cuda()
        sc = recorded(ops, xc, T, k, p, cf)[0].cpu()
        fin = torch.isfinite(sc)
        assert torch.equal(fin, keep), (name, trial, int(fin.sum()), int(keep.sum()))
        assert torch.equal(sc[fin], (x[0] / torch.tensor(T, dtype=torch.float32))[fin]), (name, trial)
        assert torch.equal(sc.isfinite(), torch.isfinite(hf_scores(x, T, k, p, **kw))[0]), (name, trial)
        us = torch.cat([grid(257), top_of_unit(16)])
        picks = draw(ops, xc[0], T, k, p, cf, us)
        res = osm.check_draws(x[0].cuda(), T, keep.cuda(), us.cuda(), picks)
        assert bool(res["inside"].all()), (name, trial)
        checked += 1
    assert checked >= 6, checked


@pytest.mark.parametrize("V", [1025, V_LLAMA])
def test_exact_rows(ops, V):
    """Support tokens at the row maximum (mass 1 each) on chunk edges, index 0 and V - 1; a background 12 below it that every
    cut-off removes (its mass e^-12 < min_p, its probability < epsilon / eta, its deviation far from the support's)."""
    S = exact_support(V)
    x = torch.full((V,), 3.5 - 12.0)
    x[S] = 3.5
    x[1:S[1]:3] = -math.inf
    m = len(S)
    us = torch.cat([grid(4 * m + 1), around(torch.arange(1, m).double() / m, 2), top_of_unit(8)])
    want = torch.tensor(S)[torch.floor((us.double().clamp(max=osm.U_MAX) * m).float().double()).long().clamp(max=m - 1)]
    for kw in ({"min_p": 0.01}, {"typical_p": 0.5}, {"epsilon": 1e-3}, {"eta": 1e-3},
               {"min_p": 1e-3, "typical_p": 0.9, "epsilon": 1e-4, "eta": 1e-4}):
        picks = draw(ops, x.cuda(), 1.0, 0, 1.0, cut(kw), us).cpu()
        assert torch.equal(picks, want), kw


def test_typical_drops_maximum_ties_and_zeros(ops):
    x = torch.full((1, 2000), 4.0)
    x[0, 7] = 5.0
    x[0, 1000:] = -2.0
    x = x.float().cuda()
    sc = recorded(ops, x, 1.0, 0, 1.0, (0.0, 0.5, 0.0, 0.0))[0].cpu()
    assert not math.isfinite(float(sc[7])) and bool(torch.isfinite(sc[:7]).all()) and bool(torch.isfinite(sc[8:1000]).all())
    assert torch.equal(torch.isfinite(sc), torch.isfinite(hf_scores(x.cpu(), 1.0, 0, 1.0, typical_p=0.5))[0])
    picks = draw(ops, x[0], 1.0, 0, 1.0, (0.0, 0.5, 0.0, 0.0), grid(512)).cpu()
    assert bool((picks != 7).all()) and bool((picks < 1000).all())
    # tie groups and +-0 at each cut: a coarse grid of values, so every cut falls between or on tie groups
    g = torch.Generator().manual_seed(2)
    for kw in CASES.values():
        for _ in range(6):
            y = torch.randint(-16, 1, (1, 3000), generator=g).float() * 0.5
            y[0, ::5] = 0.0
            y[0, 2::5] = -0.0
            sc = recorded(ops, y.cuda(), 1.0, 0, 1.0, cut(kw))[0].cpu()
            fin = torch.isfinite(sc)
            for v in y[0].unique():
                grp = fin[y[0] == v]
                assert bool(grp.all()) or not bool(grp.any()), (kw, float(v))
            keep = unambiguous(y, 1.0, 0, 1.0, kw)
            if keep is not None:
                assert torch.equal(fin, keep), kw


def test_all_ninf_and_batch_independence(ops):
    V = 5000
    for kw in CASES.values():
        x = torch.full((3, V), -math.inf, device="cuda")
        out = ops.sample(x, 1.0, 0, torch.rand(3, device="cuda"), None, cutoffs=cut(kw))
        assert out.tolist() == [0, 0, 0]
    g = torch.Generator().manual_seed(9)
    rows = llama_like(g, V_LLAMA, 8).cuda()
    u = torch.rand(8, generator=g).cuda()
    cf = cut(CASES["all"])
    batch = ops.sample(rows, 0.9, 50, u, None, top_p=0.95, cutoffs=cf)
    for b in range(8):
        one = ops.sample(rows[b:b + 1].contiguous(), 0.9, 50, u[b:b + 1].contiguous(), None, top_p=0.95, cutoffs=cf)
        assert int(one) == int(batch[b]), b
    rs = torch.empty(1, 8, V_LLAMA, device="cuda")
    rr = torch.empty(8, V_LLAMA, device="cuda")
    ops.record_scores(rows, 0.9, 50, 0.95, torch.zeros(1, dtype=torch.int32, device="cuda"), scores=rs, cutoffs=cf)
    ops.record_scores_rows(rows, 0.9, 50, 0.95, torch.arange(8, dtype=torch.int32, device="cuda"), scores=rr, cutoffs=cf)
    assert torch.equal(rs[0], rr)
    assert bool(torch.isfinite(rs[0].gather(1, batch[:, None])).all())      # a pick always has a finite recorded score


def test_slots_and_rows_forms_equal_scalar(ops):
    B, V = 8, V_LLAMA
    g = torch.Generator().manual_seed(4)
    rows = llama_like(g, V, B).cuda()
    settings = [(0.8, 50, 0.9, cut(CASES["min_p"])), (1.0, 0, 1.0, OFF), (1.2, 40, 1.0, cut(CASES["typical"])),
                (0.0, 0, 1.0, cut(CASES["eta"])), (0.7, 0, 0.95, cut(CASES["epsilon"])), (1.0, 50, 1.0, cut(CASES["all"])),
                (0.9, 20, 0.8, OFF), (1.0, 0, 1.0, cut(CASES["eta"]))]
    temps = torch.tensor([s[0] for s in settings], device="cuda")
    top_k = torch.tensor([s[1] for s in settings], dtype=torch.int32, device="cuda")
    top_p = torch.tensor([s[2] for s in settings], device="cuda")
    cuts = torch.tensor([s[3] for s in settings], device="cuda")
    off = torch.tensor([OFF] * B, device="cuda")
    W = 6
    u = torch.rand(B, W, generator=g).cuda()
    active = torch.ones(B, dtype=torch.int32, device="cuda")
    for step in range(W):
        n_new = torch.full((B,), step, dtype=torch.int32, device="cuda")
        got = torch.full((B,), -1, dtype=torch.int64, device="cuda")
        ops.sample_slots_cutoffs(rows, temps, top_k, top_p, cuts, u, n_new, active, got)
        for b, (t, k, p, cf) in enumerate(settings):
            if t > 0:
                want = ops.sample(rows[b:b + 1].contiguous(), t, k, u[b, step:step + 1].contiguous(), None, top_p=p, cutoffs=cf)
            else:
                want = rows[b].argmax().view(1)
            assert int(got[b]) == int(want), (step, b)
        # every row off: uvx_sample_slots bit for bit
        a = torch.empty(B, dtype=torch.int64, device="cuda")
        c = torch.empty(B, dtype=torch.int64, device="cuda")
        ops.sample_slots(rows, temps, top_k, top_p, u, n_new, active, a)
        ops.sample_slots_cutoffs(rows, temps, top_k, top_p, off, u, n_new, active, c)
        assert torch.equal(a, c), step
    # the row-mapped form: R = 16 rows of 8 slots, rows past a slot's drafts (idx -1) untouched
    R = 16
    big = torch.cat([rows, rows.flip(0)]).contiguous()
    row_slot = torch.tensor(list(range(8)) + list(range(7, -1, -1)), dtype=torch.int32, device="cuda")
    row_idx = torch.tensor([0] * 8 + [1, 2, -1, 3, 0, 1, 2, -1], dtype=torch.int32, device="cuda")
    got = torch.full((R,), -7, dtype=torch.int64, device="cuda")
    ops.sample_rows_cutoffs(big, temps, top_k, top_p, cuts, u, active, row_slot, row_idx, got)
    for r in range(R):
        s, i = int(row_slot[r]), int(row_idx[r])
        if i < 0:
            assert int(got[r]) == -7
            continue
        t, k, p, cf = settings[s]
        want = (ops.sample(big[r:r + 1].contiguous(), t, k, u[s, i:i + 1].contiguous(), None, top_p=p, cutoffs=cf) if t > 0
                else big[r].argmax().view(1))
        assert int(got[r]) == int(want), r
    a = torch.empty(R, dtype=torch.int64, device="cuda")
    c = torch.empty(R, dtype=torch.int64, device="cuda")
    ops.sample_rows(big, temps, top_k, top_p, u, active, row_slot, row_idx.clamp_min(0), a)
    ops.sample_rows_cutoffs(big, temps, top_k, top_p, off, u, active, row_slot, row_idx.clamp_min(0), c)
    assert torch.equal(a, c)


def test_abi_argument_errors(ops):
    from ultravox_b200 import _lib
    x = torch.zeros(1, 100, device="cuda")
    u = torch.rand(1, device="cuda")
    for bad in ((1.5, 1.0, 0.0, 0.0), (0.0, 0.0, 0.0, 0.0), (0.1, 1.0, 1.0, 0.0), (0.1, 1.0, 0.0, math.nan), (math.nan, 0.9, 0.0, 0.0)):
        with pytest.raises(_lib.UvxError):
            ops.sample(x, 1.0, 0, u, None, cutoffs=bad)


# ------------------------------------------------------------------------------------------------------------------------
# generate()
def _micro():
    from test_logits_constraints_gpu import _model
    return _model()


@pytest.fixture(scope="module")
def micro():
    return _micro()


GEN_CASES = {"min_p": dict(min_p=0.1), "typical": dict(typical_p=0.7), "epsilon": dict(epsilon_cutoff=0.02),
             "eta": dict(eta_cutoff=0.02), "all": dict(min_p=0.05, typical_p=0.9, epsilon_cutoff=0.01, eta_cutoff=0.01)}


def _oracle_kw(kw):
    return dict(min_p=kw.get("min_p", 0.0), typical_p=kw.get("typical_p", 1.0), epsilon=kw.get("epsilon_cutoff", 0.0),
                eta=kw.get("eta_cutoff", 0.0))


def _check_generate_scores(out, S, T, k, p, kw):
    """output_scores = HF's warpers on output_logits where the oracle's cut is unambiguous; every token has a finite score
    in both.  Returns (steps checked, ambiguous steps)."""
    seqs = out.sequences.cpu()
    ok = amb = 0
    for t in range(len(out.scores)):
        x = out.logits[t].cpu()
        got = out.scores[t].cpu()
        tok = seqs[:, S + t]
        assert bool(torch.isfinite(got.gather(1, tok[:, None])).all()), (kw, t)
        for b in range(x.shape[0]):
            if unambiguous(x[b:b + 1], T, k, p, _oracle_kw(kw)) is None:
                amb += 1
                continue
            want = hf_scores(x[b:b + 1], T, k, p, **_oracle_kw(kw))[0]
            assert torch.equal(got[b], want), (kw, t, b)
            ok += 1
    return ok, amb


@pytest.mark.parametrize("name", list(GEN_CASES))
def test_generate_scores_are_hf(micro, name):
    cfg, model = micro
    kw = GEN_CASES[name]
    ids = torch.randint(0, 1000, (1, 10), generator=torch.Generator().manual_seed(3)).cuda()
    S, n = 10, 16
    run = lambda **x: model.generate(ids, max_new_tokens=n, do_sample=True, temperature=0.9, top_k=0,  # noqa: E731
                                     generator=torch.Generator(device="cuda").manual_seed(5), **kw, **x)
    out = run(return_dict_in_generate=True, output_scores=True, output_logits=True)
    ok, amb = _check_generate_scores(out, S, 0.9, 0, 1.0, kw)
    assert ok >= n // 2 and amb <= n // 4, (ok, amb)
    assert torch.equal(run(), out.sequences)                     # reproducible for a seeded generator
    assert torch.equal(run(use_graph=False), out.sequences)      # graph replay == eager steps
    look = run(prompt_lookup_num_tokens=3)
    assert torch.equal(look, out.sequences)                      # prompt lookup: the tokens of plain decoding
    greedy = model.generate(ids, max_new_tokens=n)
    assert torch.equal(model.generate(ids, max_new_tokens=n, **kw), greedy)      # ignored when not sampling


def test_generate_padded_turn_audio_8b_and_errors(micro):
    cfg, model = micro
    kw = GEN_CASES["all"]
    B, S, n = 3, 12, 10
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(0, 1000, (B, S), generator=g)
    am = torch.ones(B, S, dtype=torch.long)
    for b in range(1, B):
        am[b, :2 * b] = 0
        ids[b, :2 * b] = 0
    ids, am = ids.cuda(), am.cuda()
    out = model.generate(ids, attention_mask=am, max_new_tokens=n, do_sample=True, top_k=40, top_p=0.95,
                         generator=torch.Generator(device="cuda").manual_seed(1), return_dict_in_generate=True,
                         output_scores=True, output_logits=True, **kw)
    ok, amb = _check_generate_scores(out, S, 1.0, 40, 0.95, kw)
    assert ok >= B * n // 2, (ok, amb)
    one = ids[:1]
    t1 = model.generate(one, max_new_tokens=6, return_dict_in_generate=True)
    follow = torch.cat([t1.sequences, torch.randint(0, 1000, (1, 4), generator=g).cuda()], 1)
    turn = model.generate(follow, past_key_values=t1.past_key_values, max_new_tokens=8, do_sample=True,
                          generator=torch.Generator(device="cuda").manual_seed(2), return_dict_in_generate=True,
                          output_scores=True, output_logits=True, **kw)
    _check_generate_scores(turn, follow.shape[1], 1.0, 50, 1.0, kw)
    from test_logprobs_gpu import audio_request
    feats = audio_request(cfg, 16000, 7)
    au = model.generate(max_new_tokens=8, do_sample=True, generator=torch.Generator(device="cuda").manual_seed(3),
                        return_dict_in_generate=True, output_scores=True, output_logits=True, **feats, **kw)
    _check_generate_scores(au, feats["input_ids"].shape[1], 1.0, 50, 1.0, kw)
    for bad in (dict(min_p=1.5), dict(min_p=-0.1), dict(typical_p=0.0), dict(typical_p=math.nan)):
        with pytest.raises(ValueError):
            model.generate(ids[:1], max_new_tokens=2, do_sample=True, **bad)
    with pytest.raises(NotImplementedError):
        model.generate(ids[:1], max_new_tokens=2, do_sample=True, num_beams=2, min_p=0.1)


def _8b_model():
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=2))
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


# ------------------------------------------------------------------------------------------------------------------------
# slots
EOS = [7, 11]


def _slot_settings(i):
    opts = [dict(do_sample=True, min_p=0.1), dict(do_sample=True, temperature=0.8, typical_p=0.8), {},
            dict(do_sample=True, top_k=40, epsilon_cutoff=0.02), dict(do_sample=True, top_p=0.9),
            dict(do_sample=True, eta_cutoff=0.01, repetition_penalty=1.2),
            dict(do_sample=True, temperature=1.1, min_p=0.05, typical_p=0.9, epsilon_cutoff=0.01, eta_cutoff=0.01),
            dict(min_p=0.2)]                                   # greedy: ignored
    return dict(opts[i % len(opts)])


def _serve(sched, reqs):
    ids = []
    for feats, n, st, seed in reqs:
        kw = dict(st)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
        ids.append(sched.submit(feats, max_new_tokens=n, **kw))
    out = sched.run()
    return [out[i] for i in ids]


def _gen(model, feats, n, st, seed, **extra):
    kw = dict(st)
    if kw.get("do_sample"):
        kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
    return model.generate(max_new_tokens=n, eos_token_id=EOS, **feats, **kw, **extra)


def test_slots_equal_generate_busy_lookup_paged(micro, ops):
    from test_logprobs_gpu import _logprobs_of_logits, audio_request, text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    reqs = [((audio_request(cfg, 16000, 100 + i) if i % 3 == 0 else text_request(cfg, 6 + 3 * i, 200 + i)), 10 + i % 5,
             _slot_settings(i), 50 + i) for i in range(12)]
    one = SlotScheduler(model, slots=1, max_len=400, eos_token_ids=EOS, max_logprobs=2)
    for feats, n, st, seed in reqs[:8]:
        kw = dict(st)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
        rid = one.submit(feats, max_new_tokens=n, logprobs=2, **kw)
        got = one.run()[rid]
        out = _gen(model, feats, n, st, seed, return_dict_in_generate=True, output_logits=True)
        assert torch.equal(got, out.sequences), st
        S = feats["input_ids"].shape[1]
        w_lp, w_ids, _ = _logprobs_of_logits(ops, torch.cat(out.logits), out.sequences[0, S:], 2)
        lp = one.logprobs[rid]
        assert torch.equal(lp.token_logprobs, w_lp) and torch.equal(lp.top_ids, w_ids), st
    assert one.engine.captures == 1
    mk = lambda **kw: SlotScheduler(model, slots=8, max_len=400, eos_token_ids=EOS, sync_every=3, **kw)  # noqa: E731
    busy = _serve(mk(), reqs)
    alone_s = mk()
    for i, r in enumerate(reqs):
        alone, = _serve(alone_s, [r])
        assert torch.equal(busy[i], alone), (i, r[2])
    eager = _serve(mk(use_graph=False), reqs)
    for i in range(len(reqs)):
        assert torch.equal(busy[i], eager[i]), i
    # a chunked prompt equals itself alone
    long = (text_request(cfg, 300, 901), 12, _slot_settings(6), 77)
    mixed = _serve(mk(), reqs[:4] + [long])
    assert torch.equal(mixed[4], _serve(alone_s, [long])[0])
    # the lookup step equals a plain engine of slots x (K + 1) slots
    base = torch.randint(1, 1000, (1, 6), generator=torch.Generator().manual_seed(8))
    lreqs = [(dict(input_ids=torch.cat([base, base, base[:, :3], torch.tensor([[20 + i]])], 1).cuda()), 14, _slot_settings(i),
              70 + i) for i in range(4)]
    look = SlotScheduler(model, slots=2, max_len=128, eos_token_ids=EOS, prompt_lookup_num_tokens=3)
    plain = SlotScheduler(model, slots=8, max_len=128, eos_token_ids=EOS)
    got = _serve(look, [(f, n, dict(s, prompt_lookup_num_tokens=3), seed) for f, n, s, seed in lreqs])
    for g_, w_, r in zip(got, _serve(plain, lreqs), lreqs):
        assert torch.equal(g_, w_), r[2]
    # a paged session turn equals chained generate()
    paged = SlotScheduler(model, slots=4, max_len=256, eos_token_ids=EOS, kv_pages=64)
    sid = paged.open_session()
    t1 = text_request(cfg, 10, 5)
    st = _slot_settings(6)
    r1, = _serve_session(paged, sid, [(t1, 8, st, 3)])
    g1 = _gen(model, t1, 8, st, 3, return_dict_in_generate=True)
    assert torch.equal(r1, g1.sequences)
    follow = torch.cat([r1, torch.randint(1, 1000, (1, 5), generator=torch.Generator().manual_seed(6)).cuda()], 1)
    r2, = _serve_session(paged, sid, [(dict(input_ids=follow), 8, st, 4)])
    g2 = _gen(model, dict(input_ids=follow), 8, st, 4, past_key_values=g1.past_key_values)
    assert torch.equal(r2, g2)


def _serve_session(sched, sid, reqs):
    ids = []
    for feats, n, st, seed in reqs:
        kw = dict(st)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
        ids.append(sched.submit(feats, max_new_tokens=n, session=sid, **kw))
    out = sched.run()
    return [out[i] for i in ids]


def test_8b_widths(ops):
    from test_logprobs_gpu import text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = _8b_model()
    reqs = [(text_request(cfg, 9 + i, 300 + i), 8, _slot_settings(i), 80 + i) for i in range(8)]
    s = SlotScheduler(model, slots=8, max_len=64, eos_token_ids=EOS)
    busy = _serve(s, reqs)
    for i, r in enumerate(reqs):
        alone, = _serve(s, [r])
        assert torch.equal(busy[i], alone), i
    one = SlotScheduler(model, slots=1, max_len=64, eos_token_ids=EOS)
    for r in reqs[:3]:
        got, = _serve(one, [r])
        assert torch.equal(got, _gen(model, *r)), r[2]
    ids = reqs[1][0]["input_ids"]
    out = model.generate(ids, max_new_tokens=6, do_sample=True, generator=torch.Generator(device="cuda").manual_seed(1),
                         return_dict_in_generate=True, output_scores=True, output_logits=True, **GEN_CASES["all"])
    _check_generate_scores(out, ids.shape[1], 1.0, 50, 1.0, GEN_CASES["all"])
