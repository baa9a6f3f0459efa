"""Log-probabilities from the graph-captured decode step: uvx_token_logprobs against torch.log_softmax in fp64,
generate(output_scores / output_logits) against transformers' own logits processors, and the slot engine's per-token
logprobs against generate() on each request alone, inside a busy engine, graph against eager."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V8B = 128256


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ builders (as test_serving_gpu)
def wave(i, n):
    return np.random.default_rng(1000 + i).standard_normal(n).astype(np.float32)


def build(name="micro", **kw):
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    cfg = preset(name, **kw)
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def audio_request(cfg, n_samples, seed, text_pre=8, text_post=5):
    """Processor-shaped features of one clip: 8 ids, the audio placeholders, 5 ids; mel computed on the device."""
    from oracle import logmel as ol
    from ultravox_b200 import ops
    padded, frames = ol.pad_batch([wave(seed, n_samples)])
    g = torch.Generator().manual_seed(seed)
    tok = int(-(-int(frames[0]) // 16))
    ids = torch.randint(0, min(cfg.vocab_size, 1000), (1, text_pre + tok + text_post), generator=g)
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    return dict(input_ids=ids.cuda(), audio_values=mel, audio_token_start_idx=torch.tensor([text_pre]).cuda(),
                audio_lens=torch.tensor([int(frames[0])]).cuda(), audio_token_len=torch.tensor([tok], dtype=torch.int32).cuda(),
                audio_batch_size=torch.ones(1, dtype=torch.int64).cuda())


def text_request(cfg, S, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(input_ids=torch.randint(0, min(cfg.vocab_size, 1000), (1, S), generator=g).cuda())


def serve(sched, reqs):
    """reqs: (features, n, settings, seed) -> submitted ids in order (settings may hold `logprobs`)."""
    ids = []
    for feats, n, settings, seed in reqs:
        kw = dict(settings)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
        ids.append(sched.submit(feats, max_new_tokens=n, **kw))
    return ids


def poison(sched):
    sched.engine.cache.k.fill_(float("nan"))
    sched.engine.cache.v.fill_(float("nan"))


def sharpen(model, cfg, logit_std=3.0):
    """Rescales the LM head so the logits have std `logit_std` (at random init they are nearly flat, and top-k / top-p would
    keep everything)."""
    ids = torch.randint(0, min(cfg.vocab_size, 1000), (1, 12), generator=torch.Generator().manual_seed(9)).cuda()
    std = float(model(ids, logits_to_keep=1).logits.float().std())
    model.language_model.lm_head.weight.data.mul_(logit_std / std)
    return model


def ranked(x):
    """Indices of a 1-D fp32 row by (value desc, index asc)."""
    x = x.double().cpu().numpy()
    return np.lexsort((np.arange(x.size), -x))


# ================================================================================================ 1. the kernel vs fp64
def _kernel_rows(V, seed):
    g = torch.Generator().manual_seed(seed)
    lg = torch.randn(8, V, generator=g) * 3
    lg[1, ::7] = -math.inf                                     # -inf entries
    lg[2, [V - 1, 40, 7, 3, V // 2]] = 30.0                    # 5-way tie at the top: n = 1 and 5 cut inside / at it
    lg[3, [11, 12, 13]] = torch.tensor([25.0, 24.0, 23.0])
    lg[3, [V - 2, 90, 50, 70]] = 20.0                          # a 4-way tie across the 5th place
    lg[5] -= 40.0
    lg[5, ::3] = -math.inf
    lg[5, torch.randperm(V // 3 - 1, generator=g)[:18] * 3 + 1] = 15.0
    lg[5, [11, 8, 5]] = 10.0                                   # a 3-way tie at the 20th place in a row of many -inf
    lg[6, [9, 2]] = 40.0                                       # a tie at the first place
    n_top = [-1, 0, 5, 5, 20, 20, 1, 1]
    return lg, n_top


@pytest.mark.parametrize("V", [1000, V8B])
def test_token_logprobs_vs_fp64(ops, V):
    lg, n_top = _kernel_rows(V, 0)
    B, cap, n_max = 8, 6, 20
    tok = torch.tensor([3, 9, 40, 90, V - 1, 8, 0, 17])
    dst = torch.tensor([0, 5, 2, 3, 1, 4, 0, 5], dtype=torch.int32)
    out_lp = torch.full((B, cap), float("nan"), device="cuda")
    out_ids = torch.full((B, cap, n_max), -7, dtype=torch.int64, device="cuda")
    out_top = torch.full((B, cap, n_max), float("nan"), device="cuda")
    lgd = lg.cuda()
    ops.token_logprobs(lgd, tok.cuda(), torch.tensor(n_top, dtype=torch.int32).cuda(), dst.cuda(), out_lp, out_ids, out_top)
    lp, ids, top = out_lp.cpu(), out_ids.cpu(), out_top.cpu()
    ref = torch.log_softmax(lg.double(), -1)
    for b in range(B):
        n, d = n_top[b], int(dst[b])
        others = [c for c in range(cap) if n < 0 or c != d]
        assert torch.isnan(lp[b, others]).all() and (ids[b, others] == -7).all() and torch.isnan(top[b, others]).all(), b
        if n < 0:
            continue
        assert abs(float(lp[b, d]) - float(ref[b, int(tok[b])])) < 1e-5, b
        want = torch.from_numpy(ranked(lg[b])[:n].copy())
        assert torch.equal(ids[b, d, :n], want), (b, ids[b, d, :n], want)
        assert float((top[b, d, :n].double() - ref[b, want]).abs().max() if n else 0.0) < 1e-5, b
        assert (ids[b, d, n:] == -7).all() and torch.isnan(top[b, d, n:]).all(), b
    assert torch.equal(ids[2, 2, :5], torch.tensor([3, 7, 40, V // 2, V - 1]))       # a tie goes to the lower index
    assert torch.equal(ids[3, 3, :5], torch.tensor([11, 12, 13, 50, 70]))
    assert torch.equal(ids[5, 4, 18:], torch.tensor([5, 8])) and int(ids[6, 0, 0]) == 2
    # the same row gives the same bits at every row position of an 8-row batch, whatever the others hold
    row = lg[3]
    outs = []
    for p in range(B):
        batch = torch.randn(B, V, generator=torch.Generator().manual_seed(100 + p)) * 3
        batch[p] = row
        o = (torch.zeros(B, 1, device="cuda"), torch.zeros(B, 1, n_max, dtype=torch.int64, device="cuda"),
             torch.zeros(B, 1, n_max, device="cuda"))
        nt = torch.full((B,), 20, dtype=torch.int32)
        ops.token_logprobs(batch.cuda(), torch.full((B,), 12, dtype=torch.int64).cuda(), nt.cuda(),
                           torch.zeros(B, dtype=torch.int32).cuda(), *o)
        outs.append(tuple(t[p].cpu() for t in o))
    for o in outs[1:]:
        for a, b_ in zip(outs[0], o):
            assert torch.equal(a, b_)


def test_token_logprobs_arguments(ops):
    lg = torch.randn(2, 100, device="cuda")
    tok = torch.zeros(2, dtype=torch.int64, device="cuda")
    n = torch.zeros(2, dtype=torch.int32, device="cuda")
    with pytest.raises(Exception):     # 21 alternatives > the kernel's 20
        ops.token_logprobs(lg, tok, n, n, torch.zeros(2, 3, device="cuda"), torch.zeros(2, 3, 21, dtype=torch.int64, device="cuda"),
                           torch.zeros(2, 3, 21, device="cuda"))
    with pytest.raises(ValueError):
        ops.record_scores(lg, 1.0, 0, 1.0, n[:1])


# ================================================================================================ 2. generate() vs HF
def hf_processed(logits, seq, T, k, p, penalty):
    """transformers' RepetitionPenalty -> Temperature -> TopK -> TopP on [B, V] fp32 CPU logits (HF adds the warpers only
    when sampling)."""
    from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    s = logits.clone()
    if penalty != 1.0:
        s = RepetitionPenaltyLogitsProcessor(penalty)(seq, s)
    if T > 0:
        s = TemperatureLogitsWarper(T)(seq, s)
        if k:
            s = TopKLogitsWarper(k)(seq, s)
        if p < 1.0:
            s = TopPLogitsWarper(p)(seq, s)
    return s


def ambiguous(s_pen, T, k, p, margin=1e-5):
    """[B] bool: the float64 cumulative mass below the maximum lies within `margin` of 1 - p (fp32 order can move the cut)."""
    if T <= 0 or p >= 1.0:
        return torch.zeros(s_pen.shape[0], dtype=torch.bool)
    x = s_pen.double() / T
    if k:
        x = x.masked_fill(x < x.topk(k, -1).values[:, -1:], -math.inf)
    c = torch.softmax(x, -1).sort(-1).values.cumsum(-1)[:, :-1]
    return ((c - (1.0 - p)).abs() < margin).any(-1)


GEN_CASES = [({}, 0), (dict(repetition_penalty=1.3), 0), (dict(do_sample=True, temperature=0.7, top_k=50), 11),
             (dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9), 12),
             (dict(do_sample=True, temperature=0.6, top_k=50, top_p=0.8, repetition_penalty=1.2), 13)]


def test_generate_scores_and_logits_match_hf():
    cfg, model = build()
    sharpen(model, cfg)
    ids = torch.randint(0, cfg.vocab_size, (2, 10), generator=torch.Generator().manual_seed(2)).cuda()
    B, S = ids.shape
    n = 12
    checked = amb = 0
    for settings, seed in GEN_CASES:
        def gen(**extra):
            kw = dict(settings, **extra)
            if kw.get("do_sample"):
                kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
            return model.generate(ids, max_new_tokens=n, return_dict_in_generate=True, **kw)

        out = gen(output_scores=True, output_logits=True)
        plain = gen()
        assert plain.scores is None and plain.logits is None
        assert torch.equal(out.sequences, plain.sequences), settings          # recording changes no token
        new = out.sequences.shape[1] - S
        assert len(out.scores) == len(out.logits) == new == n, settings
        eager = gen(output_scores=True, output_logits=True, use_graph=False)
        assert torch.equal(eager.sequences, out.sequences)
        for t in range(new):                                                    # graph == eager
            assert torch.equal(eager.scores[t], out.scores[t]) and torch.equal(eager.logits[t], out.logits[t]), (settings, t)
        T = settings.get("temperature", 0.0) if settings.get("do_sample") else 0.0
        k = settings.get("top_k", 50) if T > 0 else 0
        p = settings.get("top_p", 1.0) if T > 0 else 1.0
        pen = settings.get("repetition_penalty", 1.0)
        seqs = out.sequences.cpu()
        for t in range(new):
            lg, sc = out.logits[t].cpu(), out.scores[t].cpu()
            assert lg.shape == sc.shape == (B, cfg.vocab_size) and lg.dtype == torch.float32
            tok = seqs[:, S + t]
            want = hf_processed(lg, seqs[:, :S + t], T, k, p, pen)
            skip = ambiguous(hf_processed(lg, seqs[:, :S + t], 0.0, 0, 1.0, pen), T, k, p)
            for b in range(B):
                if skip[b]:
                    amb += 1
                    continue
                assert torch.equal(sc[b], want[b]), (settings, t, b)
                checked += 1
            assert torch.isfinite(sc.gather(1, tok[:, None])).all(), (settings, t)     # a picked token has a finite score
            if T == 0:
                assert torch.equal(sc.argmax(-1), tok), (settings, t)
            if T == 0 and pen == 1.0:
                assert torch.equal(sc, lg)
        # compute_transition_scores: a gather from log_softmax(scores)
        ts = model.compute_transition_scores(out.sequences, out.scores, normalize_logits=True)
        want = torch.stack([torch.log_softmax(out.scores[t], -1).gather(1, out.sequences[:, S + t:S + t + 1]).view(-1)
                            for t in range(new)], 1)
        assert ts.shape == (B, new) and torch.allclose(ts, want, atol=1e-6, rtol=0), settings
        raw = model.compute_transition_scores(out.sequences, out.scores)
        assert torch.equal(raw, torch.stack([out.scores[t].gather(1, out.sequences[:, S + t:S + t + 1]).view(-1)
                                             for t in range(new)], 1))
    assert amb <= 2 and checked >= len(GEN_CASES) * n * B - 2, (checked, amb)


def test_generate_scores_trimmed_to_eos_and_beams_unchanged():
    cfg, model = build()
    ids = torch.randint(0, cfg.vocab_size, (1, 10), generator=torch.Generator().manual_seed(4)).cuda()
    first = model.generate(ids, max_new_tokens=20)
    eos = int(first[0, 10 + 2])
    stop = first[0, 10:].tolist().index(eos) + 1
    out = model.generate(ids, max_new_tokens=20, eos_token_id=eos, return_dict_in_generate=True, output_scores=True,
                         output_logits=True)
    new = out.sequences.shape[1] - 10
    assert new == stop <= 3 and len(out.scores) == len(out.logits) == new   # the loop ran past the EOS; the tuples do not
    assert torch.equal(out.scores[-1].argmax(-1), out.sequences[:, -1])
    # beam search keeps its output: sequences_scores only
    beam = model.generate(ids, max_new_tokens=5, num_beams=2, return_dict_in_generate=True, output_scores=True)
    ref = model.generate(ids, max_new_tokens=5, num_beams=2, return_dict_in_generate=True, output_scores=True)
    assert beam.sequences_scores is not None and beam.scores is None and beam.logits is None
    assert torch.equal(beam.sequences, ref.sequences) and torch.equal(beam.sequences_scores, ref.sequences_scores)
    with pytest.raises(NotImplementedError):
        model.generate(ids, max_new_tokens=5, num_beams=2, return_dict_in_generate=True, output_logits=True)


# ================================================================================================ 3. one slot vs generate()
def _logprobs_of_logits(ops, logits, tokens, k):
    """uvx_token_logprobs over the rows of one request's logits [n, V] (row t = step t, index 0 of its own row)."""
    n = logits.shape[0]
    o = (torch.zeros(n, 1, device="cuda"), torch.zeros(n, 1, max(k, 1), dtype=torch.int64, device="cuda"),
         torch.zeros(n, 1, max(k, 1), device="cuda"))
    ops.token_logprobs(logits.contiguous(), tokens.contiguous(), torch.full((n,), k, dtype=torch.int32, device="cuda"),
                       torch.zeros(n, dtype=torch.int32, device="cuda"), *o)
    return o[0][:, 0], o[1][:, 0, :k], o[2][:, 0, :k]


def test_one_slot_logprobs_are_generate(ops):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    a = audio_request(cfg, 16000, 1)
    b = audio_request(cfg, 24000, 2)
    t = text_request(cfg, 11, 3)
    cases = [(a, 12, {}, 0), (b, 10, dict(do_sample=True, temperature=0.7, top_k=50), 11),
             (t, 9, dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9), 12), (a, 8, dict(repetition_penalty=1.3), 0),
             (b, 7, dict(do_sample=True, temperature=0.6, top_p=0.5, repetition_penalty=1.3), 13)]
    sched = SlotScheduler(model, slots=1, max_len=64, max_logprobs=5)
    plain = SlotScheduler(model, slots=1, max_len=64)
    for i, (feats, n, settings, seed) in enumerate(cases):
        k = i % 6                      # 0 .. 4 alternatives
        rid, = serve(sched, [(feats, n, dict(settings, logprobs=k), seed)])
        got = sched.run()[rid]
        p_rid, = serve(plain, [(feats, n, settings, seed)])
        assert torch.equal(got, plain.run()[p_rid]), settings
        kw = dict(settings)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
        out = model.generate(max_new_tokens=n, return_dict_in_generate=True, output_logits=True, **feats, **kw)
        assert torch.equal(got, out.sequences), settings
        S = feats["input_ids"].shape[1]
        lp = sched.logprobs[rid]
        assert lp.token_logprobs.shape == (n,) and lp.top_ids.shape == lp.top_logprobs.shape == (n, k)
        w_lp, w_ids, w_top = _logprobs_of_logits(ops, torch.cat(out.logits), out.sequences[0, S:], k)
        assert torch.equal(lp.token_logprobs, w_lp) and torch.equal(lp.top_ids, w_ids) and torch.equal(lp.top_logprobs, w_top), settings
    assert sched.engine.captures == 1 and sched.engine.launches_per_step == plain.engine.launches_per_step + 1


# ================================================================================================ 4. a busy engine
def _mixed_requests(cfg, n_req, seed, audio=True, long_at=None):
    settings = [{}, dict(do_sample=True, temperature=0.7, top_k=50), dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9),
                dict(repetition_penalty=1.3), dict(do_sample=True, temperature=0.8, top_p=0.6, repetition_penalty=1.2)]
    rng = np.random.default_rng(seed)
    reqs = []
    for i in range(n_req):
        if i == long_at:
            feats = text_request(cfg, 300, 900 + i)                          # > PREFILL_ROWS: prefilled in chunks
        elif audio and i % 3 == 0:
            feats = audio_request(cfg, int(rng.choice([8000, 16000, 30000])), 100 + i)
        else:
            feats = text_request(cfg, int(rng.integers(4, 30)), 200 + i)
        s = dict(settings[i % len(settings)])
        if i % 4 != 3:
            s["logprobs"] = i % 6                                              # some ask (0 .. 5 alternatives), some do not
        reqs.append((feats, int(rng.integers(2, 24)), s, 300 + i))
    return reqs


def _strip(reqs):
    return [(f, n, {k: v for k, v in s.items() if k != "logprobs"}, seed) for f, n, s, seed in reqs]


def _check_busy(model, reqs, eos, slots, max_len, alone=True, captures=1, **kw):
    """`captures`: the plain step's graph, plus the mixed step's when a prompt is prefilled in chunks."""
    from ultravox_b200.serving import SlotScheduler
    busy = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos, sync_every=3, max_logprobs=5, **kw)
    poison(busy)
    finished = []
    ids = serve(busy, reqs)
    res = busy.run(on_tokens=lambda rid, seq: finished.append((rid, rid in busy.logprobs)))
    assert busy.engine.captures == captures and len(finished) == len(reqs)
    asked = {rid for rid, r in zip(ids, reqs) if "logprobs" in r[2]}
    assert all(filled == (rid in asked) for rid, filled in finished)        # filled before on_tokens
    plain = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos, sync_every=3, **kw)
    p_ids = serve(plain, _strip(reqs))
    p_res = plain.run()
    stops = 0
    for (feats, n, s, _), rid, p_rid in zip(reqs, ids, p_ids):
        assert torch.equal(res[rid], p_res[p_rid]), rid                        # recording changes no token
        S = feats["input_ids"].shape[1]
        stops += res[rid].shape[1] < S + n
        if "logprobs" not in s:
            assert rid not in busy.logprobs
            continue
        lp = busy.logprobs[rid]
        assert lp.token_logprobs.shape[0] == res[rid].shape[1] - S, rid         # one entry per new token
        assert lp.top_ids.shape == (res[rid].shape[1] - S, s["logprobs"])
        assert bool(torch.isfinite(lp.token_logprobs).all()) and bool((lp.token_logprobs <= 0).all())
        if s["logprobs"]:
            assert bool((lp.top_logprobs[:, 0] >= lp.token_logprobs).all())
    assert stops >= 1
    eager = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos, sync_every=3, max_logprobs=5, use_graph=False,
                          **kw)
    e_ids = serve(eager, reqs)
    e_res = eager.run()
    assert eager.engine.captures == 0
    for rid, e_rid in zip(ids, e_ids):
        assert torch.equal(res[rid], e_res[e_rid]), rid
        if rid in busy.logprobs:
            a, b = busy.logprobs[rid], eager.logprobs[e_rid]
            assert all(torch.equal(x, y) for x, y in zip((a.token_logprobs, a.top_ids, a.top_logprobs),
                                                         (b.token_logprobs, b.top_ids, b.top_logprobs))), rid
    if alone:
        one = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos, max_logprobs=5, **kw)
        for rid, r in zip(ids, reqs):
            if rid not in busy.logprobs:
                continue
            poison(one)
            o_rid, = serve(one, [r])
            assert torch.equal(one.run()[o_rid], res[rid])
            a, b = busy.logprobs[rid], one.logprobs[o_rid]
            assert torch.equal(a.token_logprobs, b.token_logprobs) and torch.equal(a.top_ids, b.top_ids) and \
                torch.equal(a.top_logprobs, b.top_logprobs), rid
        assert one.engine.captures == captures
    return busy, ids, res


def _eos(model, reqs):
    first = model.generate(**reqs[0][0], max_new_tokens=24)
    return [int(first[0, reqs[0][0]["input_ids"].shape[1] + 4])]


def test_busy_engine_logprobs():
    cfg, model = build()
    reqs = _mixed_requests(cfg, 20, 0)
    _check_busy(model, reqs, _eos(model, reqs), 8, 256)


def test_busy_engine_logprobs_chunked_prompt():
    cfg, model = build()
    reqs = _mixed_requests(cfg, 12, 1, long_at=4)
    _check_busy(model, reqs, _eos(model, reqs), 8, 384, captures=2)


def test_busy_paged_engine_logprobs_prefix_hit():
    cfg, model = build()
    g = torch.Generator().manual_seed(77)
    system = torch.randint(0, 1000, (1, 128), generator=g).cuda()
    reqs = _mixed_requests(cfg, 10, 2, audio=False)
    # requests 2 and 6 open with the same 128-token system prompt: the later one takes its two pages from the cache
    for i in (2, 6):
        f, n, s, seed = reqs[i]
        reqs[i] = (dict(input_ids=torch.cat([system, f["input_ids"]], 1)), n, dict(s, logprobs=3), seed)
    busy, ids, res = _check_busy(model, reqs, _eos(model, reqs), 8, 256, alone=False, kv_pages=64, prefix_cache=True)
    assert busy.cached_tokens[ids[6]] == 128 and busy.cached_tokens[ids[2]] == 0


# ================================================================================================ 5. 8B widths
def test_logprobs_at_8b_widths():
    """Two layers at Llama-3.1-8B widths, V = 128256, 8 slots, logprobs = 20: each request's log-probs against the fp64
    log-softmax of its own generate(output_logits=True) logits, as far as their tokens agree (8 slots run the GEMM, one stream
    the GEMV, so the bf16 rounding of the two differs)."""
    from ultravox_b200.config import PRESETS
    from ultravox_b200.serving import SlotScheduler
    base = PRESETS["v0_5_8b"]
    cfg, model = build("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                       text_config=dict(base["text_config"], num_hidden_layers=2))
    sharpen(model, cfg)
    reqs = [(text_request(cfg, 6 + 3 * i, 500 + i), 5, dict(logprobs=20), 0) for i in range(8)]
    sched = SlotScheduler(model, slots=8, max_len=64, max_logprobs=20)
    ids = serve(sched, reqs)
    res = sched.run()
    compared = 0
    for rid, (feats, n, _, _) in zip(ids, reqs):
        S = feats["input_ids"].shape[1]
        lp = sched.logprobs[rid]
        assert lp.top_ids.shape == (n, 20)
        out = model.generate(max_new_tokens=n, return_dict_in_generate=True, output_logits=True, **feats)
        for t in range(n):
            if int(out.sequences[0, S + t]) != int(res[rid][0, S + t]):
                break
            ref = torch.log_softmax(out.logits[t][0].double(), -1)
            assert abs(float(lp.token_logprobs[t]) - float(ref[int(res[rid][0, S + t])])) < 0.1, (rid, t)
            assert float((lp.top_logprobs[t].double() - ref[lp.top_ids[t]]).abs().max()) < 0.1, (rid, t)
            r = ranked(out.logits[t][0])[:21]
            gaps = ref[r[:-1]] - ref[r[1:]]
            for i in range(20):            # ids that fp64 separates from both neighbours by a clear gap sit at the same rank
                if gaps[i] > 0.25 and (i == 0 or gaps[i - 1] > 0.25):
                    assert int(lp.top_ids[t, i]) == int(r[i]), (rid, t, i)
            compared += 1
        assert bool(torch.isfinite(lp.token_logprobs).all())
    assert compared >= 20, compared


# ================================================================================================ 6. validation
def test_logprobs_validation():
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    t = text_request(cfg, 10, 1)
    for bad in (21, -1, 1.5, "3", True):
        with pytest.raises(ValueError):
            SlotScheduler(model, slots=2, max_len=32, max_logprobs=bad)
    sched = SlotScheduler(model, slots=2, max_len=32, max_logprobs=3)
    for bad in (4, -1, 2.0, "1", True):
        with pytest.raises(ValueError):
            sched.submit(t, max_new_tokens=4, logprobs=bad)
    plain = SlotScheduler(model, slots=2, max_len=32)
    with pytest.raises(ValueError):
        plain.submit(t, max_new_tokens=4, logprobs=0)
    assert sched.pending() == [] and plain.pending() == []
    rid = sched.submit(t, max_new_tokens=6, logprobs=0)
    rid2 = sched.submit(t, max_new_tokens=6)
    res = sched.run()
    assert torch.equal(res[rid], model.generate(**t, max_new_tokens=6)) and torch.equal(res[rid2], res[rid])
    assert sched.logprobs[rid].top_ids.shape == (6, 0) and rid2 not in sched.logprobs
    # a default scheduler and a default generate() engine keep their step
    assert plain.engine.launches_per_step == sched.engine.launches_per_step - 1
