"""Beam search: uvx_log_softmax / uvx_beam_select / uvx_beam_update / uvx_kv_reorder, engine.BeamDecodeEngine and
generate(num_beams=...), against transformers' own ``_beam_search``.

The oracle replays our numbers through HF: random-init models are nearly tied, so comparing bf16 and fp32 end-to-end
sequences would test rounding, not the search.  Our engine is stepped eagerly and records every step's processed log-probs
and running sequences; a tiny ``LlamaForCausalLM`` on the CPU then runs ``generate(num_beams=...)`` with a logits processor
that checks the running sequences HF hands it (order and reorder of the histories) and returns our log-probs.  The returned
sequences must be identical and the scores equal to fp32 rounding.  A step whose top-K cut falls inside a group of exactly
equal values is ambiguous (torch.topk orders ties arbitrarily); such cases are counted and skipped, and must be few."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(name="micro", enc_layers=None, llm_layers=None, logit_std=3.0):
    """Seeded random model whose lm_head is rescaled so the logits have std `logit_std` (peaked enough for EOS ids to win)."""
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    kw = {}
    if enc_layers is not None:
        kw = dict(audio_config=dict(PRESETS[name]["audio_config"], encoder_layers=enc_layers),
                  text_config=dict(PRESETS[name]["text_config"], num_hidden_layers=llm_layers))
    cfg = preset(name, **kw)
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, min(cfg.vocab_size, 128000), (1, 12), generator=g).cuda()
    std = float(model(ids, logits_to_keep=1).logits.float().std())
    model.language_model.lm_head.weight.data.mul_(logit_std / std)
    return cfg, model


def _prompts(V, B, S, seed, pad=True):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, min(V, 128000), (B, S), generator=g)
    am = torch.ones(B, S, dtype=torch.long)
    if pad and B > 1:
        for b in range(1, B):
            am[b, :2 + 2 * b] = 0
            ids[b, :2 + 2 * b] = 0
    return ids, am


def _run_ours(model, ids, am, nb, eos, lp, es, nrs, pen, max_new, pad_id, use_graph=False, hook=None):
    """model._beam_search as generate calls it, with a per-step recorder: returns (sequences, scores, records) where
    records[t] = (processed log-probs of step t, running sequences after step t, running scores after step t)."""
    dev = torch.device("cuda")
    ids_d = ids.to(dev)
    kv_start = position_ids = None
    amd = None
    if am is not None and not bool(am.bool().all()):
        amd = am.to(dev)
        kv_start, _ = model._pad_bounds(amd)
        position_ids = (amd.cumsum(-1) - 1).clamp_min(0)
    rec = []

    def step_hook(eng):
        torch.cuda.synchronize()
        rec.append((eng.logprobs.cpu().clone(), eng.seq[:, :int(eng.cur_len)].cpu().clone(), eng.run_score.cpu().clone()))
        if hook is not None:
            hook(eng)

    fk = dict(audio_values=None, inputs_embeds=None, attention_mask=amd, audio_token_start_idx=None, audio_lens=None,
              audio_token_len=None, audio_batch_size=None, position_ids=position_ids, audio_waveforms=None,
              audio_num_frames=None, audio_pad_frames=None)
    seqs, scores = model._beam_search(ids_d, fk, kv_start, max_new, eos, pad_id, nb, lp, es, nrs, pen, use_graph,
                                      step_hook=step_hook)
    return seqs.cpu(), scores.cpu(), rec


def _tie_at_cut(rec, B, nb, K, V):
    """Number of steps whose top-K (over lp + running score) has an exact tie across the cut."""
    n = 0
    for t, (lp, _, _) in enumerate(rec):
        if t == 0:
            sc = torch.full((B, nb), -1e9)
            sc[:, 0] = 0.0
            sc = sc.view(-1)
        else:
            sc = rec[t - 1][2]
        a = (lp + sc[:, None]).view(B, nb * V)
        v = a.topk(K + 1, -1).values
        n += int((v[:, K - 1] == v[:, K]).any())
    return n


class _Replay:
    def __init__(self, first_ids, rec):
        self.seqs = [first_ids] + [r[1] for r in rec[:-1]]
        self.lps = [r[0] for r in rec]
        self.t = 0

    def __call__(self, input_ids, scores):
        t = self.t
        self.t += 1
        assert t < len(self.lps), "HF ran more beam steps than the engine"
        assert torch.equal(input_ids, self.seqs[t]), f"running sequences differ at step {t}"
        return self.lps[t].clone()


def _hf(V, ids, am, nb, eos, lp, es, nrs, max_new, pad_id, replay):
    from transformers import LlamaConfig, LlamaForCausalLM
    from transformers.generation.logits_process import LogitsProcessor, LogitsProcessorList

    class Replay(LogitsProcessor):
        def __call__(self, input_ids, scores):
            return replay(input_ids, scores)

    torch.manual_seed(0)
    hf = LlamaForCausalLM(LlamaConfig(vocab_size=V, hidden_size=16, intermediate_size=32, num_hidden_layers=1,
                                      num_attention_heads=2, num_key_value_heads=1, max_position_embeddings=8192,
                                      bos_token_id=None, eos_token_id=None, pad_token_id=None)).eval()
    hf.generation_config.eos_token_id = None
    hf.generation_config.bos_token_id = None
    hf.generation_config.pad_token_id = None
    with torch.no_grad():
        return hf.generate(ids, attention_mask=am, num_beams=nb, length_penalty=lp, early_stopping=es, num_return_sequences=nrs,
                           eos_token_id=eos if eos else None, pad_token_id=pad_id, max_new_tokens=max_new, do_sample=False,
                           output_scores=True, return_dict_in_generate=True, logits_processor=LogitsProcessorList([Replay()]))


def _replay_case(model, V, ids, am, nb, eos, lp, es, nrs, pen, max_new, pad_id):
    """-> (ambiguous, steps, ended early).  Asserts HF == ours when the case is not ambiguous."""
    B = ids.shape[0]
    K = max(2, 1 + len(eos)) * nb
    seqs, scores, rec = _run_ours(model, ids, am, nb, eos, lp, es, nrs, pen, max_new, pad_id)
    if _tie_at_cut(rec, B, nb, K, V):
        return True, len(rec), len(rec) < max_new
    replay = _Replay(ids.repeat_interleave(nb, 0), rec)
    out = _hf(V, ids, am, nb, eos, lp, es, nrs, max_new, pad_id, replay)
    case = (nb, B, eos, lp, es, nrs, pen)
    assert replay.t == len(rec), (case, replay.t, len(rec))
    assert torch.equal(out.sequences, seqs), (case, out.sequences, seqs)
    torch.testing.assert_close(out.sequences_scores, scores, rtol=1e-6, atol=0.0, msg=lambda m: f"{case}: {m}")
    # the generate() entry point (graph replay, done flag polled every few steps) returns the same
    g = model.generate(ids.cuda(), attention_mask=am.cuda(), num_beams=nb, length_penalty=lp, early_stopping=es,
                       num_return_sequences=nrs, eos_token_id=eos or None, pad_token_id=pad_id, max_new_tokens=max_new,
                       repetition_penalty=pen, return_dict_in_generate=True, output_scores=True)
    assert torch.equal(g.sequences.cpu(), seqs) and torch.equal(g.sequences_scores.cpu(), scores), case
    assert g.past_key_values is None
    return False, len(rec), len(rec) < max_new


def _greedy_eos(model, ids, am, steps=(2, 3, 4)):
    out = model.generate(ids.cuda(), attention_mask=am.cuda(), max_new_tokens=max(steps) + 1).cpu()
    S = ids.shape[1]
    toks = []
    for s in steps:
        t = int(out[0, S + s])
        if t not in toks:
            toks.append(t)
    return toks


def test_hf_replay_micro():
    cfg, model = _model()
    V = cfg.vocab_size
    max_new = 12
    ids1, am1 = _prompts(V, 1, 10, 1)
    ids3, am3 = _prompts(V, 3, 10, 2)
    eos_pool = {1: _greedy_eos(model, ids1, am1), 3: _greedy_eos(model, ids3, am3)}
    lps, ess = (1.0, 0.0, -0.5, 2.0), (False, True, "never")
    amb = early = full = n = 0
    i = 0
    for lp in lps:
        for es in ess:
            for nb in (2, 4, 8):
                B = (1, 3)[(i + nb) % 2]
                ids, am = (ids1, am1) if B == 1 else (ids3, am3)
                n_eos = (0, 1, 3)[i % 3]
                eos = eos_pool[B][:n_eos]
                nrs = (1, nb)[i % 2]
                pen = (1.0, 1.3)[(i // 2) % 2]
                if max(2, 1 + len(eos)) * nb > 64:
                    eos = eos[:1]
                a, steps, e = _replay_case(model, V, ids, am, nb, eos, lp, es, nrs, pen, max_new, pad_id=0)
                amb += a
                n += 1
                early += e and not a
                full += (not e) and not a
                i += 1
    print(f"replay cases {n}, ambiguous {amb}, ended by EOS + heuristic {early}, by max_new_tokens {full}")
    assert amb <= n // 10, (amb, n)
    assert early >= 1 and full >= 1, (early, full)


def test_processed_logprobs_are_hf_processors():
    """The recorded log-probs are log_softmax(logits) then HF's RepetitionPenaltyLogitsProcessor over each running beam."""
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor
    cfg, model = _model()
    ids, am = _prompts(cfg.vocab_size, 1, 10, 3)
    got = []

    def hook(eng):
        got.append((eng.logits.float().cpu(), eng.logprobs.cpu()))

    prev = [ids.repeat_interleave(4, 0)]
    _, _, rec = _run_ours(model, ids, am, 4, [], 1.0, False, 1, 1.3, 6, 0, hook=hook)
    for t, (logits, lp) in enumerate(got):
        seq = prev[0] if t == 0 else rec[t - 1][1]
        ref = RepetitionPenaltyLogitsProcessor(1.3)(seq, torch.log_softmax(logits, -1))
        torch.testing.assert_close(lp, ref, rtol=0, atol=2e-5)


def test_select_kernels_full_vocab():
    """uvx_beam_select at V = 128256, nb = 4 with the Llama-3 EOS triple (K = 16): the exact top K of lp + score per prompt,
    and uvx_beam_update driven through HF's own helpers over several steps (ours and HF's state compared every step)."""
    from transformers import GenerationMixin
    from ultravox_b200 import ops
    V, B, nb, K = 128256, 2, 4, 16
    g = torch.Generator().manual_seed(0)
    for trial in range(3):
        lp = torch.log_softmax(torch.randn(B * nb, V, generator=g) * 3, -1)
        sc = -torch.rand(B * nb, generator=g) * 10
        s, i = ops.beam_select(lp.cuda(), sc.cuda(), nb, K)
        ref = (lp + sc[:, None]).view(B, nb * V).topk(K, -1)
        assert torch.equal(s.cpu(), ref.values) and torch.equal(i.cpu(), ref.indices)
    # every row -1e9 but one: the tie rule takes the lowest flat indices
    lp = torch.log_softmax(torch.randn(B * nb, V, generator=g), -1)
    sc = torch.full((B * nb,), -1e9)
    s, i = ops.beam_select(lp.cuda(), sc.cuda(), nb, K)
    assert torch.equal(i.cpu(), torch.arange(K).expand(B, K)) and bool((s == -1e9).all())

    # the update kernel against HF's helpers, step by step on synthetic log-probs
    eos = torch.tensor([128001, 128008, 128009])
    S, max_new = 5, 6
    hf = GenerationMixin
    dev = torch.device("cuda")
    for lpen, es in ((1.0, False), (2.0, "never"), (-0.5, True)):
        st = dict(run_score=torch.zeros(B * nb, device=dev), run_seq=torch.zeros(B * nb, S + max_new + 1, dtype=torch.int64, device=dev),
                  pool_score=torch.full((B * nb,), -1e9, device=dev), pool_len=torch.zeros(B * nb, dtype=torch.int32, device=dev),
                  pool_fin=torch.zeros(B * nb, dtype=torch.int32, device=dev), parent=torch.zeros(B * nb, dtype=torch.int32, device=dev),
                  tok=torch.zeros(B * nb, dtype=torch.int64, device=dev), heur=torch.ones(B, dtype=torch.int32, device=dev),
                  flags=torch.zeros(B, dtype=torch.int32, device=dev), ticket=torch.zeros(1, dtype=torch.int32, device=dev))
        st["pool_seq"] = torch.zeros_like(st["run_seq"])
        st["run_score"].view(B, nb)[:, 1:] = -1e9
        cnt = dict(cur_len=torch.full((1,), S, dtype=torch.int32, device=dev), step_idx=torch.zeros(1, dtype=torch.int32, device=dev),
                   done=torch.zeros(1, dtype=torch.int32, device=dev))
        len_div = torch.tensor([1.0] + [float(n) ** lpen for n in range(1, 64)], dtype=torch.float32, device=dev)
        prompt = torch.randint(0, 1000, (B, S), generator=g)
        st["run_seq"][:, :S] = prompt.repeat_interleave(nb, 0).to(dev)
        st["pool_seq"][:, :S] = prompt.repeat_interleave(nb, 0).to(dev)
        # HF state
        L = S + max_new
        r_seq = torch.zeros(B, nb, L, dtype=torch.int64)
        r_seq[:, :, :S] = prompt[:, None]
        seqs = r_seq.clone()
        r_sc = torch.zeros(B, nb)
        r_sc[:, 1:] = -1e9
        b_sc = torch.full((B, nb), -1e9)
        fin = torch.zeros(B, nb, dtype=torch.bool)
        heur = torch.ones(B, 1, dtype=torch.bool)
        r_bi = torch.full((B, nb, L - S), -1, dtype=torch.int32)
        b_bi = r_bi.clone()
        mask = torch.cat([torch.ones(nb, dtype=torch.bool), torch.zeros(K - nb, dtype=torch.bool)])
        for t in range(max_new):
            cur = S + t
            lp = torch.log_softmax(torch.randn(B * nb, V, generator=g) * 4, -1)
            lp[:, eos] += 4.0 * (t % 2)                                 # EOS wins some candidates every other step
            s, i = ops.beam_select(lp.cuda(), st["run_score"], nb, K)
            ops.beam_update(s, i, V, nb, eos.cuda(), max_new, len_div, {False: 0, True: 1, "never": 2}[es], lpen > 0, st, cnt)
            acc = (lp.view(B, nb, V) + r_sc[:, :, None]).view(B, nb * V)
            tlp, tseq, tbi = hf._get_top_k_continuations(hf, acc, r_seq, r_bi, cur, S, False, K, nb, V, B)
            hits = torch.isin(tseq[:, :, cur], eos) | (cur + 1 >= L)
            r_seq, r_sc, r_bi = hf._get_running_beams_for_next_iteration(hf, tlp, tseq, tbi, hits, nb)
            seqs, b_sc, b_bi, fin = hf._update_finished_beams(hf, seqs, tseq, b_sc, tlp, b_bi, tbi, heur, fin, hits, mask, nb, cur, S,
                                                             lpen, es)
            heur = hf._check_early_stop_heuristic(heur, r_sc, b_sc, fin, cur + 1, L, S, es, lpen)
            go = bool(hf._beam_search_has_unfinished_sequences(heur, fin, hits, es))
            torch.cuda.synchronize()
            if not bool(hits.all()):        # else every running score is -1e9 + x: tied, and the search ends here
                assert torch.equal(st["run_seq"][:, :cur + 1].cpu(), r_seq.view(B * nb, L)[:, :cur + 1]), (lpen, es, t)
                assert torch.equal(st["run_score"].cpu(), r_sc.view(-1)), (lpen, es, t)
            assert torch.equal(st["pool_score"].cpu(), b_sc.view(-1)), (lpen, es, t)
            real = b_sc.view(-1) > -1e8         # entries at -1e9 tie with each other and are never returned
            assert torch.equal(st["pool_fin"].cpu().bool()[real], fin.view(-1)[real]), (lpen, es, t)
            assert torch.equal(st["pool_len"].cpu()[real], (b_bi.view(B * nb, -1) >= 0).sum(-1).int()[real]), (lpen, es, t)
            assert torch.equal(st["pool_seq"][real, :cur + 1].cpu(), seqs.view(B * nb, L)[real, :cur + 1]), (lpen, es, t)
            assert torch.equal(st["heur"].cpu().bool(), heur.view(-1)), (lpen, es, t)
            assert int(cnt["done"]) == int(not go), (lpen, es, t)
            assert int(cnt["cur_len"]) == cur + 1
            if not go:
                break


def _reorder_check(L, B, nb, smax, hkv, d, n_pos, parents):
    from ultravox_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    shape = (L, B * nb, smax, hkv, d)
    k0 = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    v0 = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    for par in parents:
        k, v = k0.clone(), v0.clone()
        p = torch.tensor(par, dtype=torch.int32, device="cuda")
        ops.kv_reorder_(k, v, p, torch.tensor([n_pos], dtype=torch.int32, device="cuda"), nb)
        ek, ev = k0.clone(), v0.clone()
        ek[:, :, :n_pos] = k0[:, :, :n_pos].index_select(1, p.long())
        ev[:, :, :n_pos] = v0[:, :, :n_pos].index_select(1, p.long())
        assert torch.equal(k, ek) and torch.equal(v, ev), par


def _maps(B, nb):
    base = [
        list(range(nb)),                                    # identity
        [0] * nb,                                           # broadcast / all duplicates of one
        [1, 0] + list(range(2, nb)),                        # a swap
        ([1, 2, 0] + list(range(3, nb))) if nb >= 3 else [1, 0],   # a 3-cycle
        [(j + 1) % nb for j in range(nb)],                  # everyone re-parented
        [nb - 1 - j if j % 2 else j // 2 for j in range(nb)],     # duplicates mixed with moves
    ]
    return [[b * nb + m[(j + b) % nb if i == 5 else j] for b in range(B) for j in range(nb)] for i, m in enumerate(base)]


def test_kv_reorder_micro():
    for nb in (2, 4, 8):
        _reorder_check(2, 3, nb, 64, 2, 64, 37, _maps(3, nb))


def test_kv_reorder_8b_widths():
    _reorder_check(32, 1, 4, 4096, 8, 128, 3001, _maps(1, 4)[1:5])


def test_engine_cache_matches_cacheless_reforward():
    """Every step, each running beam's logits equal a cacheless forward of that beam's running sequence."""
    from ultravox_b200 import ops
    cfg, model = _model()
    lm = model.language_model
    ids, am = _prompts(cfg.vocab_size, 1, 10, 5)
    prev = [ids.repeat_interleave(4, 0)]
    worst = [0.0, 0]

    def hook(eng):
        seq = prev[-1].cuda()
        for r in range(seq.shape[0]):
            emb = ops.embed_splice(seq[r:r + 1], lm.model.embed_tokens.weight, None, None)
            ref = ops.lm_head(model.llama_hidden(emb)[:, -1, :], lm.lm_head.weight)[0]
            got = eng.logits[r]
            worst[0] = max(worst[0], float((got - ref).abs().max() / ref.std()))
            worst[1] += int(int(got.argmax()) != int(ref.argmax()))
        prev.append(eng.seq[:, :int(eng.cur_len)].cpu().clone())

    _run_ours(model, ids, am, 4, [], 1.0, False, 1, 1.0, 10, 0, hook=hook)
    print(f"cache vs cacheless: max |diff| / std {worst[0]:.3e}, argmax mismatches {worst[1]}")
    assert worst[1] == 0 and worst[0] < 1e-3, worst


def test_graph_equals_eager_and_cache_tail():
    cfg, model = _model()
    ids, am = _prompts(cfg.vocab_size, 3, 10, 6)
    kw = dict(attention_mask=am.cuda(), num_beams=4, num_return_sequences=2, max_new_tokens=10, repetition_penalty=1.3,
              length_penalty=0.5, return_dict_in_generate=True, output_scores=True)
    a = model.generate(ids.cuda(), use_graph=True, **kw)
    b = model.generate(ids.cuda(), use_graph=False, **kw)
    assert torch.equal(a.sequences, b.sequences) and torch.equal(a.sequences_scores, b.sequences_scores)
    orig = model.new_cache
    runs = []
    for fill in (0.0, float("nan")):
        def poisoned(batch, max_len, fill=fill):
            c = orig(batch, max_len)
            c.k.fill_(fill)
            c.v.fill_(fill)
            return c
        model.new_cache = poisoned
        try:
            runs.append(model.generate(ids.cuda(), **kw))
        finally:
            del model.new_cache
    for r in runs:
        assert torch.equal(r.sequences, a.sequences) and torch.equal(r.sequences_scores, a.sequences_scores)


def test_num_beams_one_is_todays_generate():
    cfg, model = _model()
    ids, am = _prompts(cfg.vocab_size, 2, 10, 7)
    kw = dict(attention_mask=am.cuda(), max_new_tokens=10)
    assert torch.equal(model.generate(ids.cuda(), num_beams=1, **kw), model.generate(ids.cuda(), **kw))
    s = dict(do_sample=True, temperature=0.7, top_k=20, **kw)
    g1 = model.generate(ids.cuda(), num_beams=1, generator=torch.Generator(device="cuda").manual_seed(3), **s)
    g2 = model.generate(ids.cuda(), generator=torch.Generator(device="cuda").manual_seed(3), **s)
    assert torch.equal(g1, g2)


def test_beam_with_audio():
    """A mel-spectrogram prompt: beam search runs end to end and graph replay equals eager steps."""
    import numpy as np
    from oracle import logmel as olog
    from ultravox_b200 import ops
    cfg, model = _model()
    wave = np.random.default_rng(3).standard_normal(16000).astype(np.float32)
    padded, frames = olog.pad_batch([wave])
    n_tok = int(-(-int(frames[0]) // 16))
    g = torch.Generator().manual_seed(8)
    ids = torch.cat([torch.randint(0, cfg.vocab_size, (6,), generator=g), torch.full((n_tok,), 3),
                     torch.randint(0, cfg.vocab_size, (4,), generator=g)])[None].cuda()
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    kw = dict(audio_values=mel, audio_token_start_idx=torch.tensor([6]).cuda(), audio_lens=torch.tensor([int(frames[0])]).cuda(),
              audio_token_len=torch.tensor([n_tok], dtype=torch.int32).cuda(), audio_batch_size=torch.tensor([1]).cuda(),
              num_beams=3, max_new_tokens=6)
    a = model.generate(ids, **kw)
    assert a.shape == (1, ids.shape[1] + 6) and torch.equal(a[:, :ids.shape[1]], ids)
    assert torch.equal(model.generate(ids, use_graph=False, **kw), a)


def test_hf_replay_8b_widths():
    """Llama-3.1-8B widths (V = 128256), 2 layers, B = 2 left-padded, nb = 4, the Llama-3 EOS triple."""
    cfg, model = _model("v0_5_8b", enc_layers=1, llm_layers=2)
    V = cfg.vocab_size
    ids, am = _prompts(V, 2, 12, 11)
    eos = [128001, 128008, 128009]
    amb, steps, _ = _replay_case(model, V, ids, am, 4, eos, 1.0, False, 2, 1.0, 6, pad_id=128009)
    assert not amb and steps >= 1
    kw = dict(attention_mask=am.cuda(), num_beams=4, num_return_sequences=2, max_new_tokens=6, eos_token_id=eos,
              return_dict_in_generate=True, output_scores=True)
    a = model.generate(ids.cuda(), use_graph=True, **kw)
    b = model.generate(ids.cuda(), use_graph=False, **kw)
    assert torch.equal(a.sequences, b.sequences) and torch.equal(a.sequences_scores, b.sequences_scores)


def test_beam_argument_errors():
    cfg, model = _model()
    ids = torch.randint(0, cfg.vocab_size, (1, 8), generator=torch.Generator().manual_seed(1)).cuda()
    for bad in (0, -1, 9):
        with pytest.raises(ValueError):
            model.generate(ids, num_beams=bad, max_new_tokens=2)
    with pytest.raises(ValueError):
        model.generate(ids, num_beams=2, num_return_sequences=3, max_new_tokens=2)
    with pytest.raises(NotImplementedError):
        model.generate(ids, num_beams=2, do_sample=True, max_new_tokens=2)

    class Streamer:
        def put(self, x):
            pass

        def end(self):
            pass

    with pytest.raises(ValueError, match="`streamer` cannot be used with beam search"):
        model.generate(ids, num_beams=2, streamer=Streamer(), max_new_tokens=2)
    cache = model.generate(ids, max_new_tokens=2, return_dict_in_generate=True).past_key_values
    with pytest.raises(NotImplementedError):
        model.generate(torch.cat([ids, ids], 1), num_beams=2, past_key_values=cache, max_new_tokens=2)
    with pytest.raises(ValueError):
        model.generate(ids, num_beams=2, early_stopping="sometimes", max_new_tokens=2)
