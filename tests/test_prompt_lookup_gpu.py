"""Prompt lookup decoding in the graph-captured decode step.

Kernels bit for bit: uvx_lookup_draft against transformers' PromptLookupCandidateGenerator.get_candidates (no logits
processors) plus the budget cap, uvx_lookup_accept against HF's n_matches, the per-row penalty / record forms against the
existing kernels row by row.  generate(prompt_lookup_num_tokens=...) against generate() without it, with the decode linears
on the same decode-form GEMM (engine.GEMV_MAX_B = 0): tokens, scores, logits, caches and the per-step accepted-draft log."""
import pytest
import torch

pytestmark = pytest.mark.gpu

V8B = 128256


# ------------------------------------------------------------------------------------------------ host references
def hf_drafts(seq, k, n, eos, max_length, max_new, n_new):
    """HF's candidates for seq (list of ids) with logits_processor=None, then the budget cap n_new + d + 1 <= max_new."""
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor(list(eos), dtype=torch.int64), num_output_tokens=k,
                                         max_matching_ngram_size=n, max_length=max_length)
    ids = torch.tensor([seq], dtype=torch.int64)
    out, _ = gen.get_candidates(ids)
    d = out[0, len(seq):].tolist()
    return d[:max(0, max_new - n_new - 1)]


def hf_n_matches(drafts, picks):
    """hf:generation/utils.py _assisted_decoding: ((~(candidates == selected[:, :-1])).cumsum(-1) < 1).sum()."""
    c = torch.tensor([drafts], dtype=torch.int64)
    s = torch.tensor([picks], dtype=torch.int64)
    return int(((~(c == s[:, :c.shape[1]])).cumsum(dim=-1) < 1).sum())


def replay_log(tokens, S, k, n, eos, max_new):
    """The accepted-draft counts a lookup run must log for the plain run's tokens (prompt + new, a list)."""
    log, cur, n_new = [], S + 1, 1
    while n_new < max_new and tokens[cur - 1] not in eos:
        d = hf_drafts(tokens[:cur], k, n, eos, S + max_new, max_new, n_new)
        m = 0
        while m < len(d) and cur + m < len(tokens) and tokens[cur + m] == d[m]:
            m += 1
        log.append(m)
        cur += m + 1
        n_new += m + 1
    return log


# ------------------------------------------------------------------------------------------------ kernels
def _draft(ops, seq_list, S, max_new, k, n, eos, cap=None, done=0):
    L = len(seq_list)
    W = (cap or S + max_new + k) + 1
    dev = "cuda"
    seq = torch.full((W,), -7, dtype=torch.int64, device=dev)
    seq[:L] = torch.tensor(seq_list, dtype=torch.int64)
    i32 = dict(dtype=torch.int32, device=dev)
    cur, nn, dn = torch.tensor([L], **i32), torch.tensor([L - S], **i32), torch.tensor([done], **i32)
    tok = torch.zeros(k + 1, dtype=torch.int64, device=dev)
    nd = torch.zeros(1, **i32)
    rows = [torch.full((k + 1,), -1, **i32) for _ in range(5)]
    e = torch.tensor(eos, dtype=torch.int64, device=dev) if eos else None
    ops.lookup_draft(seq, cur, nn, max_new, k, n, e, dn, tok, nd, *rows)
    return seq.cpu(), tok.cpu(), int(nd), [r.cpu() for r in rows]


def _check_draft(ops, seq_list, S, max_new, k, n, eos, cap=None, expect=None):
    L = len(seq_list)
    want = hf_drafts(seq_list, k, n, eos, S + max_new, max_new, L - S)
    if expect is not None:
        assert want == expect
    seq, tok, d, (pos, lens, rope, pen, idx) = _draft(ops, seq_list, S, max_new, k, n, eos, cap)
    assert d == len(want), (L, k, n, d, want)
    assert seq[L:L + d].tolist() == want and seq[:L].tolist() == seq_list
    assert tok[0] == seq_list[-1] and tok[1:d + 1].tolist() == want and (tok[d + 1:] == seq_list[-1]).all()
    i = torch.arange(k + 1, dtype=torch.int32)
    assert torch.equal(pos, L - 1 + i) and torch.equal(rope, L - 1 + i)
    assert torch.equal(lens, L + i) and torch.equal(pen, L + i) and torch.equal(idx, (L - S) + i)
    return d


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("k", [1, 4, 10, 31])
@pytest.mark.parametrize("n_eos", [0, 1, 3])
def test_lookup_draft_matches_hf(ops, k, n, n_eos):
    """Random sequences over a vocabulary of 6 (matches everywhere), lengths 1 .. 40000, against get_candidates + the cap."""
    g = torch.Generator().manual_seed(100 * k + 10 * n + n_eos)
    eos = list(range(n_eos))
    found = 0
    for L in (1, 2, 3, 5, 9, 33, 200, 1500, 40000):
        seq = torch.randint(0, 6, (L,), generator=g).tolist()
        for S, max_new in ((max(1, L - 3), 40), (1, L + 5), (max(1, L - 1), 2), (max(1, L - 2), 3)):
            if L - S >= max_new:
                continue
            found += _check_draft(ops, seq, S, max_new, k, n, eos) > 0
    assert found > 0


def test_lookup_draft_edge_cases(ops):
    k = 5
    # no match: every token distinct
    _check_draft(ops, list(range(50)), 40, 20, k, 3, [], expect=[])
    # the only match of the last 2-gram is the n-gram itself (empty continuation); the 1-gram falls back to the earlier 9
    _check_draft(ops, [9, 1, 2, 3, 4, 9], 3, 20, k, 2, [], expect=[1, 2, 3, 4, 9])
    # an EOS as the first draft: no drafts, and no further search (the 1-gram [4] would have found [8, 3, 4])
    _check_draft(ops, [4, 8, 3, 4, 0, 5, 3, 4], 2, 20, k, 2, [0], expect=[])
    # an EOS inside the continuation cuts it
    _check_draft(ops, [3, 4, 5, 6, 0, 8, 3, 4], 2, 20, k, 2, [0], expect=[5, 6])
    # max_length == cur_len + 1: no drafts
    _check_draft(ops, [1, 2, 1, 2, 1], 2, 4, k, 2, [], expect=[])
    # the budget cap: HF proposes k, at most max_new - n_new - 1 remain
    _check_draft(ops, [1, 2, 3, 4, 5, 6, 7, 1], 6, 4, k, 2, [], expect=[2])
    # the leftmost occurrence wins, the largest n-gram size first
    _check_draft(ops, [2, 7, 1, 2, 5, 3, 1, 2], 4, 30, 2, 2, [], expect=[5, 3])
    # done: no drafts whatever the sequence
    seq, tok, d, _ = _draft(ops, [1, 2, 1, 2, 1, 2], 2, 30, k, 2, [], done=1)
    assert d == 0 and (tok == 2).all()


def test_lookup_draft_at_cache_capacity(ops):
    """A sequence that fills a 131072-position cache (Llama 3.1's RoPE table) but for its last k checks."""
    k, max_new, cap = 4, 64, 131072
    S = cap - k - max_new                                   # the cache holds S + max_new + k positions
    g = torch.Generator().manual_seed(5)
    seq = torch.randint(0, 50, (S + max_new - 1,), generator=g).tolist()      # the longest sequence a step sees
    seq[-3:] = seq[100:103]
    _check_draft(ops, seq, S, max_new, k, 3, [], cap=cap, expect=[])          # no budget left for drafts
    seq = seq[:-8]
    seq[-3:] = seq[100:103]
    assert _check_draft(ops, seq, S, max_new, k, 3, [50], cap=cap) > 0


def _accept(ops, drafts, picks, L, n_new, max_new, eos, done=0, log=True):
    dev = "cuda"
    R = len(picks)
    i32 = dict(dtype=torch.int32, device=dev)
    tok = torch.tensor([99] + drafts + [99] * (R - 1 - len(drafts)), dtype=torch.int64, device=dev)
    seq = torch.full((L + R + 4,), -5, dtype=torch.int64, device=dev)
    seq[L:L + len(drafts)] = tok[1:1 + len(drafts)]
    cur, nn, dn = torch.tensor([L], **i32), torch.tensor([n_new], **i32), torch.tensor([done], **i32)
    step, acc = torch.tensor([2], **i32), torch.full((6,), -1, **i32)
    e = torch.tensor(eos, dtype=torch.int64, device=dev) if eos else None
    ops.lookup_accept(torch.tensor(picks, dtype=torch.int64, device=dev), tok, torch.tensor([len(drafts)], **i32), e, seq, cur, nn,
                      max_new, dn, step if log else None, acc if log else None)
    return seq.cpu(), int(cur), int(nn), int(dn), int(step), acc.cpu()


def test_lookup_accept_matches_hf(ops):
    g = torch.Generator().manual_seed(3)
    for trial in range(300):
        k = int(torch.randint(1, 32, (1,), generator=g))
        d = int(torch.randint(0, k + 1, (1,), generator=g))
        drafts = torch.randint(5, 9, (d,), generator=g).tolist()
        picks = torch.randint(5, 11, (k + 1,), generator=g).tolist()      # drafts hold no EOS, picks may
        agree = int(torch.randint(0, d + 1, (1,), generator=g))
        picks[:agree] = drafts[:agree]
        eos = [9 + trial % 2] if trial % 3 == 0 else []
        L, n_new = 50, 3
        max_new = n_new + d + 1 + int(torch.randint(0, 3, (1,), generator=g))
        m = hf_n_matches(drafts, picks[:d + 1])
        seq, cur, nn, dn, step, acc = _accept(ops, drafts, picks, L, n_new, max_new, eos)
        assert seq[L:L + m + 1].tolist() == picks[:m + 1] and (cur, nn, step) == (L + m + 1, n_new + m + 1, 3)
        assert acc[2] == m and (acc[:2] == -1).all()
        assert dn == int(n_new + m + 1 >= max_new or picks[m] in eos)
    # an EOS as the last valid token ends the sequence there
    seq, cur, nn, dn, _, _ = _accept(ops, [4, 6, 7], [4, 6, 0, 3], 10, 1, 50, [0])
    assert seq[10:13].tolist() == [4, 6, 0] and (cur, nn, dn) == (13, 4, 1)
    # once done nothing changes
    seq, cur, nn, dn, step, acc = _accept(ops, [4, 6], [4, 6, 1], 10, 1, 50, [], done=1)
    assert (cur, nn, dn, step) == (10, 1, 1, 2) and (acc == -1).all() and seq[10:12].tolist() == [4, 6]
    # without a log (the first pick): counters only
    _, cur, nn, dn, step, _ = _accept(ops, [], [8], 10, 0, 1, [], log=False)
    assert (cur, nn, dn, step) == (11, 1, 1, 2)


@pytest.mark.parametrize("V", [1024, V8B])
def test_penalty_rows_and_record_rows_match_row_by_row(ops, V):
    """uvx_repetition_penalty_rows over one shared sequence row (stride 0) with lengths L + i equals uvx_repetition_penalty on
    each row alone; uvx_record_scores_rows at per-row indices equals uvx_record_scores at that step, greedy and sampled."""
    g = torch.Generator(device="cuda").manual_seed(7)
    R, L, W = 9, 300, 400
    seq = torch.randint(0, V, (1, W), device="cuda", generator=g)
    logits = torch.randn(R, V, device="cuda", generator=g) * 3
    lens = (L + torch.arange(R, dtype=torch.int32)).cuda()
    got = logits.clone()
    ops.repetition_penalty_rows_(got, seq.expand(R, -1), lens, 1.3, torch.empty(R, W, device="cuda"))
    for i in range(R):
        want = logits[i:i + 1].clone()
        ops.repetition_penalty_(want, seq, torch.tensor([L + i], dtype=torch.int32, device="cuda"), 1.3, torch.empty(1, W, device="cuda"))
        assert torch.equal(got[i], want[0]), i
    steps = 12
    idx = torch.tensor([3, 4, 5, 6, 7, 8, 9, 10, 11], dtype=torch.int32, device="cuda")
    idx[-1] = steps + 2                                     # outside: not written
    for temp, top_k, top_p in ((0.0, 0, 1.0), (0.7, 50, 1.0), (0.9, 0, 0.9), (1.3, 20, 0.8)):
        sc = torch.full((steps, V), 5.0, device="cuda")
        raw = torch.full((steps, V), 5.0, device="cuda")
        ops.record_scores_rows(got, temp, top_k, top_p, idx, scores=sc, raw=raw)
        for i in range(R):
            s = int(idx[i])
            if s >= steps:
                continue
            ws = torch.empty(1, 1, V, device="cuda")
            wr = torch.empty(1, 1, V, device="cuda")
            ops.record_scores(got[i:i + 1].contiguous(), temp, top_k, top_p, torch.zeros(1, dtype=torch.int32, device="cuda"),
                              scores=ws, raw=wr)
            assert torch.equal(sc[s], ws[0, 0]) and torch.equal(raw[s], wr[0, 0]), (temp, i)
        assert (sc[:3] == 5).all() and (raw[:3] == 5).all()


# ------------------------------------------------------------------------------------------------ engine
def build(name="micro", **kw):
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    cfg = preset(name, **kw)
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def sharpen(model, V, logit_std=3.0):
    ids = torch.randint(0, min(V, 1000), (1, 12), generator=torch.Generator().manual_seed(9)).cuda()
    std = float(model(ids, logits_to_keep=1).logits.float().std())
    model.language_model.lm_head.weight.data.mul_(logit_std / std)
    return model


@pytest.fixture(scope="module")
def micro():
    cfg, model = build()
    return sharpen(model, cfg.vocab_size)


@pytest.fixture(scope="module")
def wide():
    from ultravox_b200.config import PRESETS
    base = PRESETS["v0_5_8b"]
    cfg, model = build("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                       text_config=dict(base["text_config"], num_hidden_layers=2))
    # the LM head reads the embedding table and the layers' residual branches are damped, so the fed token's own embedding
    # dominates its logits and replies fall into loops the lookup catches (the random 2-layer model at these widths does not
    # repeat itself within a test's budget); attention and MLP still add their bits to every row
    lm = model.language_model
    lm.lm_head.weight.data.copy_(lm.model.embed_tokens.weight.data)
    for layer in lm.model.layers:
        layer.self_attn.o_proj.weight.data.mul_(0.05)
        layer.mlp.down_proj.weight.data.mul_(0.05)
    model._tiled = None             # the prefill's pre-tiled weight images are rebuilt from the new weights
    return sharpen(model, V8B)


@pytest.fixture
def gemm_decode(monkeypatch):
    """Plain decoding's linears on the decode-form GEMM, as the lookup step's."""
    from ultravox_b200 import engine
    monkeypatch.setattr(engine, "GEMV_MAX_B", 0)


def prompt(seed, S, vocab=1000, loop=0):
    """Random ids, the last `loop` of them repeating an earlier stretch (a quoted span the reply can look up)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (1, S), generator=g)
    if loop:
        ids[0, S - loop:] = ids[0, 2:2 + loop]
    return ids.cuda()


def pair(model, ids, max_new, k=4, n=None, **kw):
    ref = model.generate(ids, max_new_tokens=max_new, **kw)
    got = model.generate(ids, max_new_tokens=max_new, prompt_lookup_num_tokens=k, max_matching_ngram_size=n, **kw)
    return ref, got


@pytest.mark.parametrize("which", ["micro", "wide"])
def test_greedy_tokens_and_accept_log(request, gemm_decode, which):
    model = request.getfixturevalue(which)
    S, N, k = 40, 48, 4
    accepted_total = 0
    for seed in range(4):
        ids = prompt(seed, S, loop=12 if seed % 2 else 0)
        ref, got = pair(model, ids, N, k=k, n=2)
        assert torch.equal(ref, got), seed
        log = model.lookup_stats["accepted"]
        assert log == replay_log(ref[0].tolist(), S, k, 2, [], N), seed
        assert len(log) == model.lookup_stats["steps"] and got.shape[1] == S + N
        accepted_total += sum(log)
    assert accepted_total > 0


def test_k10_matches_row0_of_eleven_streams(micro):
    """k = 10: 11 rows on gemm_swap_kernel<16>; compared at the same instantiation: row 0 of plain generate over 11 copies."""
    S, N = 30, 40
    for seed in range(3):
        ids = prompt(10 + seed, S, loop=10)
        ref = micro.generate(ids.expand(11, -1).contiguous(), max_new_tokens=N)
        got = micro.generate(ids, max_new_tokens=N, prompt_lookup_num_tokens=10, max_matching_ngram_size=3)
        assert torch.equal(ref[:1], got), seed
        assert micro.lookup_stats["accepted"] == replay_log(ref[0].tolist(), S, 10, 3, [], N)


@pytest.mark.parametrize("which", ["micro", "wide"])
def test_sampled_tokens_match(request, gemm_decode, which):
    model = request.getfixturevalue(which)
    S, N = 32, 40
    for seed in range(3):
        ids = prompt(20 + seed, S, loop=10)
        kw = dict(do_sample=True, temperature=0.8, top_k=40, top_p=0.9, repetition_penalty=1.1)
        ref = model.generate(ids, max_new_tokens=N, generator=torch.Generator(device="cuda").manual_seed(seed), **kw)
        got = model.generate(ids, max_new_tokens=N, generator=torch.Generator(device="cuda").manual_seed(seed),
                             prompt_lookup_num_tokens=5, **kw)
        assert torch.equal(ref, got), seed


def test_budgets_and_eos(micro, gemm_decode):
    S, k = 36, 4
    ids = prompt(3, S, loop=14)
    for N in (1, 2, k, k + 1, 2 * k + 3, 37):
        ref, got = pair(micro, ids, N, k=k)
        assert got.shape[1] == S + N and torch.equal(ref, got), N
    full = micro.generate(ids, max_new_tokens=40)[0].tolist()
    new = full[S:]
    # EOS ids only in the prompt: drafts are cut before them, the output is unchanged
    quiet = sorted(set(full[:S]) - set(new))[:3]
    ref, got = pair(micro, ids, 40, k=k, eos_token_id=quiet)
    assert torch.equal(ref, got) and micro.lookup_stats["accepted"] == replay_log(ref[0].tolist(), S, k, 2, quiet, 40)
    # an EOS picked mid-generation: same tokens, same stop
    for j in (1, 5, 11, 23):
        eos = [new[j]]
        ref, got = pair(micro, ids, 40, k=k, eos_token_id=eos)
        assert torch.equal(ref, got), j
        assert got[0, -1].item() == new[j] and micro.lookup_stats["accepted"] == replay_log(ref[0].tolist(), S, k, 2, eos, 40)


def test_conversation_turns(micro, gemm_decode):
    S, N, k = 30, 24, 4
    ids = prompt(4, S, loop=8)
    outs = {}
    for name, extra in (("ref", {}), ("look", dict(prompt_lookup_num_tokens=k))):
        o1 = micro.generate(ids, max_new_tokens=N, return_dict_in_generate=True, **extra)
        turn2 = torch.cat([o1.sequences, prompt(5, 12), o1.sequences[:, 5:15]], dim=1)
        o2 = micro.generate(turn2, max_new_tokens=N, return_dict_in_generate=True, past_key_values=o1.past_key_values, **extra)
        outs[name] = (o1, o2)
    for i in range(2):
        a, b = outs["ref"][i], outs["look"][i]
        assert torch.equal(a.sequences, b.sequences), i
        n = a.past_key_values.length
        assert b.past_key_values.length == n
        assert torch.equal(a.past_key_values.k[:, :, :n], b.past_key_values.k[:, :, :n])
        assert torch.equal(a.past_key_values.v[:, :, :n], b.past_key_values.v[:, :, :n])


class Collect:
    def __init__(self):
        self.parts, self.ended = [], False

    def put(self, t):
        self.parts.append(t.detach().cpu().reshape(1, -1))

    def end(self):
        self.ended = True


def test_streamer(micro, gemm_decode):
    S, N = 30, 40
    ids = prompt(6, S, loop=10)
    st = Collect()
    out = micro.generate(ids, max_new_tokens=N, prompt_lookup_num_tokens=4, streamer=st)
    assert st.ended and torch.equal(torch.cat(st.parts, 1), out.cpu())
    assert torch.equal(st.parts[0], ids.cpu())
    assert len(st.parts) == 2 + micro.lookup_stats["steps"]          # the prompt, the first token, one per step
    assert [p.shape[1] - 1 for p in st.parts[2:]] == micro.lookup_stats["accepted"]
    assert torch.equal(out, micro.generate(ids, max_new_tokens=N))


@pytest.mark.parametrize("sampled", [False, True])
def test_scores_and_logits(micro, gemm_decode, sampled):
    S, N = 30, 32
    ids = prompt(7, S, loop=10)
    kw = dict(max_new_tokens=N, return_dict_in_generate=True, output_scores=True, output_logits=True, repetition_penalty=1.2)
    if sampled:
        kw.update(do_sample=True, temperature=0.7, top_k=30, top_p=0.9)
    ref = micro.generate(ids, generator=torch.Generator(device="cuda").manual_seed(1), **kw)
    got = micro.generate(ids, generator=torch.Generator(device="cuda").manual_seed(1), prompt_lookup_num_tokens=4, **kw)
    assert torch.equal(ref.sequences, got.sequences)
    assert len(got.scores) == len(got.logits) == N
    for t in range(N):
        assert torch.equal(ref.scores[t], got.scores[t]) and torch.equal(ref.logits[t], got.logits[t]), t
    assert sum(micro.lookup_stats["accepted"]) > 0
    tr = micro.compute_transition_scores(got.sequences, got.scores, normalize_logits=True)
    assert tr.shape == (1, N) and torch.isfinite(tr).all()


def test_graph_matches_eager_and_captures_once(micro):
    S, N = 30, 30
    ids = prompt(8, S, loop=10)
    g = micro.generate(ids, max_new_tokens=N, prompt_lookup_num_tokens=6)
    stats = dict(micro.lookup_stats)
    e = micro.generate(ids, max_new_tokens=N, prompt_lookup_num_tokens=6, use_graph=False)
    assert torch.equal(g, e) and micro.lookup_stats["accepted"] == stats["accepted"]
    assert stats["captures"] == 1 and stats["launches_per_step"] > 0 and micro.lookup_stats["captures"] == 0


def test_audio_prompt(micro, gemm_decode):
    """The prefill does not change: a processor-shaped audio request decodes the same with and without lookup."""
    import numpy as np
    from oracle import logmel as ol
    from ultravox_b200 import ops as o
    cfg = micro.config
    padded, frames = ol.pad_batch([np.random.default_rng(3).standard_normal(16000).astype(np.float32)])
    tok = int(-(-int(frames[0]) // 16))
    ids = torch.cat([prompt(9, 8), torch.full((1, tok), 3, device="cuda"), prompt(9, 8)], dim=1)
    mel = o.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    feats = dict(audio_values=mel, audio_token_start_idx=torch.tensor([8]).cuda(), audio_lens=torch.tensor([int(frames[0])]).cuda(),
                 audio_token_len=torch.tensor([tok], dtype=torch.int32).cuda(), audio_batch_size=torch.ones(1, dtype=torch.int64).cuda())
    ref, got = pair(micro, ids, 30, k=3, **feats)
    assert torch.equal(ref, got)


def test_errors(micro):
    ids = prompt(1, 10)
    with pytest.raises(ValueError, match="batch_size = 1"):
        micro.generate(ids.expand(2, -1), max_new_tokens=4, prompt_lookup_num_tokens=4)
    with pytest.raises(ValueError):
        micro.generate(ids, max_new_tokens=4, prompt_lookup_num_tokens=4, num_beams=2)
    for k in (0, 32):
        with pytest.raises(ValueError):
            micro.generate(ids, max_new_tokens=4, prompt_lookup_num_tokens=k)
    with pytest.raises(ValueError):
        micro.generate(ids, max_new_tokens=4, prompt_lookup_num_tokens=4, max_matching_ngram_size=0)
    mask = torch.ones_like(ids)
    mask[0, :3] = 0
    with pytest.raises(NotImplementedError):
        micro.generate(ids, max_new_tokens=4, prompt_lookup_num_tokens=4, attention_mask=mask)
