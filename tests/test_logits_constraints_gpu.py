"""Token constraints in the graph-captured decode step: uvx_logits_constraints (all four forms) against transformers' own
processors in transformers' order, bit for bit, and generate() with no_repeat_ngram_size / sequence_bias / bad_words_ids /
min_length / min_new_tokens / suppress_tokens / begin_suppress_tokens - greedy, sampled, padded, conversation turns, audio,
graph against eager, prompt lookup and beams."""
import numpy as np
import pytest
import torch
from transformers.generation import logits_process as lp

from test_logits_constraints_cpu import hf_processors

pytestmark = pytest.mark.gpu

V8B = 128256


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def hf_chain(V, eos, S, pen=1.0, **kw):
    """transformers' processors in _get_logits_processor's order, the repetition penalty after the sequence bias."""
    procs = hf_processors(V, eos, S, **kw)
    if pen != 1.0:
        at = 1 if kw.get("sequence_bias") is not None else 0
        procs.insert(at, lp.RepetitionPenaltyLogitsProcessor(pen))
    return procs


def hf_run(procs, scores, seqs):
    s = scores.clone()
    for p in procs:
        s = p(seqs, s)
    return s


def build_c(V, eos, S, **kw):
    from ultravox_b200.constraints import LogitsConstraints
    return LogitsConstraints.build(V, eos, S, **kw)


# ================================================================================================ 1. the kernel
def _case(rng, V, L, n, B=2):
    """B sequences of length L (a small alphabet, so n-grams repeat), options whose entries match the sequences' ends, logits
    with planted +-inf / NaN, and a seq tail that would ban or bias tokens if it were read."""
    alpha = 6 if L < 64 else 40
    seq = rng.integers(0, alpha, size=(B, L))
    width = L + 64
    full = np.empty((B, width), np.int64)
    full[:, :L] = seq
    poison = np.tile(np.concatenate([seq[0, max(0, L - 4):L], [V - 1, V - 2]]), width)[:width - L]
    full[:, L:] = poison
    tail0 = [int(t) for t in seq[0, max(0, L - 3):L]]
    t1, t2 = int(rng.integers(0, alpha)), V - 3
    sb = [[[t1], float(rng.normal())], [tail0[-1:] + [t1], 2.5], [tail0[-2:] + [t1], float("-inf")],
          [[int(seq[1, -1]), t2], 1.25], [[t2], -0.5], [tail0[-1:] + [t1], float("inf")], [[V - 2], 0.75]]
    sb = [e for e in sb if all(i > 0 for i in e[0])]
    bad = [tail0[-2:] + [t2], [int(rng.integers(0, alpha))], [V - 1, V - 1]]
    x = (rng.standard_normal((B, V)) * 3).astype(np.float32)
    x[0, [t1, t2, V - 1]] = [np.inf, np.nan, -np.inf]
    x[1, t1] = -np.inf
    kw = dict(no_repeat_ngram_size=n, sequence_bias=sb, bad_words_ids=bad, suppress_tokens=[1, V - 4],
              begin_suppress_tokens=[2, t1])
    return full, seq, x, kw


@pytest.mark.parametrize("V", [1024, V8B])
def test_kernel_equals_hf(ops, V):
    rng = np.random.default_rng(V)
    checked = 0
    for L in (1, 2, 3, 5, 17, 1000, 8192, 131072):
        for n in ((1, 2, 3, 4, 5) if L <= 1000 else (2, 4)):
            full, seq, x, kw = _case(rng, V, L, n)
            eos = [0, 3]
            for S, mn, ml in ((L, 0, None), (L, None, L + 1), (max(1, L - 1), 1, None), (max(1, L - 1), 2, None),
                              (max(1, L - 1), None, L)):
                pen = 1.3 if (L + n) % 2 else 1.0
                c = build_c(V, eos, S, min_new_tokens=mn, min_length=ml, **kw)
                logits = torch.from_numpy(x).cuda()
                sd = torch.from_numpy(full).cuda()
                cur = torch.tensor([L], dtype=torch.int32, device="cuda")
                ops.logits_constraints_(logits, sd, cur, c.device_tables("cuda"))
                if pen != 1.0:
                    ops.repetition_penalty_(logits, sd, cur, pen, torch.empty(sd.shape, dtype=torch.float32, device="cuda"))
                want = hf_run(hf_chain(V, eos, S, pen, min_new_tokens=mn, min_length=ml, **kw), torch.from_numpy(x),
                              torch.from_numpy(seq))
                got = logits.cpu()
                assert torch.equal(got.isnan(), want.isnan()), (L, n, S, mn, ml)
                assert torch.equal(got.nan_to_num(0.0), want.nan_to_num(0.0)), (L, n, S, mn, ml)
                checked += 1
                if L > 1000:
                    break
    assert checked > 40


def test_forms_equal_plain_row_by_row(ops):
    from ultravox_b200.constraints import LogitsConstraints
    rng = np.random.default_rng(5)
    V, slots, W, T = 1024, 4, 300, 64
    seq = torch.from_numpy(rng.integers(0, 8, size=(slots, W))).cuda()
    lens = [40, 1, 257, 90]
    cs = [LogitsConstraints.build(V, [0, 5], l - i, no_repeat_ngram_size=2 + i % 3, bad_words_ids=[[3, 4]],
                                  sequence_bias={(2, 7): 1.5, (7,): -1.0}, min_new_tokens=1, begin_suppress_tokens=[6])
          for i, l in enumerate(lens)]
    tabs = [c.tables(T) for c in cs]
    table = tuple(torch.from_numpy(np.stack([t[k] for t in tabs])).cuda() for k in range(5))
    x = torch.randn(slots, V, device="cuda") * 3

    def plain(s, L, xrow):
        out = xrow.clone()[None]
        ops.logits_constraints_(out, seq[s:s + 1], torch.tensor([L], dtype=torch.int32, device="cuda"), cs[s].device_tables("cuda"))
        return out[0]

    active = torch.tensor([1, 1, 0, 1], dtype=torch.int32, device="cuda")
    cur = torch.tensor(lens, dtype=torch.int32, device="cuda")
    got = ops.logits_constraints_slots_(x.clone(), seq, cur, active, table)
    for s in range(slots):
        assert torch.equal(got[s], plain(s, lens[s], x[s]) if s != 2 else x[s]), s
    # rows: one shared sequence, row i over its first 40 + i tokens
    R = 5
    rl = torch.arange(40, 40 + R, dtype=torch.int32, device="cuda")
    xr = torch.randn(R, V, device="cuda")
    got = ops.logits_constraints_rows_(xr.clone(), seq[0].view(1, -1).expand(R, -1), rl, cs[0].device_tables("cuda"))
    for i in range(R):
        assert torch.equal(got[i], plain(0, 40 + i, xr[i])), i
    # rows_map: rows of slots 3, 0, 2 (inactive), 3 with idx < 0
    row_slot = torch.tensor([3, 3, 0, 2, 3], dtype=torch.int32, device="cuda")
    row_len = torch.tensor([90, 91, 40, 257, 92], dtype=torch.int32, device="cuda")
    row_idx = torch.tensor([0, 1, 0, 0, -1], dtype=torch.int32, device="cuda")
    got = ops.logits_constraints_rows_map_(xr.clone(), seq, active, row_slot, row_len, row_idx, table)
    for r in range(R):
        s, L = int(row_slot[r]), int(row_len[r])
        want = xr[r] if s == 2 or int(row_idx[r]) < 0 else plain(s, L, xr[r])
        assert torch.equal(got[r], want), r


# ================================================================================================ 2. generate()
def _model(logit_std=3.0):
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    cfg = preset("micro")
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    ids = torch.randint(0, min(cfg.vocab_size, 1000), (1, 12), generator=torch.Generator().manual_seed(9)).cuda()
    std = float(model(ids, logits_to_keep=1).logits.float().std())
    model.language_model.lm_head.weight.data.mul_(logit_std / std)
    return cfg, model


@pytest.fixture(scope="module")
def micro():
    return _model()


def _options(ids, out0, S):
    """Per-option settings built from an unconstrained reply out0 [B, S + n], so each one changes something."""
    r = out0[0, S:].tolist()
    eos = [r[2]]
    return eos, {
        "ngram": dict(no_repeat_ngram_size=2),
        "bias": dict(sequence_bias=[[[r[0]], -4.0], [[r[0], r[1]], -20.0], [[r[3]], 2.0]]),
        "bad": dict(bad_words_ids=[[r[1]], [r[3], r[4]], [eos[0]]]),
        "min_new": dict(min_new_tokens=6),
        "min_len": dict(min_length=S + 5),
        "suppress": dict(suppress_tokens=[r[4], r[5]]),
        "begin": dict(begin_suppress_tokens=[r[0]]),
        "all": dict(no_repeat_ngram_size=3, sequence_bias={(r[1],): 1.0, (r[0], r[1]): -3.0}, bad_words_ids=[[r[2], r[3]]],
                    min_new_tokens=4, suppress_tokens=[r[5]], begin_suppress_tokens=[r[0]], repetition_penalty=1.2),
    }


def _check_scores(cfg, out, S, eos, kw, pen):
    seqs = out.sequences.cpu()
    opts = {k: v for k, v in kw.items() if k != "repetition_penalty"}
    procs = hf_chain(cfg.vocab_size, eos, S, pen, **opts)
    for t in range(len(out.scores)):
        want = hf_run(procs, out.logits[t].cpu(), seqs[:, :S + t])
        got = out.scores[t].cpu()
        assert torch.equal(got.isnan(), want.isnan()) and torch.equal(got.nan_to_num(0.0), want.nan_to_num(0.0)), (kw, t)
        assert torch.equal(got.argmax(-1), seqs[:, S + t]), (kw, t)


def test_generate_each_option_and_all(micro):
    cfg, model = micro
    ids = torch.randint(0, 1000, (1, 10), generator=torch.Generator().manual_seed(3)).cuda()
    S, n = 10, 14
    out0 = model.generate(ids, max_new_tokens=n)
    eos, options = _options(ids, out0, S)
    changed = 0
    for name, kw in options.items():
        pen = kw.get("repetition_penalty", 1.0)
        out = model.generate(ids, max_new_tokens=n, eos_token_id=eos, return_dict_in_generate=True, output_scores=True,
                             output_logits=True, **kw)
        _check_scores(cfg, out, S, eos, kw, pen)
        eager = model.generate(ids, max_new_tokens=n, eos_token_id=eos, use_graph=False, **kw)
        assert torch.equal(eager, out.sequences), name
        plain = model.generate(ids, max_new_tokens=n, eos_token_id=eos, return_dict_in_generate=True, output_logits=True)
        assert torch.equal(plain.logits[0], out.logits[0]), name          # output_logits stay raw
        changed += not torch.equal(plain.sequences, out.sequences)
        reply = out.sequences[0, S:].tolist()
        if name == "ngram":
            grams = list(zip(out.sequences[0].tolist(), out.sequences[0].tolist()[1:]))
            assert len(set(grams[S - 1:])) == len(grams[S - 1:]) and not set(grams[S - 1:]) & set(grams[:S - 1])
        if name == "min_new":
            assert eos[0] not in reply[:6]
    assert changed >= 4, changed


def test_generate_padded_batch_turns_audio(micro):
    cfg, model = micro
    B, S, n = 3, 12, 10
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(0, 1000, (B, S), generator=g)
    am = torch.ones(B, S, dtype=torch.long)
    for b in range(1, B):
        am[b, :2 * b] = 0
        ids[b, :2 * b] = 0
    ids, am = ids.cuda(), am.cuda()
    out0 = model.generate(ids, attention_mask=am, max_new_tokens=n)
    eos, options = _options(ids, out0, S)
    kw = options["all"]
    out = model.generate(ids, attention_mask=am, max_new_tokens=n, eos_token_id=eos, return_dict_in_generate=True,
                         output_scores=True, output_logits=True, **kw)
    _check_scores(cfg, out, S, eos, kw, 1.2)
    # sampled: every token lies where HF's processed scores are finite
    gen = torch.Generator(device="cuda").manual_seed(4)
    smp = model.generate(ids, attention_mask=am, max_new_tokens=n, eos_token_id=eos, do_sample=True, top_k=20, generator=gen,
                         return_dict_in_generate=True, output_scores=True, output_logits=True, **kw)
    seqs = smp.sequences.cpu()
    procs = hf_chain(cfg.vocab_size, eos, S, 1.2, **{k: v for k, v in kw.items() if k != "repetition_penalty"})
    for t in range(len(smp.scores)):
        proc = hf_run(procs, smp.logits[t].cpu(), seqs[:, :S + t])
        tok = seqs[:, S + t]
        assert torch.isfinite(proc.gather(1, tok[:, None])).all() and torch.isfinite(smp.scores[t].cpu().gather(1, tok[:, None])).all()
    # a conversation turn: the second call's constraints see the whole conversation
    one = ids[:1]
    t1 = model.generate(one, max_new_tokens=6, return_dict_in_generate=True)
    follow = torch.cat([t1.sequences, torch.randint(0, 1000, (1, 4), generator=g).cuda()], 1)
    S2 = follow.shape[1]
    kw2 = dict(no_repeat_ngram_size=2, sequence_bias=[[[int(follow[0, -1]), 5], 3.0]], begin_suppress_tokens=[5])
    turn = model.generate(follow, past_key_values=t1.past_key_values, max_new_tokens=8, return_dict_in_generate=True,
                          output_scores=True, output_logits=True, **kw2)
    _check_scores(cfg, turn, S2, [], kw2, 1.0)
    # audio
    from oracle import logmel as ol
    from ultravox_b200 import ops
    padded, frames = ol.pad_batch([np.random.default_rng(1).standard_normal(16000).astype(np.float32)])
    tok = int(-(-int(frames[0]) // 16))
    aids = torch.cat([torch.randint(0, 1000, (1, 8), generator=g), torch.full((1, tok), 3),
                      torch.randint(0, 1000, (1, 5), generator=g)], 1).cuda()
    feats = dict(audio_values=ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins),
                 audio_token_start_idx=torch.tensor([8]).cuda(), audio_lens=torch.tensor([int(frames[0])]).cuda(),
                 audio_token_len=torch.tensor([tok], dtype=torch.int32).cuda(), audio_batch_size=torch.ones(1, dtype=torch.int64).cuda())
    kw3 = dict(no_repeat_ngram_size=1, suppress_tokens=[3])       # n = 1 bans every id already there, placeholders included
    au = model.generate(aids, max_new_tokens=8, return_dict_in_generate=True, output_scores=True, output_logits=True, **feats, **kw3)
    _check_scores(cfg, au, aids.shape[1], [], kw3, 1.0)
    assert not set(au.sequences[0, aids.shape[1]:].tolist()) & set(aids[0].tolist())


def test_generate_defaults_unchanged_and_errors(micro):
    cfg, model = micro
    ids = torch.randint(0, 1000, (1, 10), generator=torch.Generator().manual_seed(3)).cuda()
    a = model.generate(ids, max_new_tokens=6)
    b = model.generate(ids, max_new_tokens=6, no_repeat_ngram_size=0, min_new_tokens=3)     # off, and no EOS ids
    assert torch.equal(a, b)
    for bad in (dict(bad_words_ids=[5]), dict(sequence_bias={(5,): 1}), dict(no_repeat_ngram_size=2.5),
                dict(bad_words_ids=[[cfg.vocab_size]])):
        with pytest.raises(ValueError):
            model.generate(ids, max_new_tokens=3, **bad)


# ================================================================================================ 3. prompt lookup and beams
def test_prompt_lookup_equals_plain(micro):
    cfg, model = micro
    base = torch.randint(0, 1000, (1, 6), generator=torch.Generator().manual_seed(8))
    ids = torch.cat([base, base, base[:, :3]], 1).cuda()        # repeats, so drafts are proposed
    S = ids.shape[1]
    out0 = model.generate(ids, max_new_tokens=16)
    eos, options = _options(ids, out0, S)
    for name in ("ngram", "bias", "all"):
        kw = options[name]
        plain = model.generate(ids, max_new_tokens=16, eos_token_id=eos, return_dict_in_generate=True, output_scores=True, **kw)
        look = model.generate(ids, max_new_tokens=16, eos_token_id=eos, prompt_lookup_num_tokens=4, return_dict_in_generate=True,
                              output_scores=True, **kw)
        assert torch.equal(plain.sequences, look.sequences), name
        for t in range(len(plain.scores)):
            assert torch.equal(plain.scores[t].nan_to_num(0.0), look.scores[t].nan_to_num(0.0)), (name, t)


def test_beam_processed_logprobs_are_hf(micro, ops):
    """Beam search: the log-probs the engine selects from are log_softmax(logits), then transformers' processors (the
    constraints and the penalty) over each running beam."""
    from ultravox_b200.engine import BeamDecodeEngine
    cfg, model = micro
    ids = torch.randint(0, 1000, (2, 10), generator=torch.Generator().manual_seed(12)).cuda()
    S, nb = 10, 3
    out0 = model.generate(ids, max_new_tokens=8)
    eos, options = _options(ids, out0, S)
    kw = options["all"]
    opts = {k: v for k, v in kw.items() if k != "repetition_penalty"}
    c = build_c(cfg.vocab_size, eos, S, **opts)
    rec = []

    def hook(eng):
        torch.cuda.synchronize()
        raw_lp = ops.log_softmax(eng.logits.contiguous(), out=torch.empty_like(eng.logprobs))
        rec.append((raw_lp.cpu(), eng.logprobs.cpu().clone()))

    seqs_before = []
    orig_pick = BeamDecodeEngine._pick

    def pick(self, logits):         # the running sequences each pick sees
        seqs_before.append(self.seq[:, :int(self.cur_len)].cpu().clone())
        return orig_pick(self, logits)

    BeamDecodeEngine._pick = pick
    try:
        fk = dict(audio_values=None, inputs_embeds=None, attention_mask=None, audio_token_start_idx=None, audio_lens=None,
                  audio_token_len=None, audio_batch_size=None, position_ids=None, audio_waveforms=None, audio_num_frames=None,
                  audio_pad_frames=None)
        seqs, _ = model._beam_search(ids, fk, None, 8, eos, 0, nb, 1.0, False, 1, 1.2, False, step_hook=hook, constraints=c)
    finally:
        BeamDecodeEngine._pick = orig_pick
    procs = hf_chain(cfg.vocab_size, eos, S, 1.2, **opts)
    assert len(rec) == len(seqs_before) >= 2
    for t, ((raw_lp, got), run) in enumerate(zip(rec, seqs_before)):
        want = hf_run(procs, raw_lp, run)
        assert torch.equal(got.nan_to_num(0.0), want.nan_to_num(0.0)), t
    g = model.generate(ids, num_beams=nb, max_new_tokens=8, eos_token_id=eos, repetition_penalty=1.2, **opts)
    assert torch.equal(g.cpu(), seqs.cpu())
    # transformers' own _beam_search, fed our raw log-probs and applying the same processors itself, selects the same beams
    from test_beam_gpu import _hf
    t_seen = []

    def replay(input_ids, scores):
        t = len(t_seen)
        t_seen.append(t)
        assert t < len(rec) and torch.equal(input_ids, seqs_before[t]), f"running sequences differ at step {t}"
        return hf_run(procs, rec[t][0], input_ids)

    out = _hf(cfg.vocab_size, ids.cpu(), torch.ones_like(ids.cpu()), nb, eos, 1.0, False, 1, 8, 0, replay)
    assert len(t_seen) == len(rec)
    assert torch.equal(out.sequences, seqs.cpu())
