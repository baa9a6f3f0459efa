"""Stop strings in the graph-captured decode step: uvx_stop_strings (all four forms) against the numpy walk of the packed table and
transformers' StopStringCriteria, the _stop finishing forms against their plain forms, and generate(stop_strings=...) against
the run without them cut at HF's first hit - greedy, sampled, padded, first token, EOS in the same step, the budget, a
conversation turn, the streamer, scores / logits, audio, graph against eager, prompt lookup (a hit on a non-final accepted
draft) and beam search against transformers' own _beam_search."""
import numpy as np
import pytest
import torch

from test_stop_strings_cpu import hf_hits, make_tokenizer
from ultravox_b200 import stop_strings as ss

pytestmark = pytest.mark.gpu

V8B = 128256


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


# ================================================================================================ 1. the kernel
def _rows_for(rng, tok, V, text_ids, L, B):
    """B sequences of L preceding tokens plus a candidate: mostly ends of the text (so strings match), some random ids and ids
    past the tokenizer's table."""
    out = []
    for b in range(B):
        x = list(rng.integers(0, V, size=L + 1))
        k = int(rng.integers(1, len(text_ids) + 1))
        end = text_ids[:k]
        if b % 4 != 3:
            n = min(len(end), L + 1)
            x[L + 1 - n:] = end[len(end) - n:]
        if b % 5 == 4:
            x[L - min(L, 1)] = V + 3
        out.append(x)
    return out


@pytest.mark.parametrize("V,kind", [(1024, "bytelevel"), (1024, "metaspace"), (V8B, "bytelevel")])
def test_kernel_equals_walk_and_hf(ops, V, kind):
    tok = make_tokenizer(V, kind, seed=5)
    text = " the user: hello there.\nuser: fine, ok! assistant: done."
    text_ids = tok(text, add_special_tokens=False)["input_ids"]
    dec = tok.decode(text_ids)
    rng = np.random.default_rng(V)
    sets = [["user:"], ["r: f", "ok!"], ["user", "user:", "er"], [dec[5:17], dec[-9:], "!", "ne.", dec[20:23]]]
    hits = 0
    for strings in sets:
        st = ss.StopStrings.build(tok, strings)
        tab = st.device_table("cuda")
        for L in (0, 1, 2, 5, 40, 1000, 131071):
            B = 64 if L <= 40 else 3
            rows = _rows_for(rng, tok, V, text_ids, L, B)
            width = L + 64
            seq = torch.empty(B, width, dtype=torch.int64)
            for b, x in enumerate(rows):
                seq[b, :L] = torch.tensor(x[:L])
                seq[b, L:] = torch.tensor((text_ids * (64 // len(text_ids) + 1))[:64])     # poison: never read
            cand = torch.tensor([x[L] for x in rows])
            hit = torch.full((B,), 7, dtype=torch.int32, device="cuda")
            ops.stop_strings(cand.cuda(), seq.cuda(), torch.tensor([L], dtype=torch.int32).cuda(), tab, hit)
            got = hit.cpu().tolist()
            want = [int(ss.walk(st.table, x)) for x in rows]
            assert got == want, (strings, L)
            if L <= 40:
                assert [int(h) for h in hf_hits(st.criteria, rows)] == want, (strings, L)
            hits += sum(want)
    assert hits > 20


def test_forms_equal_plain_row_by_row(ops):
    V = 1024
    tok = make_tokenizer(V, "bytelevel", seed=5)
    text_ids = tok(" user: fine, ok! user: done.", add_special_tokens=False)["input_ids"]
    rng = np.random.default_rng(2)
    tabs = [ss.StopStrings.build(tok, s) for s in (["user:"], ["ok!", "e."], ["ne", "user: d"])]
    S, W = 6, max(t.n_words for t in tabs)
    tab = torch.zeros(S, W, dtype=torch.int32)
    for s in range(S):
        if s % 3 != 2 or s == 5:
            t = tabs[s % 3].table
            tab[s, :t.size] = torch.from_numpy(t)            # slot 2: no stop strings (zero header)
    tab = tab.cuda()
    seq = torch.from_numpy(rng.integers(0, V, size=(S, 200))).cuda()
    for s in range(S):
        n = int(rng.integers(3, len(text_ids)))
        seq[s, 30:30 + n] = torch.tensor(text_ids[:n])
    lens = torch.tensor([30 + int(rng.integers(2, 12)) for _ in range(S)], dtype=torch.int32).cuda()
    cand = torch.stack([seq[s, lens[s]] for s in range(S)])
    active = torch.tensor([1, 1, 1, 0, 1, 1], dtype=torch.int32).cuda()
    hit = torch.full((S,), 9, dtype=torch.int32, device="cuda")
    ops.stop_strings_slots(cand, seq, lens, active, tab, hit)
    want = []
    for s in range(S):
        h = torch.zeros(1, dtype=torch.int32, device="cuda")
        ops.stop_strings(cand[s:s + 1], seq[s:s + 1], lens[s:s + 1], tab[s], h)
        want.append(int(h) if active[s] else 9)
    assert hit.tolist() == want
    # rows: one shared sequence, per-row lengths
    R = 5
    rl = torch.tensor([31, 33, 35, 37, 39], dtype=torch.int32).cuda()
    rc = torch.stack([seq[0, int(l)] for l in rl])
    rh = torch.zeros(R, dtype=torch.int32, device="cuda")
    ops.stop_strings_rows(rc, seq[0:1].expand(R, -1), rl, tab[0], rh)
    for r in range(R):
        h = torch.zeros(1, dtype=torch.int32, device="cuda")
        ops.stop_strings(rc[r:r + 1], seq[0:1], rl[r:r + 1], tab[0], h)
        assert int(rh[r]) == int(h)
    # rows_map: slot s owns rows s * 2 + i; idx -1 and inactive slots untouched
    row_slot = torch.tensor([s for s in range(S) for _ in range(2)], dtype=torch.int32).cuda()
    row_len = torch.tensor([int(lens[s]) + i for s in range(S) for i in range(2)], dtype=torch.int32).cuda()
    row_idx = torch.tensor([0 if i == 0 or s % 2 else -1 for s in range(S) for i in range(2)], dtype=torch.int32).cuda()
    mc = torch.stack([seq[int(row_slot[r]), int(row_len[r])] for r in range(2 * S)])
    mh = torch.full((2 * S,), 9, dtype=torch.int32, device="cuda")
    ops.stop_strings_rows_map(mc, seq, active, row_slot, row_len, row_idx, tab, mh)
    for r in range(2 * S):
        s = int(row_slot[r])
        if not active[s] or row_idx[r] < 0:
            assert int(mh[r]) == 9
            continue
        h = torch.zeros(1, dtype=torch.int32, device="cuda")
        ops.stop_strings(mc[r:r + 1], seq[s:s + 1], row_len[r:r + 1], tab[s], h)
        assert int(mh[r]) == int(h), r


def test_finish_forms_with_no_hit_equal_plain(ops):
    rng = np.random.default_rng(4)
    dev = "cuda"
    B = 7
    eos = torch.tensor([3, 9], device=dev)

    def i32(a):
        return torch.tensor(a, dtype=torch.int32, device=dev)

    # token_finish
    tok = torch.from_numpy(rng.integers(0, 12, size=B)).to(dev)
    state = dict(done=i32(rng.integers(0, 2, size=B)), seq=torch.zeros(B, 20, dtype=torch.int64, device=dev), cur=i32([5]),
                 step=i32([2]), b0=i32(rng.integers(0, 9, size=B)), b1=i32(rng.integers(0, 9, size=B)),
                 b2=i32(rng.integers(0, 9, size=B)), all_done=i32([0]))
    outs = []
    for stop in (None, (torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.int32, device=dev))):
        st = {k: v.clone() for k, v in state.items()}
        t = tok.clone()
        ops.token_finish(t, st["done"], eos, 0, st["seq"], st["cur"], st["step"], (st["b0"], st["b1"], st["b2"]), st["all_done"],
                         stop=stop)
        outs.append([t] + list(st.values()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    # slot_finish
    st0 = dict(done=i32(rng.integers(0, 2, size=B)), seq=torch.zeros(B, 20, dtype=torch.int64, device=dev),
               cur=i32(rng.integers(3, 9, size=B)), n_new=i32(rng.integers(0, 4, size=B)), pos=i32(rng.integers(0, 9, size=B)),
               lens=i32(rng.integers(0, 9, size=B)), rope=i32(rng.integers(0, 9, size=B)), n_open=i32([0]))
    max_new, active = i32(rng.integers(1, 5, size=B)), i32(rng.integers(0, 2, size=B))
    outs = []
    for hit in (None, torch.zeros(B, dtype=torch.int32, device=dev)):
        st = {k: v.clone() for k, v in st0.items()}
        ops.slot_finish(tok, st["done"], eos, st["seq"], st["cur"], st["n_new"], max_new, active, st["pos"], st["lens"], st["rope"],
                        st["n_open"], hit=hit)
        outs.append(list(st.values()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    # lookup_accept: k + 1 = 5 rows, two drafts agree
    k = 4
    pick = torch.tensor([5, 6, 7, 8, 2], device=dev)
    fed = torch.tensor([1, 5, 6, 11, 4], device=dev)
    outs = []
    for hit in (None, torch.zeros(k + 1, dtype=torch.int32, device=dev)):
        seq = torch.zeros(30, dtype=torch.int64, device=dev)
        c = [i32([10]), i32([3]), i32([0]), i32([0]), torch.zeros(8, dtype=torch.int32, device=dev)]
        ops.lookup_accept(pick, fed, i32([3]), eos, seq, c[0], c[1], 20, c[2], c[3], c[4], hit=hit)
        outs.append([seq] + c)
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    # lookup_accept_slots: 3 slots, K = 2
    K, Sl = 2, 3
    R = Sl * (K + 1)
    pick = torch.from_numpy(rng.integers(0, 12, size=R)).to(dev)
    fed = pick.clone()
    fed[1:] = pick[:-1]
    outs = []
    for hit in (None, torch.zeros(R, dtype=torch.int32, device=dev)):
        seq = torch.zeros(Sl, 30, dtype=torch.int64, device=dev)
        st = [torch.zeros(Sl, dtype=torch.int64, device=dev), i32([0, 0, 1]), i32([5, 6, 7]), i32([1, 1, 1]), i32([4, 5, 6]),
              i32([4, 5, 6]), i32([5, 6, 7]), i32([0, 0, 0]), i32([0])]
        ops.lookup_accept_slots(pick, fed, i32([2, 1, 0]), K, eos, seq, st[0], st[1], st[2], st[3], i32([9, 9, 9]), i32([1, 1, 1]),
                                st[4], st[5], st[6], st[7], st[8], hit=hit)
        outs.append([seq] + st)
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_lookup_accept_cut_at_a_hit(ops):
    """A hit at row i < m cuts the accept there: pick[0..i] appended, the sequence finished, counters as for i + 1 tokens."""
    dev = "cuda"

    def i32(a):
        return torch.tensor(a, dtype=torch.int32, device=dev)

    eos = torch.tensor([3], device=dev)
    pick = torch.tensor([5, 6, 7, 8, 2], device=dev)
    fed = torch.tensor([1, 5, 6, 7, 4], device=dev)         # three drafts, all agreeing: m = 3 without a hit
    for hit_row, m_want in ((None, 3), (1, 1), (0, 0), (3, 3)):
        hit = torch.zeros(5, dtype=torch.int32, device=dev)
        if hit_row is not None:
            hit[hit_row] = 1
        seq = torch.zeros(30, dtype=torch.int64, device=dev)
        cur, nn, done, step, acc = i32([10]), i32([3]), i32([0]), i32([0]), torch.zeros(8, dtype=torch.int32, device=dev)
        ops.lookup_accept(pick, fed, i32([3]), eos, seq, cur, nn, 20, done, step, acc, hit=hit)
        assert int(cur) == 10 + m_want + 1 and int(nn) == 3 + m_want + 1 and int(acc[0]) == m_want, hit_row
        assert int(done) == (hit_row is not None)
        assert seq[10:10 + m_want + 1].tolist() == pick[:m_want + 1].tolist() and int(seq[10 + m_want + 1]) == 0
    # slots, K = 3: slot 0 cut at row 1 by a hit, slot 1 without a hit, slot 2 with a hit past its agreeing drafts
    K, Sl = 3, 3
    pick = torch.tensor([5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16], device=dev)
    fed = torch.tensor([1, 5, 6, 7, 1, 9, 10, 4, 1, 13, 4, 4], device=dev)      # agreeing drafts: 3, 2, 1
    hit = torch.zeros(12, dtype=torch.int32, device=dev)
    hit[1] = 1
    hit[8 + 3] = 1                                          # past slot 2's accepted rows: no effect
    seq = torch.zeros(Sl, 30, dtype=torch.int64, device=dev)
    token = torch.zeros(Sl, dtype=torch.int64, device=dev)
    done, cur, nn = i32([0, 0, 0]), i32([5, 6, 7]), i32([1, 1, 1])
    pos, lens, rope, acc, n_open = i32([4, 5, 6]), i32([5, 6, 7]), i32([4, 5, 6]), i32([0, 0, 0]), i32([0])
    ops.lookup_accept_slots(pick, fed, i32([3, 2, 2]), K, eos, seq, token, done, cur, nn, i32([20, 20, 20]), i32([1, 1, 1]), pos,
                            lens, rope, acc, n_open, hit=hit)
    assert acc.tolist() == [1, 2, 1] and done.tolist() == [1, 0, 0] and int(n_open) == 2
    assert cur.tolist() == [5 + 2, 6 + 3, 7 + 2] and nn.tolist() == [3, 4, 3]
    assert pos.tolist() == [4 + 1, 5 + 3, 6 + 2] and token.tolist() == [6, 11, 14]
    assert seq[0, 5:8].tolist() == [5, 6, 0]


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
    cfg, model = _model()
    return cfg, model, make_tokenizer(cfg.vocab_size, "bytelevel", seed=1)


def expected(full, S, crit, eos, pad):
    """The run without stop strings, cut as HF's StopStringCriteria + EOS would: each row finishes at its first hit (or EOS),
    pad after, and the output ends at the step the last row finished."""
    full = full.cpu()
    B, T = full.shape
    fin = []
    for b in range(B):
        f = None
        for t in range(S, T):
            if int(full[b, t]) in eos or bool(crit(full[b:b + 1, :t + 1], None)[0]):
                f = t
                break
        fin.append(f)
    out = full.clone()
    for b, f in enumerate(fin):
        if f is not None:
            out[b, f + 1:] = pad
    if all(f is not None for f in fin):
        out = out[:, :max(fin) + 1]
    return out, fin


def _strings_from(tok, reply, a, b):
    """A stop string cut from the decoded reply, starting and ending inside tokens where the text allows."""
    txt = tok.decode(reply)
    return txt[a:b]


def test_generate_cut_at_first_hit(micro):
    cfg, model, tok = micro
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 1000, (1, 10), generator=g).cuda()
    S, n = 10, 24
    full = model.generate(ids, max_new_tokens=n)
    reply = full[0, S:].tolist()
    txt = tok.decode(reply)
    cases = [[txt[9:14]], [txt[20:23], txt[21:23]], [txt[30:36], txt[33:40]], [tok.decode(full[0, S - 2:S + 1].tolist())],
             [txt[-4:]]]
    n_hit = 0
    for strings in cases:
        strings = [s for s in strings if s]
        st = ss.StopStrings.build(tok, strings)
        want, fin = expected(full, S, st.criteria, [], 0)
        got = model.generate(ids, max_new_tokens=n, stop_strings=strings, tokenizer=tok)
        assert torch.equal(got.cpu(), want), strings
        eager = model.generate(ids, max_new_tokens=n, stop_strings=strings, tokenizer=tok, use_graph=False)
        assert torch.equal(eager, got), strings
        n_hit += fin[0] is not None
        # streamer: the same tokens, put one by one
        class Stream:
            def __init__(self):
                self.parts = []

            def put(self, t):
                self.parts.append(t.cpu().view(1, -1))

            def end(self):
                pass
        sm = Stream()
        sgot = model.generate(ids, max_new_tokens=n, stop_strings=strings, tokenizer=tok, streamer=sm)
        assert torch.equal(sgot, got) and torch.equal(torch.cat(sm.parts, 1), got.cpu())
    assert n_hit >= 4
    # EOS at the same step as the hit, and the budget before the hit
    strings = [txt[9:14]]
    st = ss.StopStrings.build(tok, strings)
    _, fin = expected(full, S, st.criteria, [], 0)
    eos = [reply[fin[0] - S]]
    want, _ = expected(model.generate(ids, max_new_tokens=n, eos_token_id=eos), S, st.criteria, eos, eos[0])
    assert torch.equal(model.generate(ids, max_new_tokens=n, eos_token_id=eos, stop_strings=strings, tokenizer=tok).cpu(), want)
    short = model.generate(ids, max_new_tokens=fin[0] - S, stop_strings=strings, tokenizer=tok)
    assert torch.equal(short, full[:, :fin[0]])
    # scores and logits: those of the run without stop strings, for the steps kept
    out = model.generate(ids, max_new_tokens=n, stop_strings=strings, tokenizer=tok, return_dict_in_generate=True,
                         output_scores=True, output_logits=True)
    ref = model.generate(ids, max_new_tokens=n, return_dict_in_generate=True, output_scores=True, output_logits=True)
    kept = out.sequences.shape[1] - S
    assert len(out.scores) == len(out.logits) == kept
    assert all(torch.equal(a, b) for a, b in zip(out.scores, ref.scores[:kept]))
    assert all(torch.equal(a, b) for a, b in zip(out.logits, ref.logits[:kept]))


def test_generate_sampled_padded_turn_audio(micro):
    cfg, model, tok = micro
    g = torch.Generator().manual_seed(11)
    # seeded sampling
    ids = torch.randint(0, 1000, (1, 9), generator=g).cuda()
    kw = dict(max_new_tokens=20, do_sample=True, top_k=30)
    full = model.generate(ids, generator=torch.Generator(device="cuda").manual_seed(5), **kw)
    txt = tok.decode(full[0, 9:].tolist())
    strings = [txt[12:17]]
    st = ss.StopStrings.build(tok, strings)
    want, fin = expected(full, 9, st.criteria, [], 0)
    got = model.generate(ids, generator=torch.Generator(device="cuda").manual_seed(5), stop_strings=strings, tokenizer=tok, **kw)
    assert fin[0] is not None and torch.equal(got.cpu(), want)
    # padded B = 3, rows stopping at different steps (and one that never stops)
    B, S, n = 3, 12, 16
    ids = torch.randint(0, 1000, (B, S), generator=g)
    am = torch.ones(B, S, dtype=torch.long)
    for b in range(1, B):
        am[b, :2 * b] = 0
        ids[b, :2 * b] = 0
    ids, am = ids.cuda(), am.cuda()
    full = model.generate(ids, attention_mask=am, max_new_tokens=n)
    strings = [tok.decode(full[0, S:].tolist())[6:10], tok.decode(full[1, S:].tolist())[25:29]]
    st = ss.StopStrings.build(tok, strings)
    for eos in ([], [int(full[2, S + 9])]):
        ref = full if not eos else model.generate(ids, attention_mask=am, max_new_tokens=n, eos_token_id=eos)
        want, fin = expected(ref, S, st.criteria, eos, eos[0] if eos else 0)
        got = model.generate(ids, attention_mask=am, max_new_tokens=n, stop_strings=strings, tokenizer=tok, eos_token_id=eos)
        assert torch.equal(got.cpu(), want), (eos, fin)
    # a conversation turn: the string may begin in the earlier turns
    one = ids[:1]
    t1 = model.generate(one, max_new_tokens=6, return_dict_in_generate=True)
    follow = torch.cat([t1.sequences, torch.randint(0, 1000, (1, 4), generator=g).cuda()], 1)
    plain = model.generate(follow, past_key_values=t1.past_key_values, max_new_tokens=10)
    S2 = follow.shape[1]
    t1b = model.generate(one, max_new_tokens=6, return_dict_in_generate=True)
    strings = [tok.decode(plain[0, S2 - 2:S2 + 3].tolist())[1:-1]]
    st = ss.StopStrings.build(tok, strings)
    want, fin = expected(plain, S2, st.criteria, [], 0)
    got = model.generate(follow, past_key_values=t1b.past_key_values, max_new_tokens=10, stop_strings=strings, tokenizer=tok)
    assert fin[0] is not None and torch.equal(got.cpu(), want)
    # audio prompt
    from oracle import logmel as ol
    from ultravox_b200 import ops
    padded, frames = ol.pad_batch([np.random.default_rng(1).standard_normal(16000).astype(np.float32)])
    ntok = int(-(-int(frames[0]) // 16))
    aids = torch.cat([torch.randint(0, 1000, (1, 8), generator=g), torch.full((1, ntok), 3),
                      torch.randint(0, 1000, (1, 5), generator=g)], 1).cuda()
    feats = dict(audio_values=ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins),
                 audio_token_start_idx=torch.tensor([8]).cuda(), audio_lens=torch.tensor([int(frames[0])]).cuda(),
                 audio_token_len=torch.tensor([ntok], dtype=torch.int32).cuda(), audio_batch_size=torch.ones(1, dtype=torch.int64).cuda())
    afull = model.generate(aids, max_new_tokens=12, **feats)
    Sa = aids.shape[1]
    strings = [tok.decode(afull[0, Sa:].tolist())[5:9]]
    st = ss.StopStrings.build(tok, strings)
    want, fin = expected(afull, Sa, st.criteria, [], 0)
    got = model.generate(aids, max_new_tokens=12, stop_strings=strings, tokenizer=tok, **feats)
    assert fin[0] is not None and torch.equal(got.cpu(), want)


def test_generate_defaults_unchanged_and_errors(micro):
    cfg, model, tok = micro
    ids = torch.randint(0, 1000, (1, 10), generator=torch.Generator().manual_seed(3)).cuda()
    a = model.generate(ids, max_new_tokens=6)
    assert torch.equal(a, model.generate(ids, max_new_tokens=6, tokenizer=tok))       # a tokenizer alone is ignored
    with pytest.raises(ValueError):
        model.generate(ids, max_new_tokens=3, stop_strings="ab")
    with pytest.raises(ValueError):
        model.generate(ids, max_new_tokens=3, stop_strings=[""], tokenizer=tok)


# ================================================================================================ 3. prompt lookup
def test_prompt_lookup_equals_plain(micro):
    cfg, model, tok = micro
    base = torch.randint(0, 1000, (1, 6), generator=torch.Generator().manual_seed(8))
    ids = torch.cat([base, base, base[:, :3]], 1).cuda()        # repeats, so drafts are proposed
    S, n = ids.shape[1], 24
    full = model.generate(ids, max_new_tokens=n)
    txt = tok.decode(full[0, S:].tolist())
    accepted_mid = 0
    for a, b in ((3, 7), (10, 13), (18, 24), (30, 33)):
        strings = [txt[a:b]]
        if not strings[0]:
            continue
        plain = model.generate(ids, max_new_tokens=n, stop_strings=strings, tokenizer=tok)
        look = model.generate(ids, max_new_tokens=n, stop_strings=strings, tokenizer=tok, prompt_lookup_num_tokens=4)
        assert torch.equal(look, plain), strings
        accepted_mid += sum(model.lookup_stats["accepted"])
    assert accepted_mid > 0
    # a hit on a non-final accepted draft: take the first token of a step that accepted drafts in the run without stop
    # strings, and a string ending with it; the run with the string must cut that step's accept short
    look0 = model.generate(ids, max_new_tokens=n, prompt_lookup_num_tokens=4)
    assert torch.equal(look0, full)
    acc0 = list(model.lookup_stats["accepted"])
    p, cut = 1, 0
    for t, a in enumerate(acc0):
        if a >= 1 and S + p < full.shape[1]:
            for w in (2, 3, 4):
                strings = [tok.decode(full[0, S:S + p + 1].tolist())[-w:]]
                crit = ss.StopStrings.build(tok, strings).criteria
                first = next((q for q in range(S, full.shape[1]) if bool(crit(full[:, :q + 1].cpu(), None)[0])), None)
                if first != S + p:
                    continue
                look = model.generate(ids, max_new_tokens=n, stop_strings=strings, tokenizer=tok, prompt_lookup_num_tokens=4)
                assert torch.equal(look, full[:, :S + p + 1]), strings
                assert model.lookup_stats["accepted"][-1] < a              # the step's accept was cut by the hit
                cut += 1
                break
        p += a + 1
    assert cut >= 1


# ================================================================================================ 4. beams
def test_beam_search_equals_hf(micro):
    """transformers' own _beam_search with the same StopStringCriteria, fed the engine's processed log-probs, returns the same
    sequences and scores."""
    from test_beam_gpu import _Replay, _tie_at_cut
    cfg, model, tok = micro
    B, S, nb, n = 2, 10, 3, 12
    ids = torch.randint(0, 1000, (B, S), generator=torch.Generator().manual_seed(21))
    fk = dict(audio_values=None, inputs_embeds=None, attention_mask=None, audio_token_start_idx=None, audio_lens=None,
              audio_token_len=None, audio_batch_size=None, position_ids=None, audio_waveforms=None, audio_num_frames=None,
              audio_pad_frames=None)
    base, _ = model._beam_search(ids.cuda(), fk, None, n, [], 0, nb, 1.0, False, nb, 1.0, False)
    changed = checked = 0
    K = 2 * nb
    for a, b in ((4, 9), (10, 15), (2, 8), (6, 10), (12, 16)):
        strings = [tok.decode(base[0, S:].tolist())[a:b], tok.decode(base[nb + 1, S:].tolist())[a:b]]
        strings = [x for x in strings if x]
        st = ss.StopStrings.build(tok, strings)
        rec = []

        def hook(eng):
            torch.cuda.synchronize()
            rec.append((eng.logprobs.cpu().clone(), eng.seq[:, :int(eng.cur_len)].cpu().clone(), eng.run_score.cpu().clone()))
            hits.append(eng.beam_hit.view(B, K).sum(-1).max().item())

        hits = []
        seqs, scores = model._beam_search(ids.cuda(), fk, None, n, [], 0, nb, 1.0, False, nb, 1.0, False, step_hook=hook, stop=st)
        seqs, scores = seqs.cpu(), scores.cpu()
        # ambiguous: a top-K cut inside a tie, or more than K - nb hits in a prompt, so finished candidates (all at -1e9 in
        # fp32) must fill running beams and HF's topk orders those exact ties arbitrarily
        if _tie_at_cut(rec, B, nb, K, cfg.vocab_size) or max(hits) > K - nb:
            continue
        checked += 1
        replay = _Replay(ids.repeat_interleave(nb, 0), rec)
        out = _hf_stop(cfg.vocab_size, ids, nb, n, replay, strings, tok)
        assert replay.t == len(rec), (strings, replay.t, len(rec))
        assert torch.equal(out.sequences, seqs), strings
        torch.testing.assert_close(out.sequences_scores, scores, rtol=1e-6, atol=0.0)
        g = model.generate(ids.cuda(), num_beams=nb, num_return_sequences=nb, max_new_tokens=n, stop_strings=strings,
                           tokenizer=tok, return_dict_in_generate=True, output_scores=True)
        assert torch.equal(g.sequences.cpu(), seqs) and torch.equal(g.sequences_scores.cpu(), scores), strings
        changed += not (seqs.shape == base.shape and torch.equal(seqs, base.cpu()))
    assert checked >= 2 and changed >= 1, (checked, changed)


def _hf_stop(V, ids, nb, max_new, replay, strings, tok):
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
        return hf.generate(ids, attention_mask=torch.ones_like(ids), num_beams=nb, num_return_sequences=nb, pad_token_id=0,
                           max_new_tokens=max_new, do_sample=False, output_scores=True, return_dict_in_generate=True,
                           logits_processor=LogitsProcessorList([Replay()]), stop_strings=strings, tokenizer=tok)
