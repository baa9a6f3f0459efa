"""Prompt lookup decoding inside the continuous-batching slot step.

Kernels bit for bit: uvx_lookup_draft_slots against uvx_lookup_draft slot by slot and against HF's
PromptLookupCandidateGenerator plus the budget cap; uvx_lookup_accept_slots against uvx_lookup_accept plus uvx_slot_finish's rule;
the row-mapped penalty / sampler / log-prob kernels against the slot kernels row by row; the row-mapped decode attention against
the unmapped call (contiguous, paged bf16, paged e4m3); the decode-form GEMM's rows at 8, 16 and 32 rows.  SlotScheduler with
prompt_lookup_num_tokens against a plain SlotScheduler of slots * (K + 1) slots (the lookup step's row count): tokens,
log-probs, sessions, the prefix cache, the e4m3 pool, host swap, chunked prompts, graph against eager."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V8B = 128256
NAN = float("nan")


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ host references
def hf_drafts(seq, k, n, eos, max_length, max_new, n_new):
    """HF's candidates for seq (list of ids) with logits_processor=None, then the budget cap n_new + d + 1 <= max_new."""
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor(list(eos), dtype=torch.int64), num_output_tokens=k,
                                         max_matching_ngram_size=n, max_length=max_length)
    out, _ = gen.get_candidates(torch.tensor([seq], dtype=torch.int64))
    return out[0, len(seq):].tolist()[:max(0, max_new - n_new - 1)]


def replay_accepted(tokens, S, k, n, eos, max_new, plain_at=()):
    """The accepted drafts a lookup run must count for the plain run's tokens (prompt + new, a list).  ``plain_at``: the
    sequence lengths at which the request decoded one token without drafting (a mixed step)."""
    total, cur, n_new = 0, S + 1, 1
    while n_new < max_new and tokens[cur - 1] not in eos:
        d = hf_drafts(tokens[:cur], k, n, eos, S + max_new, max_new, n_new) if k and cur not in plain_at else []
        m = 0
        while m < len(d) and cur + m < len(tokens) and tokens[cur + m] == d[m]:
            m += 1
        total += m
        cur += m + 1
        n_new += m + 1
    return total


# ------------------------------------------------------------------------------------------------ 1. draft slots
def _slot_arrays(n_slots, K, seed, long_len=0):
    """Per-slot state of a mix of open, idle, done and prefilling slots; returns (host dict, device tensors)."""
    g = torch.Generator().manual_seed(seed)
    W = max(200, long_len + 64)
    seq = torch.full((n_slots, W), -7, dtype=torch.int64)
    st = dict(cur=[], nn=[], mx=[], k=[], n=[], done=[], act=[], pf=[], pos=[], lens=[], rope=[], tok=[], eos=[])
    for s in range(n_slots):
        kind = ["open", "open", "open", "idle", "done", "prefilling"][s % 6]
        L = long_len if (s == 1 and long_len) else int(torch.randint(1, 150, (1,), generator=g))
        vocab = 3 + s % 4
        seq[s, :L] = torch.randint(0, vocab, (L,), generator=g)
        S = max(1, L - int(torch.randint(0, 6, (1,), generator=g)))
        n_new = L - S
        left = [1, 2, 3, 40][s % 4]
        st["cur"].append(L if kind != "idle" else 0)
        st["nn"].append(n_new if kind != "idle" else 0)
        st["mx"].append(n_new + left)
        st["k"].append(int(torch.randint(0, K + 1, (1,), generator=g)))
        st["n"].append(1 + s % 3)
        st["done"].append(int(kind == "done"))
        st["act"].append(int(kind in ("open", "done")))
        st["pf"].append(int(kind == "prefilling"))
        pad = s % 3
        st["pos"].append(L - 1 if kind != "idle" else 0)
        st["lens"].append(L if kind != "idle" else 1)
        st["rope"].append(L - 1 - pad if kind != "idle" else 0)
        st["tok"].append(int(seq[s, L - 1]) if kind != "idle" else 1000)
    return seq, st


@pytest.mark.parametrize("n_eos", [0, 1, 3])
@pytest.mark.parametrize("K", [1, 3, 7])
def test_draft_slots_match_single_and_hf(ops, K, n_eos):
    n_slots = min(12, 256 // (K + 1))
    for trial in range(3):
        long_len = 32000 if trial == 2 else 0
        seq, st = _slot_arrays(n_slots, K, 100 * K + 10 * n_eos + trial, long_len)
        eos = list(range(n_eos))
        i32 = lambda key: torch.tensor(st[key], dtype=torch.int32, device="cuda")       # noqa: E731
        dseq = seq.cuda()
        R = n_slots * (K + 1)
        tok = torch.zeros(R, dtype=torch.int64, device="cuda")
        nd = torch.full((n_slots,), -3, dtype=torch.int32, device="cuda")
        rows = [torch.full((R,), -9, dtype=torch.int32, device="cuda") for _ in range(7)]
        e = torch.tensor(eos, dtype=torch.int64, device="cuda") if eos else None
        ops.lookup_draft_slots(dseq, torch.tensor(st["tok"], dtype=torch.int64, device="cuda"), i32("cur"), i32("nn"), i32("mx"),
                               i32("k"), i32("n"), i32("done"), i32("act"), i32("pf"), i32("pos"), i32("lens"), i32("rope"), K, e,
                               tok, nd, *rows)
        got_seq, tok, nd = dseq.cpu(), tok.cpu(), nd.cpu()
        rpos, rlens, rrope, pen, idx, rslot, wrow = [r.cpu() for r in rows]
        for s in range(n_slots):
            L, nn, mx, k, n = st["cur"][s], st["nn"][s], st["mx"][s], st["k"][s], st["n"][s]
            openq = st["act"][s] and not st["done"][s] and not st["pf"][s]
            want = []
            if openq and k:
                want = hf_drafts(seq[s, :L].tolist(), k, n, eos, L - nn + mx, mx, nn)
                # the single-sequence kernel on this slot's sequence
                one = seq[s].clone().cuda()
                t1 = torch.zeros(k + 1, dtype=torch.int64, device="cuda")
                d1 = torch.zeros(1, dtype=torch.int32, device="cuda")
                r1 = [torch.zeros(k + 1, dtype=torch.int32, device="cuda") for _ in range(5)]
                c = lambda v: torch.tensor([v], dtype=torch.int32, device="cuda")      # noqa: E731
                ops.lookup_draft(one, c(L), c(nn), mx, k, n, e, c(0), t1, d1, *r1)
                assert int(d1) == len(want) and one.cpu()[L:L + len(want)].tolist() == want
            d = len(want)
            assert int(nd[s]) == d, (s, trial)
            assert got_seq[s, :L].tolist() == seq[s, :L].tolist() and got_seq[s, L:L + d].tolist() == want
            assert torch.equal(got_seq[s, L + d:], seq[s, L + d:])
            r0 = s * (K + 1)
            for i in range(K + 1):
                r, real = r0 + i, i <= d
                j = i if real else 0
                assert int(tok[r]) == (want[i - 1] if 1 <= i <= d else st["tok"][s])
                assert (int(rpos[r]), int(rlens[r]), int(rrope[r])) == (st["pos"][s] + j, st["lens"][s] + j, st["rope"][s] + j)
                assert int(pen[r]) == L + j and int(idx[r]) == (nn + i if real else -1) and int(rslot[r]) == s
                writes = real and (i > 0 or not (st["done"][s] or st["pf"][s]))
                assert int(wrow[r]) == (s if writes else -1), (s, i)


# ------------------------------------------------------------------------------------------------ 2. accept slots
def test_accept_slots_match_single_and_slot_finish(ops):
    g = torch.Generator().manual_seed(11)
    K, n_slots, W = 5, 20, 80
    R = n_slots * (K + 1)
    eos = [9, 10]
    picks = torch.randint(5, 11, (R,), generator=g)
    tok = torch.randint(5, 9, (R,), generator=g)
    nd = torch.randint(0, K + 1, (n_slots,), generator=g).to(torch.int32)
    for s in range(n_slots):             # agree on a random prefix of the drafts
        a = int(torch.randint(0, int(nd[s]) + 1, (1,), generator=g))
        picks[s * (K + 1):s * (K + 1) + a] = tok[s * (K + 1) + 1:s * (K + 1) + 1 + a]
    cur = torch.randint(20, 40, (n_slots,), generator=g).to(torch.int32)
    nn = torch.randint(1, 5, (n_slots,), generator=g).to(torch.int32)
    mx = (nn + nd + 1 + torch.randint(0, 3, (n_slots,), generator=g)).to(torch.int32)
    act = torch.tensor([int(s % 5 != 4) for s in range(n_slots)], dtype=torch.int32)
    done = torch.tensor([int(s % 7 == 3) for s in range(n_slots)], dtype=torch.int32)
    seq = torch.randint(0, 50, (n_slots, W), generator=g)
    for s in range(n_slots):
        seq[s, int(cur[s]):int(cur[s]) + int(nd[s])] = tok[s * (K + 1) + 1:s * (K + 1) + 1 + int(nd[s])]
    pos, lens, rope = cur - 1, cur.clone(), cur - 3
    token = torch.randint(0, 50, (n_slots,), generator=g)
    acc = torch.randint(0, 4, (n_slots,), generator=g).to(torch.int32)
    dev = [t.cuda() for t in (seq, token, done, cur, nn, mx, act, pos, lens, rope, acc)]
    n_open = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    ops.lookup_accept_slots(picks.cuda(), tok.cuda(), nd.cuda(), K, torch.tensor(eos, device="cuda"), dev[0], dev[1], dev[2], dev[3],
                            dev[4], dev[5], dev[6], dev[7], dev[8], dev[9], dev[10], n_open)
    gseq, gtoken, gdone, gcur, gnn, _, _, gpos, glens, grope, gacc = [t.cpu() for t in dev]
    opened = 0
    for s in range(n_slots):
        r0 = s * (K + 1)
        if not act[s] or done[s]:
            assert torch.equal(gseq[s], seq[s]) and (int(gcur[s]), int(gnn[s]), int(gpos[s]), int(gacc[s]), int(gtoken[s])) == \
                (int(cur[s]), int(nn[s]), int(pos[s]), int(acc[s]), int(token[s]))
            continue
        # the single-sequence kernel
        one = seq[s].clone().cuda()
        i32 = lambda v: torch.tensor([int(v)], dtype=torch.int32, device="cuda")     # noqa: E731
        c1, n1, d1 = i32(cur[s]), i32(nn[s]), i32(0)
        ops.lookup_accept(picks[r0:r0 + K + 1].cuda(), tok[r0:r0 + K + 1].cuda(), i32(nd[s]), torch.tensor(eos, device="cuda"), one, c1,
                          n1, int(mx[s]), d1)
        assert torch.equal(gseq[s], one.cpu()) and int(gcur[s]) == int(c1) and int(gnn[s]) == int(n1) and int(gdone[s]) == int(d1)
        m = int(gcur[s]) - int(cur[s]) - 1
        assert int(gacc[s]) == int(acc[s]) + m and int(gtoken[s]) == int(picks[r0 + m])
        # uvx_slot_finish's rule, one token at a time
        p, fin = int(pos[s]), False
        for i in range(m + 1):
            t = int(picks[r0 + i])
            fin = int(nn[s]) + i + 1 >= int(mx[s]) or t in eos
            if not fin:
                p += 1
        assert int(gdone[s]) == int(fin)
        bump = p - int(pos[s])
        assert (int(gpos[s]), int(glens[s]), int(grope[s])) == (p, int(lens[s]) + bump, int(rope[s]) + bump)
        opened += int(not fin)
    assert int(n_open) == opened


# ------------------------------------------------------------------------------------------------ 3. row-mapped pick
@pytest.mark.parametrize("V", [1024, V8B])
def test_row_mapped_pick_matches_slot_kernels(ops, V):
    g = torch.Generator(device="cuda").manual_seed(V)
    n_slots, K, W = 5, 3, 300
    R = n_slots * (K + 1)
    logits = torch.randn(R, V, device="cuda", generator=g) * 3
    logits[2, :] = -float("inf")                             # all -inf
    logits[5, 10:20] = 50.0                                  # a tie at the top
    logits[9, ::2] = logits[9, 1::2]                         # ties everywhere
    seq = torch.randint(0, V, (n_slots, W), device="cuda", generator=g)
    temps = torch.tensor([0.0, 0.7, 1.3, 0.9, 1.0], device="cuda")
    top_k = torch.tensor([0, 50, 0, 20, 7], dtype=torch.int32, device="cuda")
    top_p = torch.tensor([1.0, 1.0, 0.8, 0.9, 0.5], device="cuda")
    pen = torch.tensor([1.3, 1.0, 1.2, 0.8, 1.1], device="cuda")
    active = torch.tensor([1, 1, 1, 1, 0], dtype=torch.int32, device="cuda")
    n_top = torch.tensor([3, -1, 0, 5, -1], dtype=torch.int32, device="cuda")     # an idle slot asks for none
    u = torch.rand(n_slots, W, device="cuda", generator=g)
    cur = torch.tensor([50, 120, 7, 260, 30], dtype=torch.int32)
    row_slot = torch.arange(R, dtype=torch.int32) // (K + 1)
    i = torch.arange(R, dtype=torch.int32) % (K + 1)
    d = torch.tensor([3, 1, 0, 2, 3], dtype=torch.int32)[row_slot.long()]
    row_idx = torch.where(i <= d, 10 * row_slot + i, torch.full_like(i, -1))
    row_len = cur[row_slot.long()] + i
    rs, ri, rl = row_slot.cuda(), row_idx.cuda(), row_len.cuda()
    raw = logits.clone()
    got = logits.clone()
    ops.repetition_penalty_rows_map_(got, seq, pen, active, rs, rl, ri, torch.empty(R, W, device="cuda"))
    pick = torch.full((R,), -5, dtype=torch.int64, device="cuda")
    ops.sample_rows(got, temps, top_k, top_p, u, active, rs, ri, pick)
    cap, nmax = 64, 6
    lp = torch.full((n_slots, cap), 7.0, device="cuda")
    lid = torch.full((n_slots, cap, nmax), -2, dtype=torch.int64, device="cuda")
    ltop = torch.full((n_slots, cap, nmax), 7.0, device="cuda")
    ops.token_logprobs_rows(raw, pick, n_top, rs, ri, lp, lid, ltop)
    for r in range(R):
        s = int(row_slot[r])
        one = slice(s, s + 1)
        if int(row_idx[r]) < 0 or not int(active[s]):
            assert int(pick[r]) == -5, r
            continue
        want = logits[r:r + 1].clone()
        ops.repetition_penalty_slots_(want, seq[one], torch.tensor([int(row_len[r])], dtype=torch.int32, device="cuda"), pen[one],
                                      active[one], torch.empty(1, W, device="cuda"))
        assert torch.equal(got[r], want[0]), r
        wp = torch.full((1,), -5, dtype=torch.int64, device="cuda")
        ops.sample_slots(want, temps[one], top_k[one], top_p[one], u[one], torch.tensor([int(row_idx[r])], dtype=torch.int32,
                                                                                      device="cuda"), active[one], wp)
        assert int(pick[r]) == int(wp), r
        if int(n_top[s]) < 0:
            continue
        wl = torch.full((1, cap), 7.0, device="cuda")
        wi = torch.full((1, cap, nmax), -2, dtype=torch.int64, device="cuda")
        wt = torch.full((1, cap, nmax), 7.0, device="cuda")
        ops.token_logprobs(raw[r:r + 1].contiguous(), wp, n_top[one], torch.tensor([int(row_idx[r])], dtype=torch.int32, device="cuda"),
                           wl, wi, wt)
        c = int(row_idx[r])
        assert torch.equal(lp[s, c].nan_to_num(9), wl[0, c].nan_to_num(9)) and torch.equal(lid[s, c], wi[0, c]), r
        assert torch.equal(ltop[s, c].nan_to_num(9), wt[0, c].nan_to_num(9)), r
    for s in range(n_slots):             # nothing written outside the rows' indices
        used = {int(row_idx[r]) for r in range(R) if int(row_slot[r]) == s and int(row_idx[r]) >= 0}
        if int(n_top[s]) < 0 or not int(active[s]):
            used = set()
        for c in range(cap):
            if c not in used:
                assert float(lp[s, c]) == 7.0


# ------------------------------------------------------------------------------------------------ 4. row-mapped attention
def _pool(cache, table, n_pages, fill):
    """[rows, smax, Hkv, D] -> pool [n_pages, 64, Hkv, D] with row b's tile t at page table[b][t]."""
    rows, smax, Hkv, D = cache.shape
    pool = torch.full((n_pages, 64, Hkv, D), fill, dtype=cache.dtype, device=cache.device)
    for b in range(rows):
        for t in range(smax // 64):
            if table[b][t] >= 0:
                pool[table[b][t]] = cache[b, t * 64:(t + 1) * 64]
    return pool


@pytest.mark.parametrize("D,Hq,Hkv", [(128, 32, 8), (64, 16, 4)])
@pytest.mark.parametrize("form", ["contiguous", "paged", "fp8"])
def test_row_mapped_attention_matches_unmapped(ops, D, Hq, Hkv, form):
    g = torch.Generator().manual_seed(D + len(form))
    rows, smax = 5, 640
    R = 14
    kv_row = torch.tensor([3, 0, 0, 1, 3, 3, 2, 0, 1, 1, 2, 3, 0, 3], dtype=torch.int32)     # row 4 is never read
    lens = torch.randint(1, smax + 1, (R,), generator=g).to(torch.int32)
    lens[:3] = torch.tensor([1, 64, 65], dtype=torch.int32)
    kc = (torch.randn(rows, smax, Hkv, D, generator=g) * 2).to(torch.bfloat16)
    vc = torch.randn(rows, smax, Hkv, D, generator=g).to(torch.bfloat16)
    longest = torch.zeros(rows, dtype=torch.int32)
    for r in range(R):
        longest[kv_row[r]] = max(int(longest[kv_row[r]]), int(lens[r]))
    for b in range(rows):                # keys no row may read are NaN
        kc[b, int(longest[b]):] = NAN
        vc[b, int(longest[b]):] = NAN
    rs = (Hq + 2 * Hkv) * D
    qkv = (torch.randn(R, rs, generator=g) * 2).to(torch.bfloat16).cuda()
    kcd, vcd = kc.cuda(), vc.cuda()
    kl, kr = lens.cuda(), kv_row.cuda()
    got = torch.zeros(R, Hq * D, dtype=torch.bfloat16, device="cuda")
    want = torch.zeros_like(got)
    if form == "contiguous":
        ops.attention_rows(qkv[:, :Hq * D], kcd, vcd, got, Hq, D ** -0.5, kl, kr)
        gk, gv = kcd[kv_row.long()].contiguous(), vcd[kv_row.long()].contiguous()
        ops.attention(qkv.data_ptr(), gk.data_ptr(), gv.data_ptr(), want, R, Hq, Hkv, 1, smax, D,
                      (rs, rs, Hkv * D, smax * Hkv * D, Hkv * D, smax * Hkv * D, Hq * D, Hq * D), D ** -0.5, False, kl)
    else:
        Wt = smax // 64
        n_pages = rows * Wt + 9
        perm = torch.randperm(n_pages, generator=g)[:rows * Wt].view(rows, Wt).to(torch.int32)
        for b in range(rows):
            perm[b, -(-int(longest[b]) // 64):] = -1           # pages past a row's keys are not in its table
        table = perm.cuda()
        sc = None
        if form == "fp8":
            # the NaN tails and the pages nobody's table holds become NaN bytes (0x7F / 0xFF)
            kp = _pool(kcd, perm.tolist(), n_pages, NAN).to(ops.FP8)
            vp = _pool(vcd, perm.tolist(), n_pages, NAN).to(ops.FP8)
            for b in range(rows):
                n = int(longest[b])
                if n % 64:
                    last = int(perm[b, n // 64])
                    assert torch.isnan(kp[last, n % 64:].float()).all() and torch.isnan(vp[last, n % 64:].float()).all()
            sc = torch.tensor([0.5, 2.0], device="cuda")
        else:
            kp = _pool(kcd, perm.tolist(), n_pages, NAN)
            vp = _pool(vcd, perm.tolist(), n_pages, NAN)
        ops.attention_paged(qkv[:, :Hq * D], kp, vp, got, Hq, D ** -0.5, table, kl, kv_scale=sc, kv_row=kr)
        ops.attention_paged(qkv[:, :Hq * D], kp, vp, want, Hq, D ** -0.5, table[kv_row.long()].contiguous(), kl, kv_scale=sc)
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ 5. decode-form GEMM rows
@pytest.mark.parametrize("N,K", [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)])
def test_decode_gemm_rows_at_8_16_32(ops, N, K):
    """The 8B projections (q|k|v, o, gate|up, down): the same 8 activation rows inside calls of 8, 16 and 32 rows, with the
    engine's (default) workspace.  Records whether a row's bits depend on the call's row count (DESIGN.md §6)."""
    g = torch.Generator(device="cuda").manual_seed(N + K)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    x = torch.randn(32, K, device="cuda", generator=g).to(torch.bfloat16)
    res = torch.randn(32, N, device="cuda", generator=g).to(torch.bfloat16)
    outs = {rows: ops.linear(x[:rows].contiguous(), w) for rows in (8, 16, 32)}
    outs_r = {rows: ops.linear(x[:rows].contiguous(), w, residual=res[:rows].contiguous()) for rows in (8, 16, 32)}
    for rows in (16, 32):
        assert torch.equal(outs[rows][:8], outs[8]), rows
        assert torch.equal(outs_r[rows][:8], outs_r[8]), rows
    assert torch.equal(outs[32][:16], outs[16])


# ------------------------------------------------------------------------------------------------ engine and scheduler
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


def looping(model, V):
    """The LM head reads the embedding table and o / down are damped: the fed token dominates its logits, so replies fall into
    loops the lookup catches (a synthetic construction; random weights otherwise never repeat themselves)."""
    lm = model.language_model
    lm.lm_head.weight.data.copy_(lm.model.embed_tokens.weight.data)
    for layer in lm.model.layers:
        layer.self_attn.o_proj.weight.data.mul_(0.05)
        layer.mlp.down_proj.weight.data.mul_(0.05)
    model._tiled = None
    return sharpen(model, V)


@pytest.fixture(scope="module")
def micro():
    cfg, model = build()
    return cfg, looping(model, cfg.vocab_size)


@pytest.fixture(scope="module")
def wide():
    from ultravox_b200.config import PRESETS
    base = PRESETS["v0_5_8b"]
    cfg, model = build("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                       text_config=dict(base["text_config"], num_hidden_layers=2))
    return cfg, looping(model, V8B)


def prompt(seed, S, vocab=1000, loop=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (1, S), generator=g)
    if loop:
        ids[0, S - loop:] = ids[0, 2:2 + loop].clone()
    return dict(input_ids=ids.cuda())


def audio_request(cfg, n_samples, seed, text_pre=8, text_post=5):
    from oracle import logmel as ol
    from ultravox_b200 import ops
    padded, frames = ol.pad_batch([np.random.default_rng(1000 + seed).standard_normal(n_samples).astype(np.float32)])
    g = torch.Generator().manual_seed(seed)
    tok = int(-(-int(frames[0]) // 16))
    ids = torch.randint(0, min(cfg.vocab_size, 1000), (1, text_pre + tok + text_post), generator=g)
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    return dict(input_ids=ids.cuda(), audio_values=mel, audio_token_start_idx=torch.tensor([text_pre]).cuda(),
                audio_lens=torch.tensor([int(frames[0])]).cuda(), audio_token_len=torch.tensor([tok], dtype=torch.int32).cuda(),
                audio_batch_size=torch.ones(1, dtype=torch.int64).cuda())


SETTINGS = [dict(), dict(do_sample=True, temperature=0.8, top_k=40), dict(repetition_penalty=1.3),
            dict(do_sample=True, temperature=1.1, top_p=0.9), dict(do_sample=True, temperature=0.6, repetition_penalty=1.2)]


def workload(cfg, n_req, seed=0, audio=True, vocab=1000):
    """(features, max_new, settings, seed, lookup kwargs) of mixed requests: looped prompts, audio, k = 0, budgets 1..40."""
    reqs = []
    for i in range(n_req):
        S = 20 + (7 * i) % 50
        feats = audio_request(cfg, 16000 + 4000 * (i % 3), seed + i) if audio and i % 4 == 3 else \
            prompt(seed + i, S, vocab, loop=min(S - 4, 6 + i % 10))
        n = [1, 2, 3, 12, 40, 25][i % 6]
        lk = dict(prompt_lookup_num_tokens=0) if i % 5 == 4 else (dict(max_matching_ngram_size=1 + i % 3) if i % 3 else {})
        reqs.append((feats, n, SETTINGS[i % len(SETTINGS)], 1000 + i, lk))
    return reqs


def serve(sched, reqs, lookup=True, logprobs=None):
    ids = []
    for feats, n, settings, seed, lk in reqs:
        kw = dict(settings)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
        if lookup:
            kw.update(lk)
        if logprobs is not None:
            kw["logprobs"] = logprobs
        ids.append(sched.submit(feats, max_new_tokens=n, **kw))
    res = sched.run()
    return [res[i] for i in ids], ids


def track(sched):
    """Wraps the scheduler's engine.step to log every step: (graph kind, {request id: (cur_len, accepted) before the step}) for
    the requests decoding in slots, and to count each request's drafted tokens (n_draft after each lookup step)."""
    eng = sched.engine
    log, drafted, orig = [], {}, eng.step

    def step():
        kind = "mixed" if eng.prefilling is not None else ("lookup" if any(eng._slot_k) else "plain")
        running = {j: r.rid for j, r in sched._running.items()}
        cur, acc = eng.cur_len.tolist(), (eng.accepted.tolist() if eng.K else None)
        log.append((kind, {rid: (cur[j], acc[j] if acc else 0) for j, rid in running.items()}))
        out = orig()
        if kind == "lookup":
            nd = eng.n_draft.tolist()
            for j, rid in running.items():
                drafted[rid] = drafted.get(rid, 0) + nd[j]
        return out
    eng.step = step
    return log, drafted


def _same_logprobs(a, b):
    return torch.equal(a.token_logprobs, b.token_logprobs) and torch.equal(a.top_ids, b.top_ids) and \
        torch.equal(a.top_logprobs, b.top_logprobs)


def _check_against_plain(cfg, model, slots, K, reqs, eos, max_len=160, logprobs=None, **kw):
    from ultravox_b200.serving import SlotScheduler
    lp = dict(max_logprobs=logprobs) if logprobs else {}
    look = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos, prompt_lookup_num_tokens=K, **lp, **kw)
    plain = SlotScheduler(model, slots=slots * (K + 1), max_len=max_len, eos_token_ids=eos, **lp, **kw)
    got, gids = serve(look, reqs, logprobs=logprobs)
    want, wids = serve(plain, reqs, lookup=False, logprobs=logprobs)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), (i, a.tolist(), b.tolist())
    for i, ((feats, n, _, _, lk), seq, rid) in enumerate(zip(reqs, want, gids)):
        S = int(feats["input_ids"].shape[1])
        k = lk.get("prompt_lookup_num_tokens", K)
        expect = replay_accepted(seq[0].tolist(), S, k, lk.get("max_matching_ngram_size") or 2, eos, n)
        assert look.accepted_drafts[rid] == expect, (i, look.accepted_drafts[rid], expect)
    if logprobs:
        for a, b in zip(gids, wids):
            assert _same_logprobs(look.logprobs[a], plain.logprobs[b])
    return look, plain


def test_served_requests_match_plain_engine_of_r_slots(micro):
    cfg, model = micro
    reqs = workload(cfg, 14)
    look, _ = _check_against_plain(cfg, model, 2, 3, reqs, eos=[5, 17])
    assert sum(look.accepted_drafts.values()) > 0
    assert look.engine.captures == 2 and look.engine._mixed_graph is None      # plain + lookup, each once


def test_logprobs_and_k7(micro):
    cfg, model = micro
    _check_against_plain(cfg, model, 4, 7, workload(cfg, 10, seed=50, audio=False), eos=[3], logprobs=4)


def test_served_requests_match_plain_at_8b_widths(wide):
    cfg, model = wide
    reqs = workload(cfg, 8, seed=7, audio=False, vocab=V8B)
    look, _ = _check_against_plain(cfg, model, 2, 3, reqs, eos=[128001], max_len=128, logprobs=2)
    assert sum(look.accepted_drafts.values()) > 0


def test_busy_equals_alone_graph_equals_eager(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    reqs = workload(cfg, 9, seed=30)
    busy = SlotScheduler(model, slots=3, max_len=160, eos_token_ids=[5], prompt_lookup_num_tokens=4)
    got, _ = serve(busy, reqs)
    eager = SlotScheduler(model, slots=3, max_len=160, eos_token_ids=[5], prompt_lookup_num_tokens=4, use_graph=False)
    got_e, _ = serve(eager, reqs)
    for a, b in zip(got, got_e):
        assert torch.equal(a, b)
    for i in (0, 3, 5):
        alone = SlotScheduler(model, slots=3, max_len=160, eos_token_ids=[5], prompt_lookup_num_tokens=4)
        one, _ = serve(alone, [reqs[i]])
        assert torch.equal(one[0], got[i]), i
    plain = SlotScheduler(model, slots=3, max_len=160, eos_token_ids=[5])
    assert not hasattr(plain.engine, "_lk_tok") and plain.engine.K == 0
    assert plain.engine.launches_per_step == busy.engine.launches_per_step and busy.engine.captures == 2
    assert busy.engine.launches_per_lookup_step > busy.engine.launches_per_step


def test_paged_sessions_prefix_cache_fp8_and_swap(micro):
    """Session turns, prefix-cache hits (shared pages byte-identical afterwards), the e4m3 pool and a host swap of a session
    whose last turn rejected drafts: each equals the plain paged scheduler of slots * (K + 1) slots."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    for kw in (dict(kv_pages=80), dict(kv_pages=80, kv_cache_dtype="fp8_e4m3"), dict(kv_pages=80, host_kv_pages=40)):
        runs = []
        swap = None
        for K in (3, None):
            slots = 2 if K else 8
            sched = SlotScheduler(model, slots=slots, max_len=320, eos_token_ids=[5], prompt_lookup_num_tokens=K, **kw)
            _, drafted = track(sched)
            sids = [sched.open_session() for _ in range(3)]
            ctx = {s: prompt(60 + s, 30, loop=10)["input_ids"] for s in sids}
            outs = []
            for turn in range(3):
                rids = []
                for j, s in enumerate(sids):
                    kw2 = dict(SETTINGS[(turn + j) % len(SETTINGS)])
                    if kw2.get("do_sample"):
                        kw2["generator"] = torch.Generator(device="cuda").manual_seed(turn * 10 + j)
                    rids.append((s, sched.submit(dict(input_ids=ctx[s]), max_new_tokens=15, session=s, **kw2)))
                res = sched.run()
                for s, rid in rids:
                    outs.append(res[rid])
                    extra = prompt(200 + turn * 10 + s, 6)["input_ids"]
                    if turn == 0:           # the next turn ends on an early prompt token: its first drafts follow that token's
                        extra[0, -1] = ctx[s][0, 5]         # first occurrence, which the repeating reply does not take
                    ctx[s] = torch.cat([res[rid], extra], dim=1)
                    assert sched.session_length(s) == res[rid].shape[1] - 1
                if kw.get("host_kv_pages") and turn == 1:
                    if swap is None:        # the lookup run: a session whose last turn rejected drafts
                        rejected = [i for i, (s, rid) in enumerate(rids) if drafted.get(rid, 0) > sched.accepted_drafts[rid]]
                        assert rejected, [(drafted.get(rid, 0), sched.accepted_drafts[rid]) for _, rid in rids]
                        swap = rejected[0]
                    sched.offload_session(sids[swap])
                    assert sched.session_on_host(sids[swap])
            runs.append(outs)
        for a, b in zip(*runs):
            assert torch.equal(a, b)
    # prefix cache: shared pages are never written by any step
    runs = []
    for K in (3, None):
        sched = SlotScheduler(model, slots=2 if K else 8, max_len=320, eos_token_ids=[5], prompt_lookup_num_tokens=K, kv_pages=60,
                              prefix_cache=True)
        head = prompt(77, 130)["input_ids"]
        reqs = [(dict(input_ids=torch.cat([head, prompt(80 + i, 10 + i, loop=6)["input_ids"]], 1)), 20, SETTINGS[i % 3], i, {})
                for i in range(6)]
        first, _ = serve(sched, reqs[:1])
        shared = sorted(sched.pool._key)
        assert len(shared) == 2
        snap = (sched.engine.pool_k[:, shared].clone(), sched.engine.pool_v[:, shared].clone())
        rest, ids = serve(sched, reqs[1:])
        assert torch.equal(sched.engine.pool_k[:, shared].view(torch.uint8), snap[0].view(torch.uint8))
        assert torch.equal(sched.engine.pool_v[:, shared].view(torch.uint8), snap[1].view(torch.uint8))
        assert all(sched.cached_tokens[i] > 0 for i in ids)
        runs.append(first + rest)
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_pages_outside_reservations_never_written(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    sched = SlotScheduler(model, slots=3, max_len=200, eos_token_ids=[5], prompt_lookup_num_tokens=5, kv_pages=40)
    sched.engine.pool_k.fill_(NAN)
    sched.engine.pool_v.fill_(NAN)
    reqs = workload(cfg, 6, seed=90, audio=False)
    seen = set()
    orig = sched.pool.reserve

    def reserve(*a, **kw):
        p = orig(*a, **kw)
        if p is not None:
            seen.update(p)
        return p
    sched.pool.reserve = reserve
    serve(sched, reqs)
    untouched = [p for p in range(40) if p not in seen]
    assert untouched
    assert torch.isnan(sched.engine.pool_k[:, untouched].float()).all()
    assert torch.isnan(sched.engine.pool_v[:, untouched].float()).all()


def test_submit_accepts_and_refuses_as_plain(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    look = SlotScheduler(model, slots=2, max_len=64, kv_pages=3, prompt_lookup_num_tokens=3)
    plain = SlotScheduler(model, slots=2, max_len=64, kv_pages=3)
    for S, n in ((60, 4), (60, 5), (30, 34), (30, 35), (150, 20), (1, 63)):
        outcome = []
        for sched in (look, plain):
            try:
                sched.submit(prompt(S, S), max_new_tokens=n)
                outcome.append("ok")
            except ValueError as e:
                outcome.append(str(e))
        assert outcome[0] == outcome[1], (S, n, outcome)


def test_chunked_prompt_while_lookup_slots_decode(micro):
    """Two looping requests decode with lookup steps (and accept drafts); a 300-row prompt is admitted into the slot the short
    one frees, so the long one goes lookup -> mixed (two chunks, no drafting) -> lookup.  The chunked request gets the plain
    engine's bits and drafts after its last chunk; every request's accepted drafts equal the HF replay of its tokens with no
    drafting at the steps it decoded inside a mixed step; graph == eager through the handoffs."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    reqs = [(prompt(21, 40, loop=20), 8, dict(), 0, {}), (prompt(22, 50, loop=30), 120, dict(), 0, {}),
            (prompt(99, 300, loop=40), 30, dict(), 0, {})]
    eos = [5]
    outs = []
    for use_graph in (False, True):              # the graph run's log is checked below
        look = SlotScheduler(model, slots=2, max_len=400, eos_token_ids=eos, prompt_lookup_num_tokens=3, use_graph=use_graph)
        log, _ = track(look)
        got, ids = serve(look, reqs)
        outs.append(got)
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    kinds = [k for k, _ in log]
    first_mixed = kinds.index("mixed")
    last_mixed = len(kinds) - 1 - kinds[::-1].index("mixed")
    assert "lookup" in kinds[:first_mixed] and "lookup" in kinds[last_mixed + 1:] and kinds[first_mixed:last_mixed + 1] == \
        ["mixed"] * (last_mixed + 1 - first_mixed) and last_mixed > first_mixed
    long_id = ids[1]
    cur0, acc0 = log[first_mixed][1][long_id]
    S1, n1 = int(reqs[1][0]["input_ids"].shape[1]), reqs[1][1]
    assert acc0 > 0 and cur0 < S1 + n1                      # it accepted drafts before, and is still open at the handoff
    n_mixed = last_mixed + 1 - first_mixed
    assert log[last_mixed + 1][1][long_id][0] == cur0 + n_mixed       # one token per mixed step, no drafting
    assert look.accepted_drafts[ids[2]] > 0                 # the chunked request drafts after its last chunk
    assert any(k == "lookup" and snap[long_id][1] > acc0 for k, snap in log[last_mixed + 1:] if long_id in snap)
    for (feats, n, _, _, _), seq, rid in zip(reqs, got, ids):
        plain_at = {snap[rid][0] for k, snap in log if k == "mixed" and rid in snap}
        S = int(feats["input_ids"].shape[1])
        assert look.accepted_drafts[rid] == replay_accepted(seq[0].tolist(), S, 3, 2, eos, n, plain_at), rid
    # the chunked request against a plain engine of slots * (K + 1) slots
    plain = SlotScheduler(model, slots=8, max_len=400, eos_token_ids=eos)
    want, _ = serve(plain, reqs, lookup=False)
    assert torch.equal(got[2], want[2])
    assert look.engine.captures == 3                       # plain, lookup and mixed step, each once


def test_served_greedy_request_matches_stepwise_oracle(wide):
    """A greedy request at 8B widths through the lookup step against the fp32 oracle stepped token by token (the bar of
    test_serving_gpu.py::test_served_greedy_request_matches_stepwise_oracle: all but two tokens exact)."""
    from oracle import model as om
    from ultravox_b200.serving import SlotScheduler
    cfg, model = wide
    sched = SlotScheduler(model, slots=2, max_len=96, eos_token_ids=[], prompt_lookup_num_tokens=3)
    feats = prompt(5, 24, V8B, loop=8)
    n_new = 12
    out, rid = serve(sched, [(feats, n_new, {}, 0, {})])
    toks = out[0][0].tolist()
    assert sched.accepted_drafts[rid[0]] > 0
    sd, sh = om.state_dict_fp32(model), om.shapes_from_config(cfg)
    table = sd["language_model.model.embed_tokens.weight"]
    cur = table[feats["input_ids"][0].cpu()][None]
    exact = 0
    for t in range(n_new):
        ref = om.llama_forward(sd, sh, cur, last_only=True).view(-1)
        tok = toks[24 + t]
        assert tok in ref.topk(5).indices.tolist(), t
        exact += int(tok == int(ref.argmax()))
        cur = torch.cat([cur, table[tok][None, None]], dim=1)
    assert exact >= n_new - 2, exact


def test_validation_errors(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    for bad in (0, 32, True, 2.0, "3"):
        with pytest.raises(ValueError, match="prompt_lookup_num_tokens"):
            SlotScheduler(model, slots=2, max_len=64, prompt_lookup_num_tokens=bad)
    with pytest.raises(ValueError, match="rows per step"):
        SlotScheduler(model, slots=65, max_len=64, prompt_lookup_num_tokens=3)
    plain = SlotScheduler(model, slots=2, max_len=64)
    with pytest.raises(ValueError, match="per scheduler"):
        plain.submit(prompt(1, 10), max_new_tokens=3, prompt_lookup_num_tokens=2)
    with pytest.raises(ValueError, match="per scheduler"):
        plain.submit(prompt(1, 10), max_new_tokens=3, max_matching_ngram_size=2)
    look = SlotScheduler(model, slots=2, max_len=64, prompt_lookup_num_tokens=3)
    with pytest.raises(ValueError, match="exceeds"):
        look.submit(prompt(1, 10), max_new_tokens=3, prompt_lookup_num_tokens=4)
    for bad in (-1, True, 1.5):
        with pytest.raises(ValueError, match="prompt_lookup_num_tokens"):
            look.submit(prompt(1, 10), max_new_tokens=3, prompt_lookup_num_tokens=bad)
    for bad in (0, -2, True, 2.5):
        with pytest.raises(ValueError, match="max_matching_ngram_size"):
            look.submit(prompt(1, 10), max_new_tokens=3, max_matching_ngram_size=bad)


def test_infer_many_same_replies_with_lookup():
    from ultravox_b200.data_proc import VoiceSample
    from ultravox_b200.inference import LocalInference
    from ultravox_b200.processing import MelSpec, UltravoxProcessor
    from test_serving_gpu import _ChatTok, wave
    cfg, model = build()
    tok = _ChatTok()
    proc = UltravoxProcessor(MelSpec(feature_size=80), tok, mel_device="cuda")
    inf = LocalInference(model, proc, tok, conversation_mode=False)
    samples = [VoiceSample.from_prompt_and_raw("Listen to <|audio|> and answer", wave(1, 16000), 16000),
               VoiceSample.from_prompt("plain text question without audio plain text question"),
               VoiceSample.from_prompt_and_raw("tell me about <|audio|>", wave(3, 32000), 16000)]
    want = inf.infer_many(samples, max_tokens=9, slots=8)          # the lookup step's 2 * (3 + 1) rows
    got = inf.infer_many(samples, max_tokens=9, slots=2, prompt_lookup_num_tokens=3)
    assert [(o.text, o.input_tokens, o.output_tokens) for o in got] == [(o.text, o.input_tokens, o.output_tokens) for o in want]


def test_served_requests_match_plain_engine_of_same_slots_at_8b_widths(wide):
    """The decode-form GEMM gives a row the same bits at 8, 16 and 32 rows (test_decode_gemm_rows_at_8_16_32), so at the 8B
    widths a lookup engine of 8 slots x (3 + 1) rows also equals a plain engine of the same 8 slots."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = wide
    reqs = workload(cfg, 10, seed=70, audio=False, vocab=V8B)
    look = SlotScheduler(model, slots=8, max_len=128, eos_token_ids=[128001], prompt_lookup_num_tokens=3)
    plain = SlotScheduler(model, slots=8, max_len=128, eos_token_ids=[128001])
    got, ids = serve(look, reqs)
    want, _ = serve(plain, reqs, lookup=False)
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), i
    assert sum(look.accepted_drafts[i] for i in ids) > 0
