"""Paged KV cache: the paged attention kernels, the page map and the page copy against their contiguous twins (bit for bit, with
every page that holds no live data NaN), PagedSlotDecodeEngine against SlotDecodeEngine (bit for bit, also with a pool too
small to admit every slot at once, at the 8B widths, graph and eager), conversation sessions against chained
generate(past_key_values=...) calls, and the capacity a shared pool gives."""
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def build(name="micro", **kw):
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    cfg = preset(name, **kw)
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def build_8b():
    from ultravox_b200.config import PRESETS
    base = PRESETS["v0_5_8b"]
    return build("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=2, vocab_size=32000))


def to_pool(k, pages, n_pages):
    """Contiguous rows k [B, S, Hkv, D] -> a NaN pool [n_pages, 64, Hkv, D] with row b's tile t in page pages[b][t]."""
    B, S, Hkv, D = k.shape
    pool = torch.full((n_pages, 64, Hkv, D), NAN, dtype=k.dtype, device=k.device)
    for b in range(B):
        for t in range(-(-S // 64)):
            if pages[b][t] < 0:
                continue
            n = min(64, S - 64 * t)
            pool[pages[b][t], :n] = k[b, 64 * t:64 * t + n]
    return pool


def shuffled_table(B, W, n_pages, seed):
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(n_pages, generator=g)[:B * W].view(B, W)
    return perm.to(torch.int32)


# ================================================================================================ 1. kernels
@pytest.mark.parametrize("Hq,Hkv,D", [(32, 8, 128), (4, 2, 64)])
def test_attention_paged_matches_contiguous(ops, Hq, Hkv, D):
    lens = [1, 63, 64, 65, 300, 4000]
    B, smax = len(lens), 4032
    W = smax // 64
    g = torch.Generator().manual_seed(D)
    kc = (torch.randn(B, smax, Hkv, D, generator=g) * 2).to(torch.bfloat16).cuda()
    vc = torch.randn(B, smax, Hkv, D, generator=g).to(torch.bfloat16).cuda()
    for b, n in enumerate(lens):            # the tail past each row's length holds NaN in both layouts
        kc[b, n:] = NAN
        vc[b, n:] = NAN
    rs = (Hq + 2 * Hkv) * D
    qkv = (torch.randn(B, rs, generator=g) * 2).to(torch.bfloat16).cuda()
    kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    want = torch.zeros(B, Hq * D, dtype=torch.bfloat16, device="cuda")
    ops.attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), want, B, Hq, Hkv, 1, smax, D,
                  (rs, rs, Hkv * D, smax * Hkv * D, Hkv * D, smax * Hkv * D, Hq * D, Hq * D), D ** -0.5, False, kv_len)
    n_pages = B * W + 7
    table = shuffled_table(B, W, n_pages, 3)
    for b, n in enumerate(lens):
        table[b, -(-n // 64):] = -1         # entries past a row's pages are never read
    kp, vp = to_pool(kc, table.tolist(), n_pages), to_pool(vc, table.tolist(), n_pages)
    got = torch.zeros_like(want)
    ops.attention_paged(qkv[:, :Hq * D], kp, vp, got, Hq, D ** -0.5, table.cuda(), kv_len)
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, want)


@pytest.mark.parametrize("C", [64, 70, 248])
def test_attention_indexed_paged_matches_indexed(ops, C):
    Hq, Hkv, D = 32, 8, 128
    slots, smax = 3, 4096 + 256
    W = smax // 64
    j = 1
    g = torch.Generator().manual_seed(C)
    kc = (torch.randn(slots, smax, Hkv, D, generator=g) * 2).to(torch.bfloat16).cuda()
    vc = torch.randn(slots, smax, Hkv, D, generator=g).to(torch.bfloat16).cuda()
    rs = (Hq + 2 * Hkv) * D
    qkv = (torch.randn(C, rs, generator=g) * 2).to(torch.bfloat16).cuda()
    q = qkv[:, :Hq * D].unsqueeze(0)
    i32 = dict(dtype=torch.int32, device="cuda")
    n_pages = slots * W + 5
    table = shuffled_table(slots, W, n_pages, C)
    kp, vp = to_pool(kc, table.tolist(), n_pages), to_pool(vc, table.tolist(), n_pages)
    table = table.cuda()
    for past in (0, 1, 63, 64, 300, 4000):
        end = past + C
        args = (torch.tensor([j], **i32), torch.tensor([past], **i32), torch.tensor([end], **i32))
        want = torch.zeros(1, C, Hq * D, dtype=torch.bfloat16, device="cuda")
        ops.attention_indexed(q, kc, vc, want, Hq, D ** -0.5, *args)
        t2 = table.clone()
        t2[j, -(-end // 64):] = -1
        kp2, vp2 = kp.clone(), vp.clone()
        for r in range(slots):               # pages of the other rows, and of this row past its keys, hold NaN
            dead = table[r].long() if r != j else table[j, -(-end // 64):].long()
            kp2[dead] = NAN
            vp2[dead] = NAN
        got = torch.zeros_like(want)
        ops.attention_indexed_paged(q, kp2, vp2, got, Hq, D ** -0.5, t2, *args)
        assert torch.isfinite(got.float()).all(), past
        assert torch.equal(got, want), past


@pytest.mark.parametrize("Hq,Hkv,D", [(32, 8, 128), (4, 2, 64)])
def test_page_map_and_append_match_contiguous(ops, Hq, Hkv, D):
    R, slots, smax = 24, 4, 256
    W = smax // 64
    g = torch.Generator().manual_seed(11 + D)
    inv = 1.0 / (500000.0 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    cos, sin = ops.rope_tables(inv, smax, "cuda")
    qkv = torch.randn(R, (Hq + 2 * Hkv) * D, generator=g).to(torch.bfloat16).cuda()
    crow = torch.randint(0, slots, (R,), generator=g)
    crow[::5] = -1
    pos = torch.randperm(smax, generator=g)[:R]
    frozen = torch.zeros(R // 2, dtype=torch.int32)
    frozen[3] = 1                            # a done row writes nothing
    rope = torch.randint(0, smax, (R,), generator=g)
    i32 = lambda t: t.to(torch.int32).cuda()
    crow_eff = crow.clone()
    crow_eff[3] = -1
    sentinel = 7.0
    kc = torch.full((slots, smax, Hkv, D), sentinel, dtype=torch.bfloat16, device="cuda")
    vc = kc.clone()
    want = qkv.clone()
    ops.rope_kv_append_map_(want, Hq, Hkv, D, cos, sin, i32(rope), kc, vc, i32(crow_eff), i32(pos))
    n_pages = slots * W + 3
    table = shuffled_table(slots, W, n_pages, 5).cuda()
    page, off = torch.zeros(R, dtype=torch.int32, device="cuda"), torch.zeros(R, dtype=torch.int32, device="cuda")
    ops.kv_page_map(table, i32(crow), i32(pos), page, off, frozen=i32(frozen))
    exp_page = torch.where(crow_eff >= 0, table.cpu()[crow_eff.clamp_min(0), pos // 64], torch.full_like(crow, -1))
    assert torch.equal(page.cpu(), exp_page.to(torch.int32))
    assert torch.equal(off.cpu(), torch.where(crow_eff >= 0, pos % 64, torch.zeros_like(pos)).to(torch.int32))
    kp = torch.full((n_pages, 64, Hkv, D), sentinel, dtype=torch.bfloat16, device="cuda")
    vp = kp.clone()
    got = qkv.clone()
    ops.rope_kv_append_map_(got, Hq, Hkv, D, cos, sin, i32(rope), kp, vp, page, off)
    assert torch.equal(got, want)
    tl = table.tolist()
    assert torch.equal(kp, to_pool(kc, tl, n_pages).nan_to_num(sentinel)) and torch.equal(vp, to_pool(vc, tl, n_pages).nan_to_num(sentinel))


def test_pages_copy_round_trip(ops):
    L, smax, Hkv, D = 3, 320, 8, 128
    n_pages = 16
    g = torch.Generator().manual_seed(1)
    k = torch.randn(L, 1, smax, Hkv, D, generator=g).to(torch.bfloat16).cuda()
    v = torch.randn(L, 1, smax, Hkv, D, generator=g).to(torch.bfloat16).cuda()
    pages = torch.tensor([9, 2, 14, 0, 5], dtype=torch.int32, device="cuda")
    kp = torch.full((L, n_pages, 64, Hkv, D), NAN, dtype=torch.bfloat16, device="cuda")
    vp = kp.clone()
    p0, p1 = 70, 300
    ops.kv_pages_copy(k, v, kp, vp, pages, p0, p1, to_pages=True)
    untouched = [p for p in range(n_pages) if p not in pages.tolist()]
    assert torch.isnan(kp[:, untouched].float()).all() and torch.isnan(vp[:, untouched].float()).all()
    for p in (p0, 127, 128, p1 - 1):
        assert torch.equal(kp[:, pages[p // 64], p % 64], k[:, 0, p]) and torch.equal(vp[:, pages[p // 64], p % 64], v[:, 0, p])
    assert torch.isnan(kp[:, 2, :p0 - 64].float()).all()       # positions before p0 of a partly copied page are not written
    k2, v2 = torch.full_like(k, NAN), torch.full_like(v, NAN)
    ops.kv_pages_copy(k2, v2, kp, vp, pages, p0, p1, to_pages=False)
    assert torch.equal(k2[:, :, p0:p1], k[:, :, p0:p1]) and torch.equal(v2[:, :, p0:p1], v[:, :, p0:p1])
    assert torch.isnan(k2[:, :, :p0].float()).all() and torch.isnan(k2[:, :, p1:].float()).all()


# ================================================================================================ 2. paged engine == contiguous
def _serve(sched, reqs):
    ids = []
    for feats, n, settings, seed in reqs:
        kw = dict(settings)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
        ids.append(sched.submit(feats, max_new_tokens=n, **kw))
    res = sched.run()
    return [res[i] for i in ids]


def _poison(sched):
    eng = sched.engine
    for t in ((eng.pool_k, eng.pool_v) if hasattr(eng, "pool_k") else ()) + (eng.cache.k, eng.cache.v):
        t.fill_(NAN)


def _compare(model, reqs, slots, max_len, kv_pages, use_graph=True, eos=None):
    from ultravox_b200.serving import SlotScheduler
    ref = SlotScheduler(model, slots=slots, max_len=max_len, sync_every=3, eos_token_ids=eos)
    _poison(ref)
    want = _serve(ref, reqs)
    paged = SlotScheduler(model, slots=slots, max_len=max_len, sync_every=3, kv_pages=kv_pages, use_graph=use_graph, eos_token_ids=eos)
    _poison(paged)
    got = _serve(paged, reqs)
    for i, (x, y) in enumerate(zip(got, want)):
        assert torch.equal(x, y), i
    assert paged.free_pages == kv_pages
    return ref, paged


def test_paged_engine_equals_contiguous_busy():
    """The mixed workload of the chunked-prefill busy test (greedy, top-k, top-p, repetition penalty, one chunked audio prompt,
    8 slots): identical sequences from the paged and the contiguous engine, with a pool that fits every slot and with one
    that makes requests wait for pages; graph == eager; each graph captured once."""
    from test_chunked_prefill_gpu import _busy_requests, long_audio_request
    cfg, model = build()
    reqs = _busy_requests(cfg, long_audio_request(cfg, 45, 2))
    ref, paged = _compare(model, reqs, 8, 512, 64)
    assert paged.engine.captures == 2 == ref.engine.captures
    _, small = _compare(model, reqs, 8, 512, 8)           # the long request alone needs 5 of the 8 pages
    assert small.engine.captures == 2
    _, eager = _compare(model, reqs, 8, 512, 64, use_graph=False)
    assert eager.engine.captures == 0


def test_paged_engine_equals_contiguous_8b_widths():
    from test_serving_gpu import _mixed_requests
    cfg, model = build_8b()
    reqs = _mixed_requests(cfg, 10, 1, audio=False)
    _compare(model, reqs, 8, 64, 12)


# ================================================================================================ 3. sessions == generate()
def _turn_features(cfg, prev: torch.Tensor, n_samples: int, seed: int, text_pre=6, text_post=4):
    """The next turn of a conversation: the previous sequence (earlier audio stays as its placeholder ids), then text, one new
    clip's placeholders and text, with the new clip's features (as LocalInference's conversation mode builds them)."""
    from test_serving_gpu import audio_request
    a = audio_request(cfg, n_samples, seed, text_pre=text_pre, text_post=text_post)
    P = prev.shape[1]
    a["input_ids"] = torch.cat([prev, a["input_ids"]], dim=1)
    a["audio_token_start_idx"] = a["audio_token_start_idx"] + P
    return a


def _generate_chain(model, cfg, first, n_turns, max_new, eos, settings):
    outs, past, feats = [], None, first
    for t in range(n_turns):
        o = model.generate(max_new_tokens=max_new, eos_token_id=eos, past_key_values=past, return_dict_in_generate=True,
                           **feats, **settings)
        outs.append(o.sequences)
        past = o.past_key_values
        feats = _turn_features(cfg, o.sequences, 12000 + 4000 * t, 50 + t)
    return outs


def _session_chain(sched, cfg, first, n_turns, max_new, settings):
    sid = sched.open_session()
    outs, feats = [], first
    for t in range(n_turns):
        rid = sched.submit(feats, max_new_tokens=max_new, session=sid, **settings)
        seq = sched.run()[rid]
        outs.append(seq)
        assert sched.session_length(sid) == seq.shape[1] - 1
        feats = _turn_features(cfg, seq, 12000 + 4000 * t, 50 + t)
    return sid, outs


def test_session_turns_equal_chained_generate():
    from test_serving_gpu import audio_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    first = audio_request(cfg, 16000, 1)
    probe = model.generate(max_new_tokens=10, **first)
    eos = [int(probe[0, first["input_ids"].shape[1] + 3])]
    for settings, e in (({}, None), (dict(repetition_penalty=1.3), None), ({}, eos)):
        want = _generate_chain(model, cfg, first, 3, 10, e, settings)
        sched = SlotScheduler(model, slots=1, max_len=512, kv_pages=16, eos_token_ids=e)
        _poison(sched)
        sid, got = _session_chain(sched, cfg, first, 3, 10, settings)
        for t, (x, y) in enumerate(zip(got, want)):
            assert torch.equal(x, y), (settings, e, t)
        if e is not None:
            assert int(got[0][0, -1]) == eos[0] and got[0].shape[1] < first["input_ids"].shape[1] + 10
        sched.close_session(sid)
        assert sched.free_pages == 16 and sched.engine.captures == 1


def test_interleaved_sessions_equal_alone():
    """8 conversations x 3 turns through 4 slots, each next turn submitted from on_tokens as the previous reply arrives, give
    the same bits as each conversation alone in a 4-slot engine."""
    from test_serving_gpu import audio_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    firsts = [audio_request(cfg, 8000 + 2000 * i, 300 + i) for i in range(8)]
    settings = [{}, dict(do_sample=True, temperature=0.8, top_k=40), dict(repetition_penalty=1.2)]

    def kw(i, t):
        s = dict(settings[(i + t) % 3])
        if s.get("do_sample"):
            s["generator"] = torch.Generator(device="cuda").manual_seed(1000 * i + t)
        return s

    def serve(convs):
        sched = SlotScheduler(model, slots=4, max_len=512, kv_pages=48, sync_every=3)
        _poison(sched)
        state = {}
        for i in convs:
            sid = sched.open_session()
            rid = sched.submit(firsts[i], max_new_tokens=6 + i, session=sid, **kw(i, 0))
            state[rid] = (i, sid, 0)
        out = {i: [] for i in convs}

        def on_tokens(rid, seq):
            i, sid, t = state.pop(rid)
            out[i].append(seq)
            if t + 1 < 3:
                nxt = sched.submit(_turn_features(cfg, seq, 9000 + 1000 * t, 70 + i), max_new_tokens=5 + t, session=sid,
                                   **kw(i, t + 1))
                state[nxt] = (i, sid, t + 1)
            else:
                sched.close_session(sid)
        sched.run(on_tokens)
        assert not state and sched.free_pages == 48 and sched.engine.captures == 1
        return out

    together = serve(range(8))
    for i in range(8):
        alone = serve([i])[i]
        for t in range(3):
            assert torch.equal(together[i][t], alone[t]), (i, t)


def _ulps(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.float(), b.float()
    e = torch.floor(torch.log2(b.abs().clamp_min(2.0 ** -20)))
    return float(((a - b).abs() / torch.exp2(e - 7)).max())


def test_long_suffix_turn_is_chunked_from_past():
    """A second turn whose suffix (a 45 s clip) exceeds 256 rows is prefilled in chunks from done = P: first-token logits within
    3e-2 of generate()'s and the same first token, and its pages within 4 bf16 ulps of generate()'s cache (whole-suffix prefill)."""
    from test_chunked_prefill_gpu import long_audio_request
    from test_serving_gpu import audio_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    first = audio_request(cfg, 16000, 4)
    sched = SlotScheduler(model, slots=1, max_len=1024, kv_pages=32)
    _poison(sched)
    sid = sched.open_session()
    rid = sched.submit(first, max_new_tokens=6, session=sid)
    seq1 = sched.run()[rid]
    P = sched.session_length(sid)
    nxt = long_audio_request(cfg, 45, 3)
    nxt["input_ids"] = torch.cat([seq1, nxt["input_ids"]], dim=1)
    nxt["audio_token_start_idx"] = nxt["audio_token_start_idx"] + seq1.shape[1]
    S = nxt["input_ids"].shape[1]
    assert S - P > 256
    rid = sched.submit(nxt, max_new_tokens=4, session=sid)
    seq2 = sched.run()[rid]
    eng = sched.engine
    assert eng.captures == 2
    first_logits = eng._chunk_logits.float().view(-1)
    feats = {k: v for k, v in nxt.items() if k != "input_ids"}
    o1 = model.generate(max_new_tokens=6, return_dict_in_generate=True, **first)
    assert torch.equal(o1.sequences, seq1)
    emb = model.prompt_embeds(nxt["input_ids"], **feats)
    cache = o1.past_key_values.grown(S + 4)
    ref = model.forward(nxt["input_ids"][:, P:], None, emb[:, P:].contiguous(), past_key_values=cache, logits_to_keep=1).logits.view(-1)
    assert float((first_logits - ref).norm() / ref.norm()) < 3e-2
    assert int(seq2[0, S]) == int(ref.argmax())
    pages = sched.pool.session(sid).pages
    kp = torch.cat([eng.pool_k[:, p] for p in pages], dim=1)[:, :S]
    vp = torch.cat([eng.pool_v[:, p] for p in pages], dim=1)[:, :S]
    assert torch.equal(kp[:, :P], cache.k[:, 0, :P]) and torch.equal(vp[:, :P], cache.v[:, 0, :P])
    ku, vu = _ulps(kp, cache.k[:, 0, :S]), _ulps(vp, cache.v[:, 0, :S])
    print(f"chunked session turn vs generate()'s whole-suffix cache: k {ku:.1f} ulp, v {vu:.1f} ulp")
    assert ku <= 4 and vu <= 4, (ku, vu)


# ================================================================================================ 4. capacity
def test_pool_serves_more_conversations_than_contiguous_memory():
    """A pool of 24 pages (1536 positions, less than one 1024-position row per each of 4 slots) keeps 6 conversations open
    at once, more positions in total than its memory would hold as contiguous max_len rows; free_pages returns to 24."""
    from test_serving_gpu import text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    sched = SlotScheduler(model, slots=4, max_len=1024, kv_pages=24)
    assert sched.free_pages == 24 and 24 * 64 < 4 * 1024
    sids = [sched.open_session() for _ in range(6)]
    rids = {sched.submit(text_request(cfg, 180, 900 + i), max_new_tokens=8, session=s): s for i, s in enumerate(sids)}
    res = sched.run()
    total = sum(sched.session_length(s) for s in sids)
    assert len(res) == 6 and total > (24 * 64 // 1024) * 1024, total
    for i, s in enumerate(sids):             # a second turn for each: suffix-only prefill into the pages they hold
        seq = res[next(r for r, v in rids.items() if v == s)]
        sched.submit(dict(input_ids=torch.cat([seq, text_request(cfg, 20, 950 + i)["input_ids"]], dim=1)), max_new_tokens=4,
                     session=s)
    sched.run()
    assert sum(sched.session_length(s) for s in sids) > total
    for s in sids:
        sched.close_session(s)
    assert sched.free_pages == 24
