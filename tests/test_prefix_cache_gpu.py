"""Prefix cache on the paged KV pool (SlotScheduler(kv_pages=N, prefix_cache=True)): every request served after a hit equals
generate(its ids, past_key_values=<the shared pages gathered into a cache row>), bit for bit (greedy, top-k / top-p sampling,
repetition penalty, audio and text, 8 slots, graph and eager, and at the 8B widths); shared pages are never written; a chunked
donor; sessions that open with the same system prompt; eviction in a short pool; no shared prefix gives the bits of the cache
off; a served hit against the stepwise fp32 oracle."""
import pytest
import torch

from test_chunked_prefill_gpu import _busy_requests, long_audio_request, oracle_bar
from test_paged_kv_gpu import _poison, _turn_features, build, build_8b
from test_serving_gpu import audio_request, text_request

pytestmark = pytest.mark.gpu

PAGE = 64


def system_prompt(cfg, n, seed=77):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, min(cfg.vocab_size, 1000), (1, n), generator=g).cuda()


def after(sys_ids, feats):
    """``feats`` (one request's processor output) with ``sys_ids`` in front of its ids."""
    out = dict(feats, input_ids=torch.cat([sys_ids, feats["input_ids"]], dim=1))
    if "audio_token_start_idx" in feats:
        out["audio_token_start_idx"] = feats["audio_token_start_idx"] + sys_ids.shape[1]
    return out


def settings_kw(settings, seed):
    kw = dict(settings)
    if kw.get("do_sample"):
        kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
    return kw


def pages_of(ids):
    """The token ids of the full pages of ``ids`` [1, S], as the prefix index keys them."""
    head = ids[0].tolist()
    return [tuple(head[i:i + PAGE]) for i in range(0, len(head) // PAGE * PAGE, PAGE)]


def gathered(sched, ids, P):
    """The first P positions of ``ids`` as the pool caches them, gathered into a one-row cache (``ops.kv_pages_copy``)."""
    from ultravox_b200 import ops
    from ultravox_b200.model import KVCache
    eng = sched.engine
    pages = sched.pool.match(pages_of(ids[:, :P]))
    assert len(pages) * PAGE == P
    L, _, _, hkv, d = eng.pool_k.shape
    k = torch.full((L, 1, P, hkv, d), float("nan"), dtype=torch.bfloat16, device="cuda")
    v = torch.full_like(k, float("nan"))
    ops.kv_pages_copy(k, v, eng.pool_k, eng.pool_v, torch.tensor(pages, dtype=torch.int32, device="cuda"), 0, P, to_pages=False)
    return KVCache(k, v, P)


def check_against_generate(model, sched, reqs, res, rids, eos=None):
    """Each served request == generate() with its cached prefix as past_key_values (or alone when it missed)."""
    hits = 0
    for rid, (feats, n, settings, seed) in zip(rids, reqs):
        P = sched.cached_tokens[rid]
        past = gathered(sched, feats["input_ids"], P) if P else None
        want = model.generate(max_new_tokens=n, eos_token_id=eos, past_key_values=past, **feats, **settings_kw(settings, seed))
        assert torch.equal(res[rid], want), (rid, P)
        hits += P > 0
    return hits


def serve(sched, reqs):
    rids = [sched.submit(f, max_new_tokens=n, **settings_kw(s, seed)) for f, n, s, seed in reqs]
    return rids, sched.run()


SETTINGS = [{}, dict(do_sample=True, temperature=0.7, top_k=50), dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9),
            dict(repetition_penalty=1.3), dict(do_sample=True, temperature=0.8, top_p=0.6, repetition_penalty=1.2)]


def _hit_requests(cfg, sys_ids, n):
    reqs = []
    for i in range(n):
        f = audio_request(cfg, 8000 + 4000 * (i % 3), 100 + i) if i % 3 == 0 else text_request(cfg, 5 + 3 * i, 200 + i)
        reqs.append((after(sys_ids, f), 4 + (7 * i) % 17, SETTINGS[i % len(SETTINGS)], 300 + i))
    return reqs


# ================================================================================================ 1. hits == generate()
def _one_slot_hits(model, sys_ids, donor, reqs):
    """Through one slot (the decode step then runs the matrix-vector kernels generate() runs at one stream): the donor, then
    each request, every one a hit that equals generate() over its gathered prefix."""
    from ultravox_b200.serving import SlotScheduler
    sched = SlotScheduler(model, slots=1, max_len=512, kv_pages=32, prefix_cache=True)
    _poison(sched)
    serve(sched, [donor])
    rids, res = serve(sched, reqs)
    P = (sys_ids.shape[1] // PAGE) * PAGE
    assert [sched.cached_tokens[r] for r in rids] == [P] * len(reqs)
    assert check_against_generate(model, sched, reqs, res, rids) == len(reqs)
    assert sched.engine.captures == 1 and sched.free_pages == 32
    return sched


def test_hits_equal_generate():
    """Greedy, top-k, top-p, repetition penalty, audio and text requests that hit a 3-page system prompt == generate() with
    the prompt's pages gathered out of the pool as past_key_values, bit for bit; one greedy hit also passes the stepwise fp32
    oracle bar."""
    from oracle import model as om
    cfg, model = build()
    sys_ids = system_prompt(cfg, 3 * PAGE + 10)
    donor = (after(sys_ids, text_request(cfg, 12, 1)), 6, {}, 0)
    reqs = _hit_requests(cfg, sys_ids, 10)
    sched = _one_slot_hits(model, sys_ids, donor, reqs)
    i = next(k for k, r in enumerate(reqs) if not r[2] and "audio_values" not in r[0])
    sd, sh = om.state_dict_fp32(model), om.shapes_from_config(cfg)
    rid = sched.submit(reqs[i][0], max_new_tokens=reqs[i][1])
    seq = sched.run()[rid]
    assert sched.cached_tokens[rid] == 3 * PAGE
    ids = reqs[i][0]["input_ids"].cpu()
    oracle_bar(sd, sh, sd["language_model.model.embed_tokens.weight"][ids], seq, ids.shape[1], reqs[i][1])


def test_busy_hits_never_write_shared_pages():
    """A donor registers a 3-page system prompt; then 20 requests (audio and text, every sampling setting) that all open with
    it go through 8 slots: every one hits, the shared pages keep their bytes, each request equals itself served alone after
    the same donor, graph == eager, and the step graph is captured once."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    sys_ids = system_prompt(cfg, 3 * PAGE + 10)
    donor = (after(sys_ids, text_request(cfg, 12, 1)), 6, {}, 0)
    reqs = _hit_requests(cfg, sys_ids, 20)

    def engine(use_graph=True):
        sched = SlotScheduler(model, slots=8, max_len=512, sync_every=3, kv_pages=64, prefix_cache=True, use_graph=use_graph)
        _poison(sched)
        (d,), _ = serve(sched, [donor])
        assert sched.cached_tokens[d] == 0 and sched.cached_pages == 3
        return sched

    out = {}
    for use_graph in (True, False):
        sched = engine(use_graph)
        eng = sched.engine
        cached = sched.pool.match(pages_of(sys_ids))
        assert len(cached) == 3
        snap = (eng.pool_k[:, cached].view(torch.int16).clone(), eng.pool_v[:, cached].view(torch.int16).clone())
        rids, res = serve(sched, reqs)
        assert all(sched.cached_tokens[r] == 3 * PAGE for r in rids)
        assert torch.equal(eng.pool_k[:, cached].view(torch.int16), snap[0])
        assert torch.equal(eng.pool_v[:, cached].view(torch.int16), snap[1])
        assert sched.free_pages == 64 and sched.pool.match(pages_of(sys_ids)) == cached
        assert eng.captures == (1 if use_graph else 0)
        out[use_graph] = [res[r] for r in rids]
    for i, (x, y) in enumerate(zip(out[True], out[False])):
        assert torch.equal(x, y), i
    alone = engine()
    for i, r in enumerate(reqs):
        (rid,), res = serve(alone, [r])
        assert alone.cached_tokens[rid] == 3 * PAGE and torch.equal(res[rid], out[True][i]), i
    assert alone.engine.captures == 1


def test_hits_at_8b_widths_and_bit_dependence():
    """The 8B widths (two layers): hits equal generate() over the gathered prefix.  Also records whether a hit's K / V and
    tokens equal those of prefilling the whole prompt itself (they need not: the donor's row count picked the GEMM tiling)."""
    from ultravox_b200.model import KVCache
    cfg, model = build_8b()
    sys_ids = system_prompt(cfg, 2 * PAGE + 5)
    donor = (after(sys_ids, text_request(cfg, 40, 400)), 6, {}, 0)          # 173 rows
    reqs = [(after(sys_ids, text_request(cfg, 3 + 2 * i, 401 + i)), 6 + i, SETTINGS[i % 5], 500 + i) for i in range(5)]
    sched = _one_slot_hits(model, sys_ids, donor, reqs)
    # bit dependence: request 0's shared K / V came from the donor's 173-row prefill; its own prefill has 138 rows
    ids = reqs[0][0]["input_ids"]
    own = model.new_cache(1, ids.shape[1])
    model.forward(ids, past_key_values=KVCache(own.k, own.v), logits_to_keep=1)
    shared = gathered(sched, ids, 2 * PAGE)
    kv_equal = torch.equal(shared.k, own.k[:, :, :2 * PAGE]) and torch.equal(shared.v, own.v[:, :, :2 * PAGE])
    hit = model.generate(max_new_tokens=reqs[0][1], past_key_values=shared, **reqs[0][0])
    alone = model.generate(max_new_tokens=reqs[0][1], **reqs[0][0])
    print(f"prefix-cache bit dependence at the 8B widths: shared K/V equal to the request's own prefill: {kv_equal}; "
          f"tokens equal: {torch.equal(alone, hit)}")


# ================================================================================================ 2. a chunked donor
def test_chunked_donor():
    """A donor of more than 256 rows is prefilled in chunks: a request admitted during its chunks misses (and registers its own
    pages), requests after its last chunk hit its pages; a hit whose suffix is still over 256 rows is chunked from P, with first-token logits within
    3e-2 of generate()'s over the gathered prefix and the same first token."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    sys_ids = system_prompt(cfg, 3 * PAGE, seed=78)
    donor = (after(sys_ids, text_request(cfg, 100, 1)), 5, {}, 0)           # 292 rows: chunked
    behind = (after(sys_ids, text_request(cfg, 9, 2)), 5, {}, 0)             # 201 rows: B = 1, admitted during the chunks
    sched = SlotScheduler(model, slots=8, max_len=1024, sync_every=3, kv_pages=96, prefix_cache=True)
    _poison(sched)
    (d, b), res = serve(sched, [donor, behind])
    assert sched.cached_tokens == {d: 0, b: 0} and sched.engine.captures == 2
    assert sched.cached_pages == 3                          # the request behind registered first; the donor's pages stay private
    # the donor alone: its pages are cached once its last chunk has run
    sched = SlotScheduler(model, slots=8, max_len=1024, sync_every=3, kv_pages=96, prefix_cache=True)
    _poison(sched)
    (d,), res = serve(sched, [donor])
    assert sched.cached_tokens[d] == 0 and sched.cached_pages == 4
    long_hit = after(sys_ids, long_audio_request(cfg, 45, 2))
    S = long_hit["input_ids"].shape[1]
    assert S - 3 * PAGE > 256
    reqs = [(after(sys_ids, text_request(cfg, 7 + i, 10 + i)), 6, SETTINGS[i], 20 + i) for i in range(3)]
    rids, res = serve(sched, reqs)
    assert all(sched.cached_tokens[r] == 3 * PAGE and res[r].shape[1] == f["input_ids"].shape[1] + n
               for r, (f, n, _, _) in zip(rids, reqs))
    (lh,), res = serve(sched, [(long_hit, 4, {}, 0)])
    assert sched.cached_tokens[lh] == 3 * PAGE and sched.engine.captures == 2
    first = sched.engine._chunk_logits.float().view(-1)
    feats = {k: v for k, v in long_hit.items() if k != "input_ids"}
    past = gathered(sched, long_hit["input_ids"], 3 * PAGE).grown(S + 4)
    emb = model.prompt_embeds(long_hit["input_ids"], **feats)
    ref = model.forward(long_hit["input_ids"][:, 3 * PAGE:], None, emb[:, 3 * PAGE:].contiguous(), past_key_values=past,
                        logits_to_keep=1).logits.view(-1)
    assert float((first - ref).norm() / ref.norm()) < 3e-2
    assert int(res[lh][0, S]) == int(ref.argmax())
    assert sched.free_pages == 96


# ================================================================================================ 3. sessions
def test_sessions_share_the_system_prompt():
    """Two sessions open with the same system prompt: the second one's first turn hits it, and its turns equal chained
    generate(past_key_values=...) calls that start from the gathered prefix."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    sys_ids = system_prompt(cfg, 2 * PAGE + 20, seed=79)
    sched = SlotScheduler(model, slots=2, max_len=1024, kv_pages=48, prefix_cache=True)
    _poison(sched)
    a, b = sched.open_session(), sched.open_session()
    ra = sched.submit(after(sys_ids, audio_request(cfg, 16000, 1)), max_new_tokens=8, session=a)
    sched.run()
    feats = after(sys_ids, audio_request(cfg, 12000, 2))
    past = None
    for t in range(3):
        rid = sched.submit(feats, max_new_tokens=8, session=b)
        seq = sched.run()[rid]
        if t == 0:
            assert sched.cached_tokens[ra] == 0 and sched.cached_tokens[rid] == 2 * PAGE
            past = gathered(sched, feats["input_ids"], 2 * PAGE)
        else:
            assert sched.cached_tokens[rid] == 0
        o = model.generate(max_new_tokens=8, past_key_values=past, return_dict_in_generate=True, **feats)
        assert torch.equal(seq, o.sequences), t
        past = o.past_key_values
        feats = _turn_features(cfg, seq, 8000 + 4000 * t, 60 + t)
    sched.close_session(a)
    sched.close_session(b)
    assert sched.free_pages == 48 and sched.engine.captures == 1


# ================================================================================================ 4. a short pool
def test_short_pool_evicts_and_serves_everything():
    """A 12-page pool and six system prompts of 2 pages each (more than the pool can keep cached), requests and one session
    cycling over them in rounds of three: cached pages are evicted, later rounds still hit what is left, every request is
    served in full, and every page is available again once the session is closed."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    prompts = [system_prompt(cfg, 2 * PAGE + 3, seed=90 + k) for k in range(6)]
    sched = SlotScheduler(model, slots=4, max_len=512, sync_every=3, kv_pages=12, prefix_cache=True)
    _poison(sched)
    sid = sched.open_session()
    reqs = [(after(prompts[i % 6], text_request(cfg, 5 + i, 30 + i)), 8 + i % 5, SETTINGS[i % 5], 40 + i) for i in range(18)]
    rids = []
    for i, (f, n, s, seed) in enumerate(reqs):
        rids.append(sched.submit(f, max_new_tokens=n, **settings_kw(s, seed), **({"session": sid} if i == 5 else {})))
        if i % 3 == 2:
            res = sched.run()
            for rid, (f2, n2, _, _) in zip(rids[-3:], reqs[i - 2:i + 1]):
                assert res[rid].shape[1] == f2["input_ids"].shape[1] + n2
    assert sched.pool.evicted > 0 and any(sched.cached_tokens[r] for r in rids[6:])
    sched.close_session(sid)
    assert sched.free_pages == 12


# ================================================================================================ 5. no shared prefix
def test_no_shared_prefix_gives_the_bits_of_the_cache_off():
    """The busy chunked-prefill workload plus distinct multi-page prompts: nothing hits, and prefix_cache=True serves every
    request with the bits of prefix_cache=False."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    reqs = _busy_requests(cfg, long_audio_request(cfg, 45, 2))
    reqs += [(text_request(cfg, 70 + 40 * i, 900 + i), 6, SETTINGS[i], 950 + i) for i in range(4)]
    out = []
    for on in (False, True):
        sched = SlotScheduler(model, slots=8, max_len=512, sync_every=3, kv_pages=64, prefix_cache=on)
        _poison(sched)
        rids, res = serve(sched, reqs)
        out.append([res[r] for r in rids])
        assert sched.free_pages == 64
        if on:
            assert set(sched.cached_tokens.values()) == {0} and sched.cached_pages > 0
    for i, (x, y) in enumerate(zip(*out)):
        assert torch.equal(x, y), i
