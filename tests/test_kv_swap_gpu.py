"""Host swap of idle sessions on the GPU: ``uvx_kv_pages_move`` between the device pool and a pinned host pool (byte for byte,
bf16 and e4m3, micro and 8B widths, pages outside the lists untouched, pageable memory refused before any launch), and
conversations served through a pool too small for their histories plus a host tier, turn for turn bit-identical to the same
workload on a pool that never swaps (bf16 and fp8, sampling and the penalty, the prefix cache, a chunked long suffix, the
8B widths), and the capacity a host tier gives.  Device pools, host pools and the admission scratch start as NaN."""
import pytest
import torch

from test_paged_kv_gpu import build, build_8b

pytestmark = pytest.mark.gpu

NAN = float("nan")
NAN_BYTE = 0x7F                 # e4m3fn NaN
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def _poison(sched):
    eng = sched.engine
    pools = [eng.pool_k, eng.pool_v] + ([eng.host_k, eng.host_v] if eng.host_kv_pages else [])
    for t in pools:
        if t.dtype == E4M3:
            t.view(torch.uint8).fill_(NAN_BYTE)
        else:
            t.fill_(NAN)
    eng.cache.k.fill_(NAN)
    eng.cache.v.fill_(NAN)


def _one(sched, feats, **kw):
    """Submits one request, serves the queue and returns its sequence."""
    rid = sched.submit(feats, **kw)
    return sched.run()[rid]


# ================================================================================================ 1. the kernel
@pytest.mark.parametrize("dtype", [torch.bfloat16, E4M3])
@pytest.mark.parametrize("Hkv,D", [(2, 64), (8, 128)])
def test_pages_move_round_trip_is_byte_exact(ops, dtype, Hkv, D):
    from ultravox_b200 import _lib
    L, n_dev, n_host = 4, 160, 72
    g = torch.Generator().manual_seed(Hkv * D)
    shape = (L, n_dev, 64, Hkv, D)
    nbytes = torch.empty(shape, dtype=dtype).view(torch.uint8).numel()
    raw_k = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8)
    raw_v = torch.randint(0, 256, (nbytes,), generator=g, dtype=torch.uint8)
    for raw in (raw_k, raw_v):          # NaN / Inf bit patterns of both types among the random bytes
        raw[:8] = torch.tensor([0x80, 0x7F, 0xC0, 0x7F, 0x80, 0xFF, 0x7F, 0xFF], dtype=torch.uint8)
    kp = raw_k.view(dtype).view(shape).cuda()
    vp = raw_v.view(dtype).view(shape).cuda()
    hk = torch.empty(L, n_host, 64, Hkv, D, dtype=dtype, pin_memory=True)
    hv = torch.empty(hk.shape, dtype=dtype, pin_memory=True)
    for n in (1, 4, 17, 64):
        hk.view(torch.uint8).fill_(NAN_BYTE)
        hv.view(torch.uint8).fill_(NAN_BYTE)
        perm = torch.randperm(n_dev, generator=g)
        src, back = perm[:n], perm[n:2 * n]                 # back into different device pages
        host = torch.randperm(n_host, generator=g)[:n]
        k0, v0 = kp.clone(), vp.clone()
        i32 = lambda t: t.to(torch.int32).cuda()
        ops.kv_pages_move(kp, vp, hk, hv, i32(src), i32(host))
        ops.kv_pages_move(hk, hv, kp, vp, i32(host), i32(back))
        torch.cuda.synchronize()
        b = lambda t: t.view(torch.uint8)
        assert torch.equal(b(hk)[:, host], b(k0)[:, src].cpu()) and torch.equal(b(hv)[:, host], b(v0)[:, src].cpu()), n
        rest = [p for p in range(n_host) if p not in host.tolist()]
        assert bool((b(hk)[:, rest] == NAN_BYTE).all()) and bool((b(hv)[:, rest] == NAN_BYTE).all()), n
        assert torch.equal(b(kp)[:, back], b(k0)[:, src]) and torch.equal(b(vp)[:, back], b(v0)[:, src]), n
        keep = [p for p in range(n_dev) if p not in back.tolist()]
        assert torch.equal(b(kp)[:, keep], b(k0)[:, keep]) and torch.equal(b(vp)[:, keep], b(v0)[:, keep]), n
    # pageable host memory is refused before anything is launched; nothing changes
    pageable = torch.zeros(hk.shape, dtype=torch.uint8 if dtype == E4M3 else dtype).view(dtype)
    assert not pageable.is_pinned()
    one = torch.zeros(1, dtype=torch.int32, device="cuda")
    before, k0 = _lib.launch_count(), kp.clone()
    with pytest.raises(_lib.UvxError, match="pinned host memory"):
        ops.kv_pages_move(kp, vp, pageable, hv, one, one)
    with pytest.raises(_lib.UvxError, match="pinned host memory"):
        ops.kv_pages_move(pageable, pageable, kp, vp, one, one)
    torch.cuda.synchronize()
    assert _lib.launch_count() == before and torch.equal(b(kp), b(k0)) and not bool(pageable.view(torch.uint8).any())
    with pytest.raises(_lib.UvxError, match="one dtype"):
        ops.kv_pages_move(kp, vp, hk.view(torch.uint8), hv.view(torch.uint8), one, one)


# ================================================================================================ 2. conversations
SETTINGS = [{}, dict(do_sample=True, temperature=0.8, top_k=40), dict(repetition_penalty=1.2),
            dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9)]


def _next_turn(cfg, prev, t, i):
    from test_paged_kv_gpu import _turn_features
    return _turn_features(cfg, prev, 12000 + 4000 * t, 50 + t, text_pre=40, text_post=10)


def _first_turn(cfg, i):
    from test_serving_gpu import audio_request
    return audio_request(cfg, 16000, 300 + i, text_pre=40, text_post=20)


def _conversations(model, cfg, n_conv, n_turns, lag, slots=4, **kw):
    """n_conv audio conversations x n_turns through ``slots`` slots.  A conversation 'thinks' after each reply: its next turn is
    submitted from on_tokens once ``lag`` later replies have arrived (so idle sessions exist), the rest after run() returns.
    Returns ({conv: [sequence per turn]}, scheduler)."""
    from ultravox_b200.serving import SlotScheduler
    sched = SlotScheduler(model, slots=slots, max_len=512, sync_every=3, **kw)
    _poison(sched)
    out, state, thinking = {i: [] for i in range(n_conv)}, {}, []
    sids = [sched.open_session() for _ in range(n_conv)]

    def submit(i, t, feats):
        s = dict(SETTINGS[i % len(SETTINGS)])
        if s.get("do_sample"):
            s["generator"] = torch.Generator(device="cuda").manual_seed(1000 * i + t)
        state[sched.submit(feats, max_new_tokens=12, session=sids[i], **s)] = (i, t)

    def on_tokens(rid, seq):
        i, t = state.pop(rid)
        out[i].append(seq)
        if t + 1 < n_turns:
            thinking.append((i, t + 1, _next_turn(cfg, seq, t, i)))
        if len(thinking) > lag:
            submit(*thinking.pop(0))

    for i in range(n_conv):
        submit(i, 0, _first_turn(cfg, i))
    sched.run(on_tokens)
    while thinking:
        submit(*thinking.pop(0))
        sched.run(on_tokens)
    assert not state and all(len(v) == n_turns for v in out.values())
    for s in sids:
        sched.close_session(s)
    return out, sched


def _generate_chain(model, cfg, i, n_turns, **kw):
    outs, past, feats = [], None, _first_turn(cfg, i)
    for t in range(n_turns):
        o = model.generate(max_new_tokens=12, past_key_values=past, return_dict_in_generate=True, **feats,
                           **SETTINGS[i % len(SETTINGS)], **kw)
        outs.append(o.sequences)
        past = o.past_key_values
        feats = _next_turn(cfg, o.sequences, t, i)
    return outs


def _swapped_equals_unswapped(model, cfg, **pool):
    n_conv, n_turns = 6, 3
    big, ref = _conversations(model, cfg, n_conv, n_turns, 2, kv_pages=64, **pool)
    assert ref.swapped_out_pages == ref.swapped_in_pages == 0 and ref.host_free_pages == 0
    small, sched = _conversations(model, cfg, n_conv, n_turns, 2, kv_pages=14, host_kv_pages=24, **pool)
    for i in range(n_conv):
        for t in range(n_turns):
            assert torch.equal(small[i][t], big[i][t]), (i, t)
    print(f"swapped out {sched.swapped_out_pages} pages, in {sched.swapped_in_pages}")
    assert sched.swapped_out_pages > 0 and sched.swapped_in_pages > 0
    assert sched.free_pages == 14 and sched.host_free_pages == 24
    assert sched.engine.captures == 1 == ref.engine.captures


def test_swapped_sessions_equal_unswapped():
    cfg, model = build()
    _swapped_equals_unswapped(model, cfg)
    # one slot decodes one row, as generate() does for one stream (more rows take another GEMM form, other bits): swapped
    # conversations then give chained generate(past_key_values=...)'s turns, greedy and with the penalty
    one, sched = _conversations(model, cfg, 3, 3, 1, slots=1, kv_pages=8, host_kv_pages=16)
    assert sched.swapped_out_pages > 0 and sched.swapped_in_pages > 0
    assert sched.free_pages == 8 and sched.host_free_pages == 16 and sched.engine.captures == 1
    for i in (0, 2):
        want = _generate_chain(model, cfg, i, 3)
        for t in range(3):
            assert torch.equal(one[i][t], want[t]), (i, t)


def test_swapped_sessions_equal_unswapped_fp8():
    from test_kv_fp8_gpu import _scales
    cfg, model = build()
    _swapped_equals_unswapped(model, cfg, kv_cache_dtype="fp8_e4m3", kv_scales=_scales(cfg, 5))


# ================================================================================================ 3. prefix cache, long suffix
def _text(cfg, S, seed):
    from test_serving_gpu import text_request
    return text_request(cfg, S, seed)["input_ids"]


def test_swapped_session_outlives_its_evicted_prefix():
    """A session's first turn hits a cached system prompt; the session is offloaded, the cached pages are then evicted by
    other requests, and its next turn still gives the no-swap run's bits."""
    from ultravox_b200.serving import PAGE, SlotScheduler
    cfg, model = build()
    sys_ids = _text(cfg, 2 * PAGE, 7)

    def run(swap):
        sched = SlotScheduler(model, slots=2, max_len=512, kv_pages=12 if swap else 64, prefix_cache=True,
                              host_kv_pages=8 if swap else 0)
        _poison(sched)
        sched.submit(dict(input_ids=torch.cat([sys_ids, _text(cfg, 20, 8)], 1)), max_new_tokens=4)
        sched.run()
        sid = sched.open_session()
        r1 = sched.submit(dict(input_ids=torch.cat([sys_ids, _text(cfg, 30, 9)], 1)), max_new_tokens=6, session=sid)
        seq1 = sched.run()[r1]
        assert sched.cached_tokens[r1] == 2 * PAGE
        if swap:
            sched.offload_session(sid)
            assert sched.session_on_host(sid) and sched.swapped_out_pages == 3
        others = [sched.submit(dict(input_ids=_text(cfg, 340, 20 + k)), max_new_tokens=4) for k in range(2)]
        sched.run()
        if swap:
            assert sched.pool.evicted >= 2 and sched.pool.match([tuple(sys_ids[0, :PAGE].tolist())]) == []
        r2 = sched.submit(dict(input_ids=torch.cat([seq1, _text(cfg, 25, 10)], 1)), max_new_tokens=6, session=sid)
        seq2 = sched.run()[r2]
        if swap:
            assert not sched.session_on_host(sid) and sched.swapped_in_pages == 3
        sched.close_session(sid)
        assert sched.free_pages == sched.pool.n_pages and len(others) == 2
        return seq1, seq2

    want, got = run(False), run(True)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_swapped_in_session_long_suffix_is_chunked():
    """A swapped-in session whose next suffix exceeds 256 rows is chunk-prefilled from past = kv_len: the no-swap run's bits."""
    from test_chunked_prefill_gpu import long_audio_request
    from test_serving_gpu import audio_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    first = audio_request(cfg, 16000, 4)

    def run(swap):
        sched = SlotScheduler(model, slots=1, max_len=1024, kv_pages=32, host_kv_pages=4 if swap else 0)
        _poison(sched)
        sid = sched.open_session()
        seq1 = _one(sched, first, max_new_tokens=6, session=sid)
        P = sched.session_length(sid)
        if swap:
            sched.offload_session(sid)
            assert sched.session_on_host(sid)
        nxt = long_audio_request(cfg, 45, 3)
        nxt["input_ids"] = torch.cat([seq1, nxt["input_ids"]], dim=1)
        nxt["audio_token_start_idx"] = nxt["audio_token_start_idx"] + seq1.shape[1]
        assert nxt["input_ids"].shape[1] - P > 256
        seq2 = _one(sched, nxt, max_new_tokens=4, session=sid)
        assert sched.engine.captures == 2
        if swap:
            assert sched.swapped_in_pages == sched.swapped_out_pages > 0
        return seq1, seq2

    want, got = run(False), run(True)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


# ================================================================================================ 4. capacity
def test_host_tier_serves_when_sessions_hold_every_page():
    """4 open sessions hold all 8 pages: without a host tier a new request raises the scheduler's RuntimeError; with one,
    idle sessions are swapped out and it completes.  offload_session / session_on_host, and the next turn restores the
    session with the bits of a pool that never swapped."""
    from test_serving_gpu import text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()

    def fill(sched):
        _poison(sched)
        sids = [sched.open_session() for _ in range(4)]
        rids = [sched.submit(text_request(cfg, 100, 900 + i), max_new_tokens=8, session=s) for i, s in enumerate(sids)]
        res = sched.run()
        assert sched.free_pages == sched.pool.n_pages - 8     # 2 pages each
        return sids, [res[r] for r in rids]

    plain = SlotScheduler(model, slots=4, max_len=512, kv_pages=8)
    fill(plain)
    plain.submit(text_request(cfg, 150, 1), max_new_tokens=8)
    with pytest.raises(RuntimeError, match="only 0 of 8 are free: open sessions hold 8; close some"):
        plain.run()

    big = SlotScheduler(model, slots=4, max_len=512, kv_pages=16)
    sids_b, firsts_b = fill(big)
    new_b = _one(big, text_request(cfg, 150, 1), max_new_tokens=8)
    next_b = _one(big, dict(input_ids=torch.cat([firsts_b[0], _text(cfg, 20, 3)], 1)), max_new_tokens=8, session=sids_b[0])

    sched = SlotScheduler(model, slots=4, max_len=512, kv_pages=8, host_kv_pages=8)
    sids, firsts = fill(sched)
    for x, y in zip(firsts, firsts_b):
        assert torch.equal(x, y)
    new = _one(sched, text_request(cfg, 150, 1), max_new_tokens=8)      # 3 pages: swaps 2 sessions out
    assert torch.equal(new, new_b)
    assert sched.swapped_out_pages == 4 and [sched.session_on_host(s) for s in sids] == [True, True, False, False]
    sched.offload_session(sids[2])
    assert sched.session_on_host(sids[2]) and sched.host_free_pages == 2 and sched.free_pages == 6
    nxt = _one(sched, dict(input_ids=torch.cat([firsts[0], _text(cfg, 20, 3)], 1)), max_new_tokens=8, session=sids[0])
    assert torch.equal(nxt, next_b) and not sched.session_on_host(sids[0]) and sched.swapped_in_pages == 2
    for s in sids:
        sched.close_session(s)
    assert sched.free_pages == 8 and sched.host_free_pages == 8


# ================================================================================================ 5. 8B widths
def test_swapped_sessions_8b_widths():
    from test_serving_gpu import text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build_8b()

    def run(swap):
        sched = SlotScheduler(model, slots=2, max_len=256, kv_pages=12, host_kv_pages=12 if swap else 0)
        _poison(sched)
        sids = [sched.open_session() for _ in range(3)]
        out = []
        for t in range(2):
            rids = []
            for i, s in enumerate(sids):
                ids = text_request(cfg, 70, 40 + i)["input_ids"] if t == 0 else torch.cat([out[i - 3], _text(cfg, 15, 60 + i)], 1)
                kw = dict(do_sample=True, temperature=0.9, top_k=30,
                          generator=torch.Generator(device="cuda").manual_seed(10 * i + t)) if i == 1 else {}
                rids.append(sched.submit(dict(input_ids=ids), max_new_tokens=6, session=s, **kw))
            res = sched.run()
            out += [res[r] for r in rids]
            if swap and t == 0:
                for s in sids:
                    sched.offload_session(s)
        if swap:
            assert sched.swapped_out_pages == sched.swapped_in_pages > 0
        return out

    want, got = run(False), run(True)
    for k, (x, y) in enumerate(zip(got, want)):
        assert torch.equal(x, y), k
