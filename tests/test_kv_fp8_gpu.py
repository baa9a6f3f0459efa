"""FP8 (e4m3) paged KV pool: each fp8 kernel against its bf16 twin run on the dequantized pool (bit for bit, pools NaN-filled
outside the written positions), the append and the page copy against the host quantizer, and the fp8 PagedSlotDecodeEngine /
SlotScheduler: graph == eager, busy == alone, sessions and prefix-cache hits against generate() over the dequantized pages,
shared pages never written, and the capacity half-size pages give."""
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
E4M3 = torch.float8_e4m3fn
NAN_BYTE = 0x7F                 # e4m3fn NaN


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


def quant(x: torch.Tensor, s) -> torch.Tensor:
    """The host quantizer of include/uvx.h: torch's cast is not saturating, so clamp first (NaN passes through the clamp)."""
    s = torch.as_tensor(s, dtype=torch.float32)
    return (x.float().cpu() / s).clamp(-448, 448).to(E4M3)


def dequant(q: torch.Tensor, s) -> torch.Tensor:
    s = torch.as_tensor(s, dtype=torch.float32)
    return (q.cpu().float() * s).to(torch.bfloat16)


def nan_pool(shape) -> torch.Tensor:
    return torch.full(shape, NAN_BYTE, dtype=torch.uint8, device="cuda").view(E4M3)


def bits(t: torch.Tensor) -> torch.Tensor:
    """Raw bits (so NaN compares equal to the same NaN)."""
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]).cpu()


def nan_canon(b: torch.Tensor) -> torch.Tensor:
    """e4m3 bytes with both NaN codes as 0x7F: the kernels store every NaN as 0x7F, the host cast keeps the sign."""
    return torch.where(b & 0x7F == 0x7F, torch.full_like(b, 0x7F), b)


def assert_bytes(got: torch.Tensor, want: torch.Tensor, src: torch.Tensor = None):
    """got / want e4m3 bytes of one shape, equal up to the sign of NaN; on a mismatch, report the first few (index, got,
    want[, source value])."""
    got, want = nan_canon(got), nan_canon(want)
    bad = (got != want).nonzero()
    if len(bad):
        rows = [(tuple(i.tolist()), int(got[tuple(i)]), int(want[tuple(i)]),
                 None if src is None else float(src[tuple(i)])) for i in bad[:8]]
        raise AssertionError(f"{len(bad)} bytes differ: {rows}")


def assert_bf16(got: torch.Tensor, want: torch.Tensor):
    """Bit-equal bf16 except that a NaN only has to meet a NaN (the kernels give the canonical NaN, the host keeps the payload)."""
    got, want = got.cpu(), want.cpu()
    nan = torch.isnan(want.float())
    assert torch.equal(torch.isnan(got.float()), nan)
    assert torch.equal(bits(got)[~nan], bits(want)[~nan])


def kernels_run(fn) -> str:
    """The names of the CUDA kernels ``fn`` (idempotent) launches (torch.profiler), joined."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = "\n".join(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "uvx::" in e.name)
        if names:              # now and then the profiler delivers no activity records for a window: profile the call again
            return names
    return names


def shuffled_table(B, W, n_pages, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(n_pages, generator=g)[:B * W].view(B, W).to(torch.int32)


def to_pool8(k, pages, n_pages, s):
    """Contiguous bf16 rows k [B, S, Hkv, D] -> (e4m3 pool [n_pages, 64, Hkv, D] NaN-filled outside the rows, with row b's tile t
    quantized into page pages[b][t]; the bf16 pool of its dequantized values)."""
    B, S, Hkv, D = k.shape
    pool = torch.full((n_pages, 64, Hkv, D), NAN_BYTE, dtype=torch.uint8).view(E4M3)
    for b in range(B):
        for t in range(-(-S // 64)):
            if pages[b][t] < 0:
                continue
            n = min(64, S - 64 * t)
            pool[pages[b][t], :n] = quant(k[b, 64 * t:64 * t + n], s)
    return pool.cuda(), dequant(pool, s).cuda()


SCALES = [(1.0, 1.0), (2.0 ** -3, 0.37), (0.37, 2.0 ** -3)]


# ================================================================================================ 1. append
@pytest.mark.parametrize("Hq,Hkv,D", [(32, 8, 128), (8, 2, 64)])
@pytest.mark.parametrize("sk,sv", SCALES)
def test_append_fp8_matches_bf16_and_host_quantizer(ops, Hq, Hkv, D, sk, sv):
    R, n_pages = 24, 12
    g = torch.Generator().manual_seed(D + int(sk * 100))
    inv = 1.0 / (500000.0 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    cos, sin = ops.rope_tables(inv, 256, "cuda")
    qkv = (torch.randn(R, (Hq + 2 * Hkv) * D, generator=g) * 40).to(torch.bfloat16)
    special = torch.tensor([500.0, -500.0, float("inf"), float("-inf"), NAN, 2.0 ** -10, -(2.0 ** -9), 1e-3, 448.0, 460.0])
    kv0 = Hq * D
    for r in range(0, R, 3):                 # specials in the k and v sections (k goes through RoPE first)
        qkv[r, kv0 + 3 * r % 50:kv0 + 3 * r % 50 + 10] = special
        qkv[r, kv0 + Hkv * D + 5 * r % 70:kv0 + Hkv * D + 5 * r % 70 + 10] = special
    qkv = qkv.cuda()
    page = torch.randint(0, n_pages, (R,), generator=g).to(torch.int32)
    page[::5] = -1                           # writes nothing
    off = torch.randperm(64, generator=g)[:R].to(torch.int32)      # distinct offsets: no two rows write one position
    rope = torch.randint(0, 256, (R,), generator=g).to(torch.int32).cuda()
    page, off = page.cuda(), off.cuda()
    kb = torch.zeros(n_pages, 64, Hkv, D, dtype=torch.bfloat16, device="cuda")
    vb = kb.clone()
    want = qkv.clone()
    ops.rope_kv_append_map_(want, Hq, Hkv, D, cos, sin, rope, kb, vb, page, off)
    sentinel = 0x55
    k8 = torch.full((n_pages, 64, Hkv, D), sentinel, dtype=torch.uint8, device="cuda").view(E4M3)
    v8 = k8.clone()
    scale = torch.tensor([sk, sv], dtype=torch.float32, device="cuda")
    got = qkv.clone()

    def append():                            # from the same input each time (RoPE rotates qkv in place)
        got.copy_(qkv)
        ops.rope_kv_append_map_(got, Hq, Hkv, D, cos, sin, rope, k8, v8, page, off, kv_scale=scale)

    names = kernels_run(append)
    assert "rope_kv_append_map_fp8_kernel" in names
    assert torch.equal(bits(got), bits(want))            # q and k in qkv: the bf16 form's bits
    wk = torch.full((n_pages, 64, Hkv, D), sentinel, dtype=torch.uint8)
    wv = wk.clone()
    for r in range(R):
        p, o = int(page[r]), int(off[r])
        if p >= 0:
            wk[p, o] = quant(kb[p, o], sk).view(torch.uint8)
            wv[p, o] = quant(vb[p, o], sv).view(torch.uint8)
    assert_bytes(bits(k8), wk, kb.float().cpu())
    assert_bytes(bits(v8), wv, vb.float().cpu())


# ================================================================================================ 2. page copy
def test_pages_copy_fp8_against_host(ops):
    L, smax, Hkv, D = 3, 320, 8, 128
    n_pages = 16
    g = torch.Generator().manual_seed(1)
    k = (torch.randn(L, 1, smax, Hkv, D, generator=g) * 30).to(torch.bfloat16)
    v = (torch.randn(L, 1, smax, Hkv, D, generator=g) * 30).to(torch.bfloat16)
    k[0, 0, 100, 0, :4] = torch.tensor([float("inf"), NAN, 1000.0, 2.0 ** -12])
    scales = torch.tensor([[1.0, 0.5], [2.0 ** -3, 0.37], [0.37, 2.0]], dtype=torch.float32)
    pages = torch.tensor([9, 2, 14, 0, 5], dtype=torch.int32, device="cuda")
    kp, vp = nan_pool((L, n_pages, 64, Hkv, D)), nan_pool((L, n_pages, 64, Hkv, D))
    p0, p1 = 70, 300                         # both mid-page
    sc = scales.cuda()
    names = kernels_run(lambda: ops.kv_pages_copy(k.cuda(), v.cuda(), kp, vp, pages, p0, p1, to_pages=True, kv_scales=sc))
    assert "kv_pages_copy_kernel<true>" in names
    wk = torch.full((L, n_pages, 64, Hkv, D), NAN_BYTE, dtype=torch.uint8)
    wv = wk.clone()
    pl = pages.tolist()
    for p in range(p0, p1):
        for li in range(L):
            wk[li, pl[p // 64], p % 64] = quant(k[li, 0, p], scales[li, 0]).view(torch.uint8)
            wv[li, pl[p // 64], p % 64] = quant(v[li, 0, p], scales[li, 1]).view(torch.uint8)
    assert_bytes(bits(kp), wk)               # nothing outside [p0, p1) written
    assert_bytes(bits(vp), wv)
    k2 = torch.full((L, 1, smax, Hkv, D), NAN, dtype=torch.bfloat16, device="cuda")
    v2 = k2.clone()
    ops.kv_pages_copy(k2, v2, kp, vp, pages, p0, p1, to_pages=False, kv_scales=sc)
    for li in range(L):
        pos = torch.arange(p0, p1)
        pk = bits(kp)[li, pages.cpu()[pos // 64].long(), pos % 64].view(E4M3)
        pv = bits(vp)[li, pages.cpu()[pos // 64].long(), pos % 64].view(E4M3)
        assert_bf16(k2[li, 0, p0:p1], dequant(pk, scales[li, 0]))
        assert_bf16(v2[li, 0, p0:p1], dequant(pv, scales[li, 1]))
    assert torch.isnan(k2[:, :, :p0].float()).all() and torch.isnan(k2[:, :, p1:].float()).all()
    with pytest.raises(ValueError):
        ops.kv_pages_copy(k2, v2, kp, vp, pages, p0, p1, to_pages=False)          # an fp8 pool needs its scales


# ================================================================================================ 3. decode attention
@pytest.mark.parametrize("Hq,Hkv,D", [(32, 8, 128), (8, 2, 64)])
@pytest.mark.parametrize("B", [1, 8, 32])
def test_attention_paged_fp8_matches_bf16_on_dequantized_pool(ops, Hq, Hkv, D, B):
    base = [1, 63, 64, 65, 4000, 300, 129, 2]
    lens = (base * (B // len(base) + 1))[:B]
    smax = 4032
    W = smax // 64
    g = torch.Generator().manual_seed(D + B)
    k = (torch.randn(B, smax, Hkv, D, generator=g) * 2).to(torch.bfloat16)
    v = torch.randn(B, smax, Hkv, D, generator=g).to(torch.bfloat16)
    rs = (Hq + 2 * Hkv) * D
    qkv = (torch.randn(B, rs, generator=g) * 2).to(torch.bfloat16).cuda()
    kv_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    n_pages = B * W + 7
    table = shuffled_table(B, W, n_pages, 3)
    for b, n in enumerate(lens):
        table[b, -(-n // 64):] = -1
    sk, sv = 0.37, 2.0 ** -3
    # only each row's first kv_len positions are written; the rest of the pool (page tails included) stays NaN
    kr = torch.stack([torch.cat([k[b, :n], torch.full((smax - n, Hkv, D), NAN, dtype=torch.bfloat16)]) for b, n in enumerate(lens)])
    vr = torch.stack([torch.cat([v[b, :n], torch.full((smax - n, Hkv, D), NAN, dtype=torch.bfloat16)]) for b, n in enumerate(lens)])
    tl = table.tolist()
    k8, kd = to_pool8(kr, tl, n_pages, sk)
    v8, vd = to_pool8(vr, tl, n_pages, sv)
    table = table.cuda()
    scale = torch.tensor([sk, sv], dtype=torch.float32, device="cuda")
    want = torch.zeros(B, Hq * D, dtype=torch.bfloat16, device="cuda")
    ops.attention_paged(qkv[:, :Hq * D], kd, vd, want, Hq, D ** -0.5, table, kv_len)
    got = torch.zeros_like(want)
    names = kernels_run(lambda: ops.attention_paged(qkv[:, :Hq * D], k8, v8, got, Hq, D ** -0.5, table, kv_len, kv_scale=scale))
    assert f"attn_fwd_kernel<{D}, true, true>" in names
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, want)
    for b in {0, B // 2, B - 1}:             # batch isolation: a row alone gives the same bits
        one = torch.zeros(1, Hq * D, dtype=torch.bfloat16, device="cuda")
        ops.attention_paged(qkv[b:b + 1, :Hq * D], k8, v8, one, Hq, D ** -0.5, table[b:b + 1], kv_len[b:b + 1], kv_scale=scale)
        assert torch.equal(one[0], got[b]), b


# ================================================================================================ 4. chunk attention
@pytest.mark.parametrize("Hq,Hkv,D", [(32, 8, 128), (8, 2, 64)])
@pytest.mark.parametrize("C", [64, 70, 248])
def test_attention_indexed_paged_fp8_matches_bf16_on_dequantized_pool(ops, Hq, Hkv, D, C):
    slots, smax = 3, 4096 + 256
    W = smax // 64
    j = 1
    g = torch.Generator().manual_seed(C + D)
    kc = (torch.randn(slots, smax, Hkv, D, generator=g) * 2).to(torch.bfloat16)
    vc = torch.randn(slots, smax, Hkv, D, generator=g).to(torch.bfloat16)
    rs = (Hq + 2 * Hkv) * D
    qkv = (torch.randn(C, rs, generator=g) * 2).to(torch.bfloat16).cuda()
    q = qkv[:, :Hq * D].unsqueeze(0)
    i32 = dict(dtype=torch.int32, device="cuda")
    n_pages = slots * W + 5
    table = shuffled_table(slots, W, n_pages, C)
    sk, sv = 2.0 ** -3, 0.37
    scale = torch.tensor([sk, sv], dtype=torch.float32, device="cuda")
    for past in (0, 63, 300, 4000):
        end = past + C
        kr, vr = kc.clone(), vc.clone()
        kr[:, end:] = NAN                    # unwritten positions: NaN bytes in the pool
        vr[:, end:] = NAN
        kr[[r for r in range(slots) if r != j]] = NAN
        vr[[r for r in range(slots) if r != j]] = NAN
        k8, kd = to_pool8(kr, table.tolist(), n_pages, sk)
        v8, vd = to_pool8(vr, table.tolist(), n_pages, sv)
        t2 = table.clone().cuda()
        t2[j, -(-end // 64):] = -1
        args = (torch.tensor([j], **i32), torch.tensor([past], **i32), torch.tensor([end], **i32))
        want = torch.zeros(1, C, Hq * D, dtype=torch.bfloat16, device="cuda")
        ops.attention_indexed_paged(q, kd, vd, want, Hq, D ** -0.5, t2, *args)
        got = torch.zeros_like(want)
        names = kernels_run(lambda: ops.attention_indexed_paged(q, k8, v8, got, Hq, D ** -0.5, t2, *args, kv_scale=scale))
        assert f"attn_wg_kernel<{D}, true, true, true>" in names
        assert torch.isfinite(got.float()).all(), past
        assert torch.equal(got, want), past


# ================================================================================================ 5. engine: graph == eager, busy == alone
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
    eng.pool_k.view(torch.uint8).fill_(NAN_BYTE)
    eng.pool_v.view(torch.uint8).fill_(NAN_BYTE)
    eng.cache.k.fill_(NAN)
    eng.cache.v.fill_(NAN)


# what an fp8 engine launches: the append and both attention forms inside its steps (the wgmma form in a mixed step), the page
# copy at a B = 1 admission
ENGINE_KERNELS = ("rope_kv_append_map_fp8_kernel", "attn_fwd_kernel<{D}, true, true>", "attn_wg_kernel<{D}, true, true, true>",
                  "kv_pages_copy_kernel<true>")


def _scales(cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    return 0.25 + torch.rand(cfg.text_config.num_hidden_layers, 2, generator=g)


def test_fp8_engine_graph_eager_and_busy_equals_alone():
    """The chunked-prefill busy workload (greedy, top-k, top-p, penalty, one chunked audio prompt, 8 slots) on an fp8 pool:
    graph == eager, and each request gets the same bits served alone through an 8-slot fp8 engine."""
    from test_chunked_prefill_gpu import _busy_requests, long_audio_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    reqs = _busy_requests(cfg, long_audio_request(cfg, 45, 2))
    kw = dict(slots=8, max_len=512, sync_every=3, kv_pages=64, kv_cache_dtype="fp8_e4m3", kv_scales=_scales(cfg))
    graph = SlotScheduler(model, **kw)
    assert graph.engine.pool_k.dtype == E4M3
    _poison(graph)
    got = _serve(graph, reqs)
    assert graph.engine.captures == 2 and graph.free_pages == 64
    eager = SlotScheduler(model, use_graph=False, **kw)
    _poison(eager)
    out = []
    names = kernels_run(lambda: out.append(_serve(eager, reqs)))     # serving again gives the same bits: see below
    for k in ENGINE_KERNELS:
        assert k.format(D=64) in names, k
    for res in out:
        for i, (x, y) in enumerate(zip(res, got)):
            assert torch.equal(x, y), i
    alone = SlotScheduler(model, **kw)
    _poison(alone)
    for i, r in enumerate(reqs):
        assert torch.equal(_serve(alone, [r])[0], got[i]), i


def test_fp8_engine_busy_equals_alone_8b_widths():
    from test_serving_gpu import _mixed_requests
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build_8b()
    reqs = _mixed_requests(cfg, 10, 1, audio=False)
    kw = dict(slots=8, max_len=64, sync_every=3, kv_pages=12, kv_cache_dtype="fp8_e4m3", kv_scales=_scales(cfg, 1))
    busy = SlotScheduler(model, use_graph=False, **kw)      # eager here, graphs alone: busy == alone and graph == eager
    _poison(busy)
    out = []
    names = kernels_run(lambda: out.append(_serve(busy, reqs)))
    for k in ("rope_kv_append_map_fp8_kernel", "attn_fwd_kernel<128, true, true>", "kv_pages_copy_kernel<true>"):
        assert k in names, k
    got = out[-1]
    alone = SlotScheduler(model, **kw)
    _poison(alone)
    for i, r in enumerate(reqs):
        assert torch.equal(_serve(alone, [r])[0], got[i]), i


# ================================================================================================ 6. sessions and prefix cache
def _deq_cache(eng, pages, P, cap):
    """KVCache [L, 1, cap, Hkv, D] holding the dequantized first P positions of ``pages``."""
    from ultravox_b200.model import KVCache
    sc = eng.kv_scales.cpu()
    out = []
    for pool, w in ((eng.pool_k, 0), (eng.pool_v, 1)):
        q = torch.cat([bits(pool[:, p]) for p in pages], dim=1)[:, :P].view(E4M3)
        d = torch.stack([dequant(q[li], sc[li, w]) for li in range(q.shape[0])])
        full = torch.zeros(q.shape[0], 1, cap, *q.shape[2:], dtype=torch.bfloat16)
        full[:, 0, :P] = d
        out.append(full.cuda())
    return KVCache(out[0], out[1], P)


def _page_bytes(eng, pages, P):
    k = torch.cat([bits(eng.pool_k[:, p]) for p in pages], dim=1)[:, :P]
    v = torch.cat([bits(eng.pool_v[:, p]) for p in pages], dim=1)[:, :P]
    return k, v


def _record_appends(monkeypatch, eng):
    """Wraps ops.rope_kv_append_map_ (eager engines call it once per layer and step): every call into ``eng``'s fp8 pool logs
    (layer found from the pool address, the rotated bf16 k rows and the v rows it appended, page, offset)."""
    from ultravox_b200 import ops as o
    real, log = o.rope_kv_append_map_, []

    def rec(qkv, Hq, Hkv, D, cos, sin, rope, kc, vc, page, off, kv_scale=None):
        real(qkv, Hq, Hkv, D, cos, sin, rope, kc, vc, page, off, kv_scale=kv_scale)
        if kc.dtype == E4M3:
            li = (kc.data_ptr() - eng.pool_k.data_ptr()) // eng.pool_k[0].nbytes
            w = Hkv * D
            log.append((li, qkv[:, Hq * D:Hq * D + w].cpu(), qkv[:, Hq * D + w:Hq * D + 2 * w].cpu(), page.tolist(), off.tolist()))

    monkeypatch.setattr(o, "rope_kv_append_map_", rec)
    return log


@pytest.mark.parametrize("widths", ["micro", "8b"])
def test_fp8_session_turns_against_generate_on_dequantized_pages(widths, monkeypatch):
    """Turn t > 0 of a session: its first token equals generate(past_key_values=<the session's pages, dequantized>).  After each
    turn its pages [past, S) hold the host quantizer applied to the bf16 scratch K / V of its admission, and the positions its
    decode steps appended hold the host quantizer applied to the rows each step appended, with that layer's own K and V scales
    (distinct per layer), so a wrong layer's or a swapped scale shows."""
    from test_paged_kv_gpu import _turn_features
    from test_serving_gpu import audio_request, text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build() if widths == "micro" else build_8b()
    sched = SlotScheduler(model, slots=2, max_len=512, kv_pages=24, kv_cache_dtype="fp8_e4m3", kv_scales=_scales(cfg, 2),
                          use_graph=False)
    _poison(sched)
    eng = sched.engine
    sc = eng.kv_scales.cpu()
    log = _record_appends(monkeypatch, eng)
    Hkv, D = cfg.text_config.num_key_value_heads, model.language_model.head_dim
    sid = sched.open_session()
    feats = audio_request(cfg, 16000, 1) if widths == "micro" else text_request(cfg, 40, 1)
    for t, settings in enumerate(({}, dict(repetition_penalty=1.3), dict(do_sample=True, temperature=0.8, top_k=40))):
        P = sched.session_length(sid)
        S = feats["input_ids"].shape[1]
        kw = dict(settings)
        if kw.get("do_sample"):
            kw["generator"] = torch.Generator(device="cuda").manual_seed(7 + t)
        want = None
        if P:
            pages = sched.pool.session(sid).pages
            cache = _deq_cache(eng, pages, P, S + 4)
            gkw = dict(settings)
            if gkw.get("do_sample"):
                gkw["generator"] = torch.Generator(device="cuda").manual_seed(7 + t)
            want = model.generate(max_new_tokens=4, past_key_values=cache, return_dict_in_generate=True, **feats, **gkw).sequences
        log.clear()
        rid = sched.submit(feats, max_new_tokens=4, session=sid, **kw)
        seq = sched.run()[rid]
        if want is not None:
            assert int(seq[0, S]) == int(want[0, S]), t
        pages = sched.pool.session(sid).pages
        K = sched.session_length(sid)               # decode steps fed positions [S, K)
        assert K > S
        kb, vb = _page_bytes(eng, pages, K)
        written = {}                                # (layer, page, offset) -> the last k / v row appended there
        for li, k, v, page, off in log:
            for r, (pg, o) in enumerate(zip(page, off)):
                if pg >= 0:
                    written[(li, pg, o)] = (k[r], v[r])
        for li in range(cfg.text_config.num_hidden_layers):
            assert torch.equal(kb[li, P:S], bits(quant(eng.cache.k[li, 0, P:S], sc[li, 0]))), (t, li)
            assert torch.equal(vb[li, P:S], bits(quant(eng.cache.v[li, 0, P:S], sc[li, 1]))), (t, li)
            for p in range(S, K):
                k, v = written[(li, pages[p // 64], p % 64)]
                assert_bytes(kb[li, p], bits(quant(k.view(Hkv, D), sc[li, 0])))
                assert_bytes(vb[li, p], bits(quant(v.view(Hkv, D), sc[li, 1])))
        if widths == "micro":
            feats = _turn_features(cfg, seq, 8000 + 1000 * t, 60 + t)
        else:
            feats = dict(input_ids=torch.cat([seq, text_request(cfg, 12, 90 + t)["input_ids"]], dim=1))
    sched.close_session(sid)
    assert sched.free_pages == 24


def test_fp8_prefix_cache_hits_against_generate_and_shared_pages_untouched():
    from test_serving_gpu import text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    system = text_request(cfg, 200, 5)["input_ids"]
    reqs = [dict(input_ids=torch.cat([system, text_request(cfg, 10 + i, 30 + i)["input_ids"]], dim=1)) for i in range(4)]
    sched = SlotScheduler(model, slots=4, max_len=512, kv_pages=32, prefix_cache=True, kv_cache_dtype="fp8_e4m3",
                          kv_scales=_scales(cfg, 3))
    _poison(sched)
    eng = sched.engine
    first = sched.submit(reqs[0], max_new_tokens=6)
    sched.run()
    shared = sched.pool.match([tuple(system[0, i:i + 64].tolist()) for i in range(0, 192, 64)])
    assert len(shared) == 3
    before = _page_bytes(eng, shared, 192)
    want = [model.generate(max_new_tokens=1, past_key_values=_deq_cache(eng, shared, 192, 300), **r) for r in reqs[1:]]
    ids = [sched.submit(r, max_new_tokens=6, do_sample=bool(i % 2), temperature=0.9 if i % 2 else None) for i, r in enumerate(reqs[1:])]
    res = sched.run()
    for i, rid in enumerate(ids):
        assert sched.cached_tokens[rid] == 192
        S = reqs[1 + i]["input_ids"].shape[1]
        if i % 2 == 0:                       # greedy hits: the first token is generate()'s over the dequantized shared pages
            assert int(res[rid][0, S]) == int(want[i][0, S]), i
    after = _page_bytes(eng, shared, 192)
    assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1])
    assert sched.cached_tokens[first] == 0


# ================================================================================================ 7. oracle bar
def _fake_quant(x: torch.Tensor, s: float) -> torch.Tensor:
    """fp32 x rounded through e4m3 with scale s, as a write into the pool and the read back do (the oracle keeps fp32)."""
    return (x / s).clamp(-448, 448).to(E4M3).float() * s


class _FakeQuantKV:
    """Passed to the oracle's llama_layer as its ``kv_out``: rounds the layer's post-RoPE K and V through e4m3 in place, before
    the layer's attention uses them."""

    def __init__(self, s):
        self.s = s

    def append(self, kv):
        k, v = kv
        k.copy_(_fake_quant(k, float(self.s[0])))
        v.copy_(_fake_quant(v, float(self.s[1])))


def _oracle_logits(sd, sh, emb, scales):
    """The fp32 oracle's last-row logits of ``emb`` [1, S, H], its K / V fake-quantized per layer with ``scales`` [L, 2] (None:
    exact) - om.llama_forward with the hook llama_layer offers."""
    import torch.nn.functional as F
    from oracle import model as om
    S = emb.shape[1]
    cos, sin = om.rope_cos_sin(sh, torch.arange(S)[None])
    mask = torch.triu(torch.full((S, S), om._finfo_min(emb.dtype), dtype=emb.dtype), diagonal=1)[None, None]
    p = "language_model.model."
    h = emb
    for i in range(sh.layers):
        h = om.llama_layer(sd, f"{p}layers.{i}.", sh, h, cos, sin, mask, kv_out=None if scales is None else _FakeQuantKV(scales[i]))
    h = om.rms_norm(h[:, -1:], sd[p + "norm.weight"], sh.rms_eps)
    head = sd[p + "embed_tokens.weight"] if sh.tie_embeddings else sd["language_model.lm_head.weight"]
    return F.linear(h, head).view(-1)


def test_fp8_served_request_matches_fake_quantized_oracle():
    """A greedy audio request in a 4-slot fp8 engine (distinct K / V scales per layer) next to three sampled text requests,
    teacher-forced through the stepwise fp32 oracle whose post-RoPE K / V are rounded through e4m3 with the same scales, with
    the bar of the serving and chunked-prefill oracle tests.  The first token comes from the bf16 admission prefill, so its
    step is checked against the exact oracle; every later token is picked by a decode step over the fp8 pool."""
    from oracle import model as om
    from test_serving_gpu import audio_request, text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    sd, sh = om.state_dict_fp32(model), om.shapes_from_config(cfg)
    scales = 0.05 + 2 * torch.rand(cfg.text_config.num_hidden_layers, 2, generator=torch.Generator().manual_seed(9))
    a = audio_request(cfg, 16000, 1)
    others = [(text_request(cfg, 7 + 5 * i, 40 + i), 10, dict(do_sample=True, temperature=0.8), 50 + i) for i in range(3)]
    sched = SlotScheduler(model, slots=4, max_len=128, kv_pages=16, kv_cache_dtype="fp8_e4m3", kv_scales=scales)
    _poison(sched)
    n_new = 8
    seq = _serve(sched, others[:2] + [(a, n_new, {}, 0)] + others[2:])[2]
    S = a["input_ids"].shape[1]
    assert seq.shape == (1, S + n_new)
    st = {}
    om.forward(sd, sh, a["input_ids"].cpu(), a["audio_values"].cpu().to(torch.bfloat16).float(), a["audio_token_start_idx"].cpu(),
               a["audio_lens"].cpu(), a["audio_token_len"].cpu(), a["audio_batch_size"].cpu(), last_only=True, stages=st)
    cur = st["inputs_embeds"]
    table = sd["language_model.model.embed_tokens.weight"]
    exact = 0
    for t in range(n_new):
        ref = _oracle_logits(sd, sh, cur, None if t == 0 else scales)
        tok = int(seq[0, S + t])
        assert tok in ref.topk(5).indices.tolist(), t
        assert float(ref.max() - ref[tok]) < 3e-2 * float(ref.abs().max()), t
        exact += int(tok == int(ref.argmax()))
        cur = torch.cat([cur, table[tok][None, None]], dim=1)
    assert exact >= n_new - 2, exact


# ================================================================================================ 8. capacity and bytes
def test_fp8_pool_half_the_bytes_and_twice_the_admissions():
    from test_serving_gpu import text_request
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    bf = SlotScheduler(model, slots=4, max_len=512, kv_pages=8)
    f8 = SlotScheduler(model, slots=4, max_len=512, kv_pages=8, kv_cache_dtype="fp8_e4m3")
    assert f8.engine.pool_k.nbytes * 2 == bf.engine.pool_k.nbytes and f8.engine.pool_v.nbytes * 2 == bf.engine.pool_v.nbytes
    assert torch.equal(f8.engine.kv_scales.cpu(), torch.ones(cfg.text_config.num_hidden_layers, 2))
    # equal pool bytes: 8 bf16 pages or 16 fp8 pages; four requests of 4 pages each
    f8 = SlotScheduler(model, slots=4, max_len=512, kv_pages=16, kv_cache_dtype="fp8_e4m3")
    page = lambda e: e.pool_k[:, 0].nbytes + e.pool_v[:, 0].nbytes      # noqa: E731
    assert 16 * page(f8.engine) == 8 * page(bf.engine)
    admitted = []
    for sched in (bf, f8):
        for i in range(4):
            sched.submit(text_request(cfg, 200, 40 + i), max_new_tokens=40)
        sched._admit()
        admitted.append(len(sched._running))
        res = sched.run()
        assert len(res) == 4
    assert admitted == [2, 4], admitted
