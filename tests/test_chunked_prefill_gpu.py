"""Chunked prefill inside the continuous-batching step: the device-indexed wgmma attention and the mapped RoPE + KV append
against the host-indexed kernels they restate (bit for bit, with poisoned cache rows around them), a long audio request
served alone against the fp32 oracle, a whole-prompt prefill and generate(), its bits inside a busy engine, and the
selection boundary at 256 prompt rows."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def build(name="micro", **kw):
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    cfg = preset(name, **kw)
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def text_request(cfg, S, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(input_ids=torch.randint(0, min(cfg.vocab_size, 1000), (1, S), generator=g).cuda())


def long_audio_request(cfg, seconds, seed, text_pre=8, text_post=5):
    """Processor-shaped features of one clip longer than the 30 s encoder context: the log-mel of the whole clip cut into
    3000-frame chunks (continuations zero-padded), one placeholder run per chunk, as ``UltravoxProcessor`` builds them."""
    from oracle import logmel as ol
    from ultravox_b200 import ops
    from ultravox_b200.processing import frame_chunks
    wav = np.random.default_rng(2000 + seed).standard_normal(int(seconds * 16000)).astype(np.float32)
    padded, frames = ol.pad_batch([wav])
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    plan, _ = frame_chunks([int(frames[0])], 3000)
    pieces = []
    for _, off, _, cont in plan:
        piece = mel[0, :, off:off + 3000]
        if cont and piece.shape[-1] < 3000:
            piece = torch.nn.functional.pad(piece, (0, 3000 - piece.shape[-1]))
        pieces.append(piece)
    lens = [p[2] for p in plan]
    toks = [-(-n // 16) for n in lens]
    starts = list(np.cumsum([text_pre] + toks[:-1]))
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, min(cfg.vocab_size, 1000), (1, text_pre + sum(toks) + text_post), generator=g)
    return dict(input_ids=ids.cuda(), audio_values=torch.stack(pieces), audio_token_start_idx=torch.tensor(starts).cuda(),
                audio_lens=torch.tensor(lens).cuda(), audio_token_len=torch.tensor(toks, dtype=torch.int32).cuda(),
                audio_batch_size=torch.tensor([len(plan)]).cuda())


def serve(sched, reqs):
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


def oracle_bar(sd, sh, emb0, seq, S, n_new, tol_exact=2):
    """Teacher-forced fp32 oracle over the served tokens, the bar of test_served_greedy_request_matches_stepwise_oracle."""
    from oracle import model as om
    table = sd["language_model.model.embed_tokens.weight"]
    cur, exact = emb0, 0
    for t in range(n_new):
        ref = om.llama_forward(sd, sh, cur, last_only=True).view(-1)
        tok = int(seq[0, S + t])
        assert tok in ref.topk(5).indices.tolist(), t
        assert float(ref.max() - ref[tok]) < 3e-2 * float(ref.abs().max()), t
        exact += int(tok == int(ref.argmax()))
        cur = torch.cat([cur, table[tok][None, None]], dim=1)
    assert exact >= n_new - tol_exact, exact


# ================================================================================================ 1. kernels
@pytest.mark.parametrize("Hq,Hkv,D", [(32, 8, 128), (32, 8, 64)])
def test_attention_indexed_matches_host_past(ops, Hq, Hkv, D):
    """Device-indexed chunk attention on cache row 5 of 8 == uvx_attention on that row with a host past, bit for bit, for
    past in {0, 1, 63, 64, 65, 300} and valid in {1, 64, C}; the other rows and the keys beyond the prompt hold NaN / 1e30."""
    slots, C, smax = 8, 248, 640
    j = 5
    g = torch.Generator().manual_seed(D)
    kc = (torch.randn(slots, smax, Hkv, D, generator=g) * 2).to(torch.bfloat16).cuda()
    vc = torch.randn(slots, smax, Hkv, D, generator=g).to(torch.bfloat16).cuda()
    rs = (Hq + 2 * Hkv) * D
    qkv = (torch.randn(C, rs, generator=g) * 2).to(torch.bfloat16).cuda()
    q = qkv[:, :Hq * D]
    scale = D ** -0.5
    i32 = dict(dtype=torch.int32, device="cuda")
    for past in (0, 1, 63, 64, 65, 300):
        for valid in (1, 64, C):
            end = past + valid
            kv_len = torch.tensor([end], **i32)
            want = torch.zeros(C, Hq * D, dtype=torch.bfloat16, device="cuda")
            ops.attention(q.data_ptr(), kc[j].data_ptr(), vc[j].data_ptr(), want, 1, Hq, Hkv, C, past + C, D,
                          (rs, C * rs, Hkv * D, smax * Hkv * D, Hkv * D, smax * Hkv * D, Hq * D, C * Hq * D), scale, True, kv_len)
            k2, v2 = kc.clone(), vc.clone()
            for r in range(slots):
                if r != j:
                    k2[r].fill_(float("nan"))
                    v2[r].fill_(float("nan"))
            k2[j, end:] = 1e30
            k2[j, end::2] = -1e30
            v2[j, end:] = float("nan")
            got = torch.zeros(1, C, Hq * D, dtype=torch.bfloat16, device="cuda")
            ops.attention_indexed(q.unsqueeze(0), k2, v2, got, Hq, scale, torch.tensor([j], **i32), torch.tensor([past], **i32),
                                  kv_len)
            assert torch.isfinite(got[0, :valid].float()).all(), (past, valid)
            assert torch.equal(got[0, :valid], want[:valid]), (past, valid)
    with pytest.raises(Exception):           # a key bound is required
        ops.attention_indexed(q.unsqueeze(0), kc, vc, got, Hq, scale, torch.tensor([j], **i32), torch.tensor([0], **i32), None)


@pytest.mark.parametrize("Hq,Hkv,D", [(32, 8, 128), (4, 2, 64)])
def test_rope_kv_append_map_matches_rope_and_write(ops, Hq, Hkv, D):
    """Mapped RoPE + append == uvx_rope at the same positions + the k / v copy into the mapped cache rows, bit for bit; rows
    mapped to -1 leave the (sentinel-filled) cache untouched."""
    R, slots, smax = 24, 4, 64
    g = torch.Generator().manual_seed(7 + D)
    inv = 1.0 / (500000.0 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    cos, sin = ops.rope_tables(inv, 128, "cuda")
    qkv = torch.randn(R, (Hq + 2 * Hkv) * D, generator=g).to(torch.bfloat16).cuda()
    crow = torch.randint(0, slots, (R,), generator=g)
    crow[::3] = -1
    pos = torch.randperm(smax, generator=g)[:R]                       # distinct (row, position) targets
    rope = torch.randint(0, 128, (R,), generator=g)
    sentinel = 7.0
    kc = torch.full((slots, smax, Hkv, D), sentinel, dtype=torch.bfloat16, device="cuda")
    vc = kc.clone()
    got = qkv.clone()
    i32 = lambda t: t.to(torch.int32).cuda()
    ops.rope_kv_append_map_(got, Hq, Hkv, D, cos, sin, i32(rope), kc, vc, i32(crow), i32(pos))
    want = qkv.clone()
    ops.rope_(want, Hq, Hkv, D, cos, sin, rows_per_seq=R, positions=i32(rope))
    assert torch.equal(got, want)
    kw = torch.full_like(kc, sentinel)
    vw = kw.clone()
    for r in range(R):
        if crow[r] >= 0:
            kw[crow[r], pos[r]] = want[r, Hq * D:(Hq + Hkv) * D].view(Hkv, D)
            vw[crow[r], pos[r]] = want[r, (Hq + Hkv) * D:].view(Hkv, D)
    assert torch.equal(kc, kw) and torch.equal(vc, vw)


# ================================================================================================ 2. one long request
def _ulps(a: torch.Tensor, b: torch.Tensor) -> float:
    """max |a - b| in bf16 units in the last place of b (magnitudes below 2^-20 count as 2^-20)."""
    a, b = a.float(), b.float()
    e = torch.floor(torch.log2(b.abs().clamp_min(2.0 ** -20)))
    return float(((a - b).abs() / torch.exp2(e - 7)).max())


def test_long_request_alone():
    """A 70 s clip (3 encoder chunks) plus text, S = 452 rows = 2 chunks of 248 in an 8-slot engine: its tokens pass the
    stepwise fp32 oracle, its cache rows match a whole-prompt prefill within 4 bf16 ulps (measured on an H100: 0) and its
    first-token logits are within 3e-2 of generate()'s prefill."""
    from oracle import model as om
    from ultravox_b200.model import KVCache
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    a = long_audio_request(cfg, 70, 1)
    S = a["input_ids"].shape[1]
    assert 400 <= S <= 700 and a["audio_values"].shape[0] == 3
    sched = SlotScheduler(model, slots=8, max_len=1024)
    poison(sched)
    rid, = serve(sched, [(a, 6, {}, 0)])
    eng = sched.engine
    n_new = 6
    seq = sched.run()[rid]
    assert eng.captures == 2 and eng.prefilling is None
    assert seq.shape == (1, S + n_new) and torch.equal(seq[:, :S], a["input_ids"])
    # the first token's logits (the mixed graph's last replay) against generate()'s prefill
    first = eng._chunk_logits.float().view(-1)
    ref = model.forward(a["input_ids"], logits_to_keep=1, **{k: v for k, v in a.items() if k != "input_ids"}).logits.view(-1)
    assert float((first - ref).norm() / ref.norm()) < 3e-2
    # cache rows [0, S) of the slot against a whole-prompt prefill (every layer)
    feats = {k: v for k, v in a.items() if k != "input_ids"}
    cache = model.new_cache(1, S)
    model.llama_hidden(model.prompt_embeds(a["input_ids"], **feats), KVCache(cache.k, cache.v))
    j = 0
    ku, vu = _ulps(eng.cache.k[:, j, :S], cache.k[:, 0]), _ulps(eng.cache.v[:, j, :S], cache.v[:, 0])
    print(f"chunked vs whole-prompt cache: k {ku:.1f} ulp, v {vu:.1f} ulp")
    assert ku <= 4 and vu <= 4, (ku, vu)
    # the served tokens, teacher-forced through the oracle
    sd, sh = om.state_dict_fp32(model), om.shapes_from_config(cfg)
    st = {}
    om.forward(sd, sh, a["input_ids"].cpu(), a["audio_values"].cpu().to(torch.bfloat16).float(), a["audio_token_start_idx"].cpu(),
               a["audio_lens"].cpu(), a["audio_token_len"].cpu(), a["audio_batch_size"].cpu(), last_only=True, stages=st)
    oracle_bar(sd, sh, st["inputs_embeds"], seq, S, n_new)


def test_long_request_at_8b_widths():
    """The same path at the 8B widths (head_dim 128, GQA 32 / 8; two layers): a 300-row text prompt in 2 chunks of 248 gives
    first-token logits within 3e-2 of a whole-prompt forward, and the same tokens next to short requests as alone."""
    from ultravox_b200.config import PRESETS
    from ultravox_b200.serving import SlotScheduler
    base = PRESETS["v0_5_8b"]
    cfg, model = build("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                       text_config=dict(base["text_config"], num_hidden_layers=2, vocab_size=32000))
    t = text_request(cfg, 300, 9)
    shorts = [(text_request(cfg, 5 + i, 90 + i), 6, {}, 0) for i in range(5)]
    sched = SlotScheduler(model, slots=8, max_len=320)
    poison(sched)
    ids = serve(sched, shorts[:2] + [(t, 8, {}, 0)] + shorts[2:])
    res = sched.run()
    assert sched.engine.captures == 2
    first = sched.engine._chunk_logits.float().view(-1)
    ref = model.forward(t["input_ids"], logits_to_keep=1).logits.view(-1)
    assert float((first - ref).norm() / ref.norm()) < 3e-2
    alone = SlotScheduler(model, slots=8, max_len=320)
    poison(alone)
    rid, = serve(alone, [(t, 8, {}, 0)])
    assert torch.equal(alone.run()[rid], res[ids[2]])


# ================================================================================================ 3. batch variance
def _busy_requests(cfg, long_req):
    """Short text requests around one long one: two in flight when it arrives, more queued behind it."""
    settings = [{}, dict(do_sample=True, temperature=0.7, top_k=50), dict(repetition_penalty=1.3),
                dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9)]
    reqs = [(text_request(cfg, 6 + 3 * i, 500 + i), 20 + i, settings[i % 4], 600 + i) for i in range(3)]
    reqs.append((long_req, 10, {}, 0))
    reqs += [(text_request(cfg, 9 + 2 * i, 700 + i), 12 + 2 * i, settings[(i + 1) % 4], 800 + i) for i in range(8)]
    return reqs


def test_long_request_in_busy_engine_is_deterministic():
    """The long request among 11 short ones in an 8-slot engine == the same request alone in an idle 8-slot engine, bit for
    bit; graph == eager and two identical served runs are bit-identical; a greedy short request that decodes through the
    mixed steps passes the stepwise oracle bar."""
    from oracle import model as om
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    long_req = long_audio_request(cfg, 45, 2)
    assert long_req["input_ids"].shape[1] > 256
    reqs = _busy_requests(cfg, long_req)

    def run(use_graph=True, only=None):
        sched = SlotScheduler(model, slots=8, max_len=512, sync_every=3, use_graph=use_graph)
        poison(sched)
        ids = serve(sched, reqs if only is None else [only])
        res = sched.run()
        return sched, [res[i] for i in ids]

    busy, res = run()
    assert busy.engine.captures == 2
    _, res2 = run()
    eager, res_e = run(use_graph=False)
    assert eager.engine.captures == 0
    for i, (x, y, z) in enumerate(zip(res, res2, res_e)):
        assert torch.equal(x, y) and torch.equal(x, z), i
    alone, (solo,) = run(only=reqs[3])
    assert alone.engine.captures == 2
    assert torch.equal(res[3], solo)
    for i, (feats, n, _, _) in enumerate(reqs):
        assert res[i].shape[1] == feats["input_ids"].shape[1] + n, i
    # request 0 (greedy) decodes next to the chunks: the oracle bar, not bit-identity with itself alone
    sd, sh = om.state_dict_fp32(model), om.shapes_from_config(cfg)
    ids0 = reqs[0][0]["input_ids"].cpu()
    emb = sd["language_model.model.embed_tokens.weight"][ids0]
    oracle_bar(sd, sh, emb, res[0], ids0.shape[1], reqs[0][1], tol_exact=4)


# ================================================================================================ 4. selection boundary
def test_selection_boundary():
    """256 rows: today's one-shot admission (one graph, bit-identical to generate()); 257 rows: chunks (the mixed graph is
    captured once), and such a request retires on EOS and with max_new_tokens = 1."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    t256, t257 = text_request(cfg, 256, 1), text_request(cfg, 257, 2)
    sched = SlotScheduler(model, slots=8, max_len=320)
    rid, = serve(sched, [(t256, 8, {}, 0)])
    assert torch.equal(sched.run()[rid], model.generate(**t256, max_new_tokens=8))
    assert sched.engine.captures == 1
    rid, = serve(sched, [(t257, 8, {}, 0)])
    full = sched.run()[rid]
    assert sched.engine.captures == 2 and full.shape == (1, 265)
    rid1, rid2 = serve(sched, [(t257, 1, {}, 0), (t256, 4, {}, 0)])
    res = sched.run()
    assert torch.equal(res[rid1], full[:, :258]) and res[rid2].shape == (1, 260)
    assert sched.engine.captures == 2
    eos = int(full[0, 257 + 2])
    first = next(i for i in range(257, 265) if int(full[0, i]) == eos)
    s_eos = SlotScheduler(model, slots=8, max_len=320, eos_token_ids=[eos])
    rid, = serve(s_eos, [(t257, 8, {}, 0)])
    got = s_eos.run()[rid]
    assert torch.equal(got, full[:, :first + 1]) and int(got[0, -1]) == eos
    assert s_eos.pending() == [] and s_eos.engine.prefilling is None and not any(s_eos.engine.busy)
