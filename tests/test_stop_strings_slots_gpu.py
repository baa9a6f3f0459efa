"""Stop strings in the continuous-batching slot step: SlotScheduler(max_stop_table=N) and submit(stop_strings=, tokenizer=)
against generate() alone - one slot, a busy 8-slot engine mixing requests with and without stop strings, a chunked prompt, the
lookup step, a paged session turn, prefix-cache hits and host swap on the bf16 and e4m3 pools, 8B widths - launch counts
without stop tables, and the argument checks."""
import pytest
import torch

from test_stop_strings_cpu import make_tokenizer
from test_stop_strings_gpu import _model

pytestmark = pytest.mark.gpu

EOS = [7]


@pytest.fixture(scope="module")
def micro():
    cfg, model = _model()
    return cfg, model, make_tokenizer(cfg.vocab_size, "bytelevel", seed=1)


def _requests(model, tok, n_req=10, seed=0):
    """Prompts, and for every other one stop strings cut from its own reply (so they hit at varied steps)."""
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n_req):
        S = 6 + 3 * (i % 4)
        ids = torch.randint(8, 1000, (1, S), generator=g).cuda()
        n = 10 + (i % 3) * 4
        kw = {}
        if i % 2 == 0:
            full = model.generate(ids, max_new_tokens=n, eos_token_id=EOS)
            txt = tok.decode(full[0, S:].tolist())
            a = 2 + i % 7
            if txt[a:a + 4]:
                kw = dict(stop_strings=[txt[a:a + 4]], tokenizer=tok)
        reqs.append((ids, n, kw))
    return reqs


def _alone(model, ids, n, kw):
    return model.generate(ids, max_new_tokens=n, eos_token_id=EOS, **kw)


def test_one_slot_and_busy_equal_generate(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model, tok = micro
    reqs = _requests(model, tok)
    want = [_alone(model, ids, n, kw) for ids, n, kw in reqs]
    assert sum(w.shape[1] < ids.shape[1] + n for w, (ids, n, kw) in zip(want, reqs) if kw) >= 2     # some stop early
    one = SlotScheduler(model, slots=1, max_len=400, eos_token_ids=EOS, max_stop_table=40000, max_logprobs=2)
    for (ids, n, kw), w in zip(reqs[:4], want[:4]):
        rid = one.submit(dict(input_ids=ids), max_new_tokens=n, logprobs=1, **kw)
        out = one.run()[rid]
        assert torch.equal(out, w)
        ref = model.generate(ids, max_new_tokens=n, eos_token_id=EOS, return_dict_in_generate=True, output_logits=True, **kw)
        lp = torch.stack(ref.logits).log_softmax(-1)[:, 0]
        new = w[0, ids.shape[1]:]
        assert torch.allclose(one.logprobs[rid].token_logprobs, lp.gather(1, new[:, None])[:, 0], atol=1e-5)
    # 8 slots: every request alone in the engine, then all at once (graph and eager)
    alone = SlotScheduler(model, slots=8, max_len=400, eos_token_ids=EOS, sync_every=3, max_stop_table=40000)
    want8 = []
    for ids, n, kw in reqs:
        rid = alone.submit(dict(input_ids=ids), max_new_tokens=n, **kw)
        want8.append(alone.run()[rid])
    for use_graph in (True, False):
        busy = SlotScheduler(model, slots=8, max_len=400, eos_token_ids=EOS, sync_every=3, max_stop_table=40000,
                             use_graph=use_graph)
        rids = [busy.submit(dict(input_ids=ids), max_new_tokens=n, **kw) for ids, n, kw in reqs]
        res = busy.run()
        for rid, w in zip(rids, want8):
            assert torch.equal(res[rid], w), rid
    # some requests stop early in the 8-slot engine too
    assert sum(w.shape[1] < ids.shape[1] + n for w, (ids, n, kw) in zip(want8, reqs) if kw) >= 2


def test_chunked_prompt_lookup_and_paged_turn(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model, tok = micro
    g = torch.Generator().manual_seed(5)
    long = torch.randint(8, 1000, (1, 300), generator=g).cuda()          # more than 256 rows: prefilled in chunks
    full = model.generate(long, max_new_tokens=12, eos_token_id=EOS)
    kw = dict(stop_strings=[tok.decode(full[0, 300:].tolist())[4:8]], tokenizer=tok)
    want = _alone(model, long, 12, kw)
    s = SlotScheduler(model, slots=4, max_len=400, eos_token_ids=EOS, max_stop_table=40000)
    short = torch.randint(8, 1000, (1, 9), generator=g).cuda()
    r0, r1 = s.submit(dict(input_ids=short), max_new_tokens=20), s.submit(dict(input_ids=long), max_new_tokens=12, **kw)
    res = s.run()
    assert torch.equal(res[r1], want) and torch.equal(res[r0], _alone(model, short, 20, {}))
    # the lookup step: the tokens of a plain engine of slots * (K + 1) = 8 slots
    base = torch.randint(8, 1000, (1, 6), generator=g)
    ids = torch.cat([base, base, base[:, :3]], 1).cuda()
    plain8 = SlotScheduler(model, slots=8, max_len=128, eos_token_ids=EOS, max_stop_table=40000)
    rid = plain8.submit(dict(input_ids=ids), max_new_tokens=24)
    full = plain8.run()[rid]
    txt = tok.decode(full[0, ids.shape[1]:].tolist())
    for a, b in ((3, 7), (12, 15)):
        kw = dict(stop_strings=[txt[a:b]], tokenizer=tok)
        look = SlotScheduler(model, slots=2, max_len=128, eos_token_ids=EOS, prompt_lookup_num_tokens=3, max_stop_table=40000)
        rid = look.submit(dict(input_ids=ids), max_new_tokens=24, **kw)
        r8 = plain8.submit(dict(input_ids=ids), max_new_tokens=24, **kw)
        ref = plain8.run()[r8]
        assert torch.equal(look.run()[rid], ref), (a, b)
    # a paged session turn: the string may begin in the earlier turn
    paged = SlotScheduler(model, slots=2, max_len=256, eos_token_ids=EOS, kv_pages=16, max_stop_table=40000)
    sid = paged.open_session()
    first = torch.randint(8, 1000, (1, 10), generator=g).cuda()
    rid = paged.submit(dict(input_ids=first), max_new_tokens=6, session=sid)
    t1 = paged.run()[rid]
    follow = torch.cat([t1, torch.randint(8, 1000, (1, 3), generator=g).cuda()], 1)
    cont = model.generate(follow, max_new_tokens=10, eos_token_id=EOS)
    kw = dict(stop_strings=[tok.decode(cont[0, follow.shape[1] - 1:].tolist())[1:6]], tokenizer=tok)
    rid = paged.submit(dict(input_ids=follow), max_new_tokens=10, session=sid, **kw)
    got = paged.run()[rid]
    assert torch.equal(got, _alone(model, follow, 10, kw))


def test_launch_counts_unchanged_and_errors(micro):
    from ultravox_b200.engine import SlotDecodeEngine
    from ultravox_b200.serving import SlotScheduler
    cfg, model, tok = micro
    plain = SlotDecodeEngine(model, 4, 128, eos_token_ids=EOS)
    off = SlotDecodeEngine(model, 4, 128, eos_token_ids=EOS, max_stop_table=None)
    on = SlotDecodeEngine(model, 4, 128, eos_token_ids=EOS, max_stop_table=64)
    assert plain.launches_per_step == off.launches_per_step == on.launches_per_step - 1
    ids = torch.randint(8, 1000, (1, 8)).cuda()
    s = SlotScheduler(model, slots=2, max_len=128, eos_token_ids=EOS)
    with pytest.raises(ValueError, match="max_stop_table"):
        s.submit(dict(input_ids=ids), stop_strings="ab", tokenizer=tok)
    s2 = SlotScheduler(model, slots=2, max_len=128, eos_token_ids=EOS, max_stop_table=8)
    with pytest.raises(ValueError, match="max_stop_table"):
        s2.submit(dict(input_ids=ids), stop_strings="ab", tokenizer=tok)
    with pytest.raises(ValueError):
        s2.submit(dict(input_ids=ids), stop_strings="ab")
    with pytest.raises(ValueError):
        SlotScheduler(model, slots=2, max_len=128, max_stop_table=3)


def _cut(full, S, crit):
    """A slot request without stop strings cut at HF's first hit of crit (EOS ids already end `full`)."""
    full = full.cpu()
    for t in range(S, full.shape[1]):
        if bool(crit(full[:, :t + 1], None)[0]):
            return full[:, :t + 1], True
    return full, False


@pytest.mark.parametrize("pool", ["bf16", "fp8_e4m3"])
def test_prefix_cache_swap_pools(micro, pool):
    """Four sessions behind a shared system prompt (prefix-cache hits), half swapped to the host tier between turns, on the
    bf16 and e4m3 pools: each request with stop strings equals the same request without them, on the same configuration, cut
    at HF's first hit."""
    from ultravox_b200.serving import SlotScheduler
    from ultravox_b200.stop_strings import StopStrings
    cfg, model, tok = micro
    system = torch.randint(8, 1000, (1, 130), generator=torch.Generator().manual_seed(5))

    def run(stops):
        s = SlotScheduler(model, slots=4, max_len=256, eos_token_ids=EOS, kv_pages=64, prefix_cache=True, host_kv_pages=16,
                          kv_cache_dtype=pool, max_stop_table=40000)
        sids = {i: s.open_session() for i in range(4)}
        ids = {i: torch.cat([system, torch.randint(8, 1000, (1, 4 + i), generator=torch.Generator().manual_seed(i))], 1).cuda()
               for i in range(4)}
        kw = lambda i, turn: stops.get((i, turn), {})        # noqa: E731
        r = {i: s.submit(dict(input_ids=ids[i]), max_new_tokens=12, session=sids[i], **kw(i, 0)) for i in range(4)}
        first = s.run()
        out = {}
        for i in range(4):
            a = first[r[i]]
            out[(i, 0)] = (a, ids[i].shape[1])
            follow = torch.cat([a, torch.randint(8, 1000, (1, 3), generator=torch.Generator().manual_seed(40 + i)).cuda()], 1)
            if i % 2:
                s.offload_session(sids[i])
                assert s.session_on_host(sids[i])
            r[i] = s.submit(dict(input_ids=follow), max_new_tokens=12, session=sids[i], **kw(i, 1))
            out[(i, 1)] = follow.shape[1]
        second = s.run()
        for i in range(4):
            out[(i, 1)] = (second[r[i]], out[(i, 1)])
        return out, s.cached_tokens

    plain, _ = run({})
    stops = {}
    for (i, turn), (seq, S) in plain.items():
        txt = tok.decode(seq[0, S:].tolist())
        if txt[3:7] and (i + turn) % 2 == 0:
            stops[(i, turn)] = dict(stop_strings=[txt[3:7]], tokenizer=tok)
    got, cached = run(stops)
    assert any(v > 0 for v in cached.values())             # prefix-cache hits happened
    cut = 0
    for key, (seq, S) in plain.items():
        if key not in stops:
            continue
        want, hit = _cut(seq, S, StopStrings.build(tok, stops[key]["stop_strings"]).criteria)
        cut += hit
        assert torch.equal(got[key][0].cpu(), want), key
    assert cut >= 2


def test_8b_widths_shallow():
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    from ultravox_b200.serving import SlotScheduler
    from ultravox_b200.stop_strings import StopStrings
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=2))
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    tok = make_tokenizer(cfg.vocab_size, "bytelevel", seed=2)
    g = torch.Generator().manual_seed(7)
    reqs = [torch.randint(8, 100000, (1, 9 + i), generator=g).cuda() for i in range(8)]
    s = SlotScheduler(model, slots=8, max_len=64, eos_token_ids=EOS, max_stop_table=1 << 21)
    plain = []
    for ids in reqs:
        rid = s.submit(dict(input_ids=ids), max_new_tokens=10)
        plain.append(s.run()[rid])
    kws = []
    for i, (ids, p) in enumerate(zip(reqs, plain)):
        txt = tok.decode(p[0, ids.shape[1]:].tolist())
        kws.append(dict(stop_strings=[txt[4 + i:8 + i]], tokenizer=tok) if i % 2 == 0 and txt[4 + i:8 + i] else {})
    rids = [s.submit(dict(input_ids=ids), max_new_tokens=10, **kw) for ids, kw in zip(reqs, kws)]
    busy = s.run()
    cut = 0
    for i, (ids, p, kw) in enumerate(zip(reqs, plain, kws)):
        want, hit = (_cut(p, ids.shape[1], StopStrings.build(tok, kw["stop_strings"]).criteria) if kw else (p.cpu(), False))
        cut += hit
        assert torch.equal(busy[rids[i]].cpu(), want), i
    assert cut >= 2
