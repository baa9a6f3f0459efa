"""Token constraints in the continuous-batching slot step: SlotScheduler(max_constraint_tokens=N) and submit(no_repeat_ngram_size=,
sequence_bias=, bad_words_ids=, min_length=, min_new_tokens=, suppress_tokens=, begin_suppress_tokens=) against generate() on
each request alone (tokens and raw log-probs), a busy 8-slot engine against the same requests alone, graph against eager, a
chunked prompt, the lookup step, paged sessions / the prefix cache / the e4m3 pool / host swap, 8B widths, the step launch
counts and the argument errors."""
import pytest
import torch

from test_logprobs_gpu import _logprobs_of_logits, audio_request, build, serve, sharpen, text_request

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def micro():
    cfg, model = build()
    sharpen(model, cfg)
    return cfg, model


EOS = [7, 11]


def _settings(i):
    """A different mix of constraints (and sampling / penalty) per request index."""
    opts = [dict(no_repeat_ngram_size=2), dict(min_new_tokens=6, suppress_tokens=[3, 5]),
            dict(sequence_bias=[[[9], 4.0], [[9, 12], -30.0]], begin_suppress_tokens=[9]),
            dict(bad_words_ids=[[12], [4, 6], [7]], no_repeat_ngram_size=3, repetition_penalty=1.2),
            dict(min_length=20, do_sample=True, temperature=0.8, top_k=40),
            dict(no_repeat_ngram_size=1, sequence_bias={(2,): 1.5}, do_sample=True, temperature=1.0, top_p=0.9),
            {},                                        # a request without constraints next to constrained ones
            dict(no_repeat_ngram_size=2, bad_words_ids=[[8, 8]], min_new_tokens=3, repetition_penalty=1.3)]
    return dict(opts[i % len(opts)])


def _requests(cfg, n_req, long_at=None):
    reqs = []
    for i in range(n_req):
        if i == long_at:
            feats = text_request(cfg, 300, 900 + i)                 # > PREFILL_ROWS: prefilled in chunks
        elif i % 3 == 0:
            feats = audio_request(cfg, 16000, 100 + i)
        else:
            feats = text_request(cfg, 6 + 3 * i, 200 + i)
        reqs.append((feats, 10 + i % 5, _settings(i), 50 + i))
    return reqs


def _generate(model, feats, n, settings, seed, **extra):
    kw = dict(settings)
    if kw.get("do_sample"):
        kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
    return model.generate(max_new_tokens=n, eos_token_id=EOS, **feats, **kw, **extra)


def test_one_slot_equals_generate(micro, ops):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    sched = SlotScheduler(model, slots=1, max_len=400, eos_token_ids=EOS, max_logprobs=3, max_constraint_tokens=16)
    for i, (feats, n, settings, seed) in enumerate(_requests(cfg, 8)):
        rid, = serve(sched, [(feats, n, dict(settings, logprobs=3), seed)])
        got = sched.run()[rid]
        out = _generate(model, feats, n, settings, seed, return_dict_in_generate=True, output_logits=True)
        assert torch.equal(got, out.sequences), settings
        S = feats["input_ids"].shape[1]
        lp = sched.logprobs[rid]
        w_lp, w_ids, w_top = _logprobs_of_logits(ops, torch.cat(out.logits), out.sequences[0, S:], 3)
        assert torch.equal(lp.token_logprobs, w_lp) and torch.equal(lp.top_ids, w_ids), settings   # the raw distribution
        if settings.get("min_new_tokens"):
            assert not set(got[0, S:S + settings["min_new_tokens"]].tolist()) & set(EOS)
        if settings.get("no_repeat_ngram_size") == 2:
            seq = got[0].tolist()
            grams = list(zip(seq, seq[1:]))
            assert len(set(grams)) == len(grams)
    assert sched.engine.captures == 1


def _serve_all(sched, reqs):
    ids = serve(sched, reqs)
    out = sched.run()
    return [out[i] for i in ids]


def test_busy_equals_alone_graph_eager_chunked(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    mk = lambda **kw: SlotScheduler(model, slots=8, max_len=400, eos_token_ids=EOS, sync_every=3,  # noqa: E731
                                    max_constraint_tokens=16, **kw)
    alone_s = mk()
    reqs = _requests(cfg, 20)
    busy = _serve_all(mk(), reqs)
    for i, r in enumerate(reqs):
        alone, = _serve_all(alone_s, [r])
        assert torch.equal(busy[i], alone), (i, r[2])
    # a prompt prefilled in chunks: graph == eager for every request; the chunked one == alone (the decode rows of a mixed
    # step run at 256 rows, so the others differ from a plain step there)
    reqs = _requests(cfg, 20, long_at=5)
    busy = _serve_all(mk(), reqs)
    eager = _serve_all(mk(use_graph=False), reqs)
    for i in range(len(reqs)):
        assert torch.equal(busy[i], eager[i]), i
    alone, = _serve_all(alone_s, [reqs[5]])
    assert torch.equal(busy[5], alone)
    # a scheduler built without constraints serves the unconstrained requests as before, with the same step launches
    plain = SlotScheduler(model, slots=8, max_len=400, eos_token_ids=EOS, sync_every=3)
    s = mk()
    free = [r for r in reqs if not ({"no_repeat_ngram_size", "min_new_tokens", "min_length", "bad_words_ids", "sequence_bias",
                                     "suppress_tokens", "begin_suppress_tokens"} & set(r[2]))]
    assert free
    for a, b in zip(_serve_all(plain, free), _serve_all(s, free)):
        assert torch.equal(a, b)
    assert s.engine.launches_per_step == plain.engine.launches_per_step + 1


def test_launch_counts_unchanged_without_constraints(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    reqs = _requests(cfg, 3, long_at=1)
    counts = []
    for kw in ({}, dict(max_constraint_tokens=None), dict(max_constraint_tokens=8)):
        s = SlotScheduler(model, slots=4, max_len=400, eos_token_ids=EOS, prompt_lookup_num_tokens=2, **kw)
        _serve_all(s, [(f, n, {"prompt_lookup_num_tokens": 2}, seed) for f, n, _, seed in reqs])
        e = s.engine
        counts.append((e.launches_per_step, e.launches_per_mixed_step, e.launches_per_lookup_step))
    assert counts[0] == counts[1]
    assert all(c > 0 for c in counts[0])
    assert counts[2] == tuple(c + 1 for c in counts[0])


def test_lookup_step_equals_plain_slots(micro):
    """Lookup with 2 slots x (K + 1 = 4) rows gives each request the tokens of a plain engine of 8 slots."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    base = torch.randint(1, 1000, (1, 6), generator=torch.Generator().manual_seed(8))
    reqs = []
    for i in range(4):
        ids = torch.cat([base, base, base[:, :3], torch.tensor([[20 + i]])], 1).cuda()     # repeats: drafts are proposed
        reqs.append((dict(input_ids=ids), 14, _settings(i), 70 + i))
    look = SlotScheduler(model, slots=2, max_len=128, eos_token_ids=EOS, prompt_lookup_num_tokens=3, max_constraint_tokens=16)
    plain = SlotScheduler(model, slots=8, max_len=128, eos_token_ids=EOS, max_constraint_tokens=16)
    got = _serve_all(look, [(f, n, dict(s, prompt_lookup_num_tokens=3), seed) for f, n, s, seed in reqs])
    want = _serve_all(plain, reqs)
    for g, w, r in zip(got, want, reqs):
        assert torch.equal(g, w), r[2]
    assert look.engine.launches_per_lookup_step > 0


@pytest.mark.parametrize("pool", ["bf16", "fp8_e4m3"])
def test_paged_sessions_prefix_swap(micro, pool):
    """Paged engine: a session's constrained turns equal chained generate(past_key_values=...) (one slot, bf16); busy == alone
    with sessions, the prefix cache and the host tier, on the bf16 and the e4m3 pool."""
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    kw = dict(kv_pages=64, max_constraint_tokens=16, eos_token_ids=EOS, kv_cache_dtype=pool)
    if pool == "bf16":
        s = SlotScheduler(model, slots=1, max_len=256, **kw)
        sid = s.open_session()
        t1 = text_request(cfg, 12, 1)
        r1, = serve(s, [(t1, 8, _settings(0), 1)])
        a1 = s.run()[r1]
        g1 = _generate(model, t1, 8, _settings(0), 1, return_dict_in_generate=True)
        assert torch.equal(a1, g1.sequences)
        s2 = SlotScheduler(model, slots=1, max_len=256, **kw)
        sid = s2.open_session()
        r1, = [s2.submit(t1, max_new_tokens=8, session=sid, **_settings(0))]
        a1 = s2.run()[r1]
        follow = torch.cat([a1, torch.randint(1, 1000, (1, 5), generator=torch.Generator().manual_seed(3)).cuda()], 1)
        r2 = s2.submit(dict(input_ids=follow), max_new_tokens=9, session=sid, **_settings(2))
        a2 = s2.run()[r2]
        g2 = _generate(model, dict(input_ids=follow), 9, _settings(2), 0, past_key_values=g1.past_key_values)
        assert torch.equal(a2, g2)
    # four sessions at once behind a shared system prompt (prefix-cache hits), second turns constrained differently, half of
    # the sessions swapped to the host tier in between: the same bits as a pool that never swaps, and graph == eager
    system = torch.randint(1, 1000, (1, 130), generator=torch.Generator().manual_seed(5))

    def opts(i):
        o = _settings(i)
        if o.get("do_sample"):
            o["generator"] = torch.Generator(device="cuda").manual_seed(60 + i)
        return o

    def run(offload, use_graph=True):
        s = SlotScheduler(model, slots=4, max_len=256, prefix_cache=True, host_kv_pages=16, use_graph=use_graph, **kw)
        outs = {}
        sids = {i: s.open_session() for i in range(4)}
        for i in range(4):
            ids = torch.cat([system, torch.randint(1, 1000, (1, 4 + i), generator=torch.Generator().manual_seed(i))], 1).cuda()
            outs[i] = [s.submit(dict(input_ids=ids), max_new_tokens=8, session=sids[i], **opts(i))]
        first = s.run()
        for i in range(4):
            a = first[outs[i][0]]
            follow = torch.cat([a, torch.randint(1, 1000, (1, 3), generator=torch.Generator().manual_seed(40 + i)).cuda()], 1)
            if offload and i % 2:
                s.offload_session(sids[i])          # restored at its next turn's admission
                assert s.session_on_host(sids[i])
            outs[i].append(s.submit(dict(input_ids=follow), max_new_tokens=8, session=sids[i], **opts(i + 3)))
        second = s.run()
        return [(first[outs[i][0]], second[outs[i][1]]) for i in range(4)]

    ref = run(False)
    for other in (run(True), run(False, use_graph=False)):
        for i in range(4):
            assert torch.equal(ref[i][0], other[i][0]) and torch.equal(ref[i][1], other[i][1]), (pool, i)


def test_8b_widths_shallow(ops):
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    from ultravox_b200.serving import SlotScheduler
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=2))
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    reqs = [(text_request(cfg, 9 + i, 300 + i), 8, _settings(i), 80 + i) for i in range(8)]
    s = SlotScheduler(model, slots=8, max_len=64, eos_token_ids=EOS, max_constraint_tokens=16)
    busy = _serve_all(s, reqs)
    for i, r in enumerate(reqs):
        alone, = _serve_all(s, [r])
        assert torch.equal(busy[i], alone), i
    one = SlotScheduler(model, slots=1, max_len=64, eos_token_ids=EOS, max_constraint_tokens=16)
    for r in reqs[:3]:
        got, = _serve_all(one, [r])
        assert torch.equal(got, _generate(model, *r)), r[2]


def test_errors(micro):
    from ultravox_b200.serving import SlotScheduler
    cfg, model = micro
    t = text_request(cfg, 8, 1)
    plain = SlotScheduler(model, slots=1, max_len=64, eos_token_ids=EOS)
    with pytest.raises(ValueError, match="max_constraint_tokens"):
        plain.submit(t, max_new_tokens=4, no_repeat_ngram_size=2)
    small = SlotScheduler(model, slots=1, max_len=64, eos_token_ids=EOS, max_constraint_tokens=4)
    with pytest.raises(ValueError, match="max_constraint_tokens"):
        small.submit(t, max_new_tokens=4, bad_words_ids=[[1, 2, 3], [4, 5]])
    with pytest.raises(ValueError):
        small.submit(t, max_new_tokens=4, sequence_bias={(5,): 1})
    with pytest.raises(ValueError):
        SlotScheduler(model, slots=1, max_len=64, max_constraint_tokens=-1)
    rid = small.submit(t, max_new_tokens=4, bad_words_ids=[[1, 2], [4, 5]])      # exactly 4 ids fit
    assert small.run()[rid].shape[1] >= 9
