"""Continuous batching: the slot kernels (uvx_sample_slots, uvx_repetition_penalty_slots, uvx_slot_finish) against the kernels
and rules they restate, SlotDecodeEngine / SlotScheduler against generate() on each request alone, row isolation inside a busy
engine (bit for bit, since every decode-step kernel is row-independent at a fixed row count), the one-time graph capture, the
fp32 oracle, and LocalInference.infer_many."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V8B = 128256


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def wave(i, n):
    return np.random.default_rng(1000 + i).standard_normal(n).astype(np.float32)


def build(name="micro", **kw):
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    cfg = preset(name, **kw)
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def audio_request(cfg, n_samples, seed, text_pre=8, text_post=5):
    """Processor-shaped features of one clip: 8 ids, the audio placeholders, 5 ids; mel computed on the device."""
    from oracle import logmel as ol
    from ultravox_b200 import ops
    padded, frames = ol.pad_batch([wave(seed, n_samples)])
    g = torch.Generator().manual_seed(seed)
    tok = int(-(-int(frames[0]) // 16))
    ids = torch.randint(0, min(cfg.vocab_size, 1000), (1, text_pre + tok + text_post), generator=g)
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    return dict(input_ids=ids.cuda(), audio_values=mel, audio_token_start_idx=torch.tensor([text_pre]).cuda(),
                audio_lens=torch.tensor([int(frames[0])]).cuda(), audio_token_len=torch.tensor([tok], dtype=torch.int32).cuda(),
                audio_batch_size=torch.ones(1, dtype=torch.int64).cuda())


def text_request(cfg, S, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(input_ids=torch.randint(0, min(cfg.vocab_size, 1000), (1, S), generator=g).cuda())


def gen_alone(model, feats, n, eos, settings, seed):
    """generate() on one request (the yardstick)."""
    kw = dict(settings)
    if kw.get("do_sample"):
        kw["generator"] = torch.Generator(device="cuda").manual_seed(seed)
    return model.generate(max_new_tokens=n, eos_token_id=eos, **feats, **kw)


def serve(sched, reqs):
    """reqs: (features, n, settings, seed) -> submitted ids in order."""
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


# ================================================================================================ 1. kernels
def test_sample_slots_bit_exact_per_row(ops):
    """8 rows of mixed settings at V = 128256: each row equals the existing kernel it maps to on the same uniform."""
    B, V, W = 8, V8B, 40
    g = torch.Generator().manual_seed(0)
    lg = torch.randn(B, V, generator=g) * 3
    lg[4] = -float("inf")                                            # all -inf, sampled
    lg[5, [17, 70000, 128000]] = 40.0                                # tied maximum across warps, greedy
    lg[6, [3, 9]] = 25.0                                             # inactive
    lg[7, [1000, 1001, 99999]] = 12.0                                # tied maximum, sampled with top-p
    lg = lg.cuda()
    # (temperature, top_k, top_p, active)
    rows = [(0.0, 0, 1.0, 1), (0.7, 50, 1.0, 1), (1.0, 0, 0.9, 1), (0.8, 50, 0.0, 1),
            (1.0, 0, 0.9, 1), (0.0, 0, 1.0, 1), (0.9, 50, 1.0, 0), (0.5, 0, 0.5, 1)]
    u = torch.rand(B, W, generator=g).cuda()
    n_new = torch.tensor([3, 0, 7, 39, 1, 2, 5, 11], dtype=torch.int32).cuda()
    f32, i32 = dict(dtype=torch.float32, device="cuda"), dict(dtype=torch.int32, device="cuda")
    temp = torch.tensor([r[0] for r in rows], **f32)
    top_k = torch.tensor([r[1] for r in rows], **i32)
    top_p = torch.tensor([r[2] for r in rows], **f32)
    active = torch.tensor([r[3] for r in rows], **i32)
    for trial in range(2):
        out = torch.full((B,), -7, dtype=torch.int64, device="cuda")
        ops.sample_slots(lg, temp, top_k, top_p, u, n_new, active, out)
        got = out.cpu().tolist()
        for b, (T, k, p, on) in enumerate(rows):
            if not on:
                assert got[b] == -7, b
                continue
            if T <= 0:
                want = int(ops.argmax(lg[b:b + 1].contiguous())[0])
            else:
                ub = u[b, int(n_new[b])].reshape(1).contiguous()
                want = int(ops.sample(lg[b:b + 1].contiguous(), T, k, ub, top_p=p)[0])
            assert got[b] == want, (trial, b, got[b], want)
        assert got[5] == 17
        n_new = (n_new + 1) % W
    # a greedy all -inf row resolves to 0 like uvx_argmax
    temp[4] = 0.0
    out = torch.full((B,), -7, dtype=torch.int64, device="cuda")
    ops.sample_slots(lg, temp, top_k, top_p, u, n_new, active, out)
    assert int(out[4]) == 0 == int(ops.argmax(lg[4:5].contiguous())[0])
    with pytest.raises(Exception):
        ops.sample_slots(lg.cpu(), temp, top_k, top_p, u, n_new, active, out)


def test_repetition_penalty_slots_matches_hf_per_row(ops):
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor
    g = torch.Generator().manual_seed(3)
    B, V, cap = 5, V8B, 60
    logits = torch.randn(B, V, generator=g) * 4
    seq = torch.randint(0, V, (B, cap), generator=g)
    seq[0, 5] = seq[0, 2]
    seq[1, :7] = 11
    lens = [23, 9, 60, 1, 30]
    pens = [1.1, 1.3, 0.8, 1.0, 1.2]
    act = [1, 1, 1, 1, 0]
    want = logits.clone()
    for b in range(B):
        if act[b] and pens[b] != 1.0:
            want[b:b + 1] = RepetitionPenaltyLogitsProcessor(pens[b])(seq[b:b + 1, :lens[b]], logits[b:b + 1].clone())
    got = logits.clone().cuda()
    ops.repetition_penalty_slots_(got, seq.cuda(), torch.tensor(lens, dtype=torch.int32).cuda(), torch.tensor(pens).cuda(),
                                  torch.tensor(act, dtype=torch.int32).cuda(), torch.empty(B, cap, device="cuda"))
    assert torch.equal(got.cpu(), want)
    assert torch.equal(got[3].cpu(), logits[3]) and torch.equal(got[4].cpu(), logits[4])


def test_slot_finish_matches_python_rule(ops):
    g = torch.Generator().manual_seed(5)
    B, W = 37, 50
    eos = [7, 9, 300]
    for trial in range(6):
        tok = torch.randint(0, 12, (B,), generator=g)
        tok[::5] = 300
        done = (torch.rand(B, generator=g) < 0.25).int()
        active = (torch.rand(B, generator=g) < 0.8).int()
        cur_len = torch.randint(5, 40, (B,), generator=g).int()
        n_new = torch.randint(0, 8, (B,), generator=g).int()
        max_new = n_new + torch.randint(1, 4, (B,), generator=g).int()
        pos = torch.randint(0, 40, (B,), generator=g).int()
        lens, rope = pos + 1, pos - torch.randint(0, 3, (B,), generator=g).int()
        seq = torch.randint(0, 1000, (B, W), generator=g)
        st = [t.clone() for t in (done, seq, cur_len, n_new, pos, lens, rope)]
        # the rule, in Python
        open_rows = 0
        for b in range(B):
            if not active[b] or done[b]:
                continue
            t = int(tok[b])
            seq[b, cur_len[b]] = t
            cur_len[b] += 1
            n_new[b] += 1
            d = int(n_new[b] >= max_new[b] or t in eos)
            done[b] = d
            if not d:
                pos[b] += 1
                lens[b] += 1
                rope[b] += 1
                open_rows += 1
        dv = [t.cuda() for t in st]
        n_open = torch.full((1,), -1, dtype=torch.int32, device="cuda")
        ops.slot_finish(tok.cuda(), dv[0], torch.tensor(eos).cuda(), dv[1], dv[2], dv[3], max_new.cuda(), active.cuda(), dv[4], dv[5],
                        dv[6], n_open)
        for a, b_ in zip(dv, (done, seq, cur_len, n_new, pos, lens, rope)):
            assert torch.equal(a.cpu(), b_), trial
        assert int(n_open) == open_rows


# ================================================================================================ 2. one slot is generate()
def test_one_slot_is_generate():
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    a = audio_request(cfg, 16000, 1)
    b = audio_request(cfg, 24000, 2)
    t = text_request(cfg, 11, 3)
    greedy = gen_alone(model, a, 12, None, {}, 0)
    S = a["input_ids"].shape[1]
    eos = [int(greedy[0, S + 3])]
    cases = [(a, 12, {}, 0), (b, 10, dict(do_sample=True, temperature=0.7, top_k=50), 11),
             (t, 9, dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9), 12), (a, 8, dict(repetition_penalty=1.3), 0),
             (b, 7, dict(do_sample=True, temperature=0.6, top_p=0.5, repetition_penalty=1.3), 13)]
    sched = SlotScheduler(model, slots=1, max_len=64)
    for feats, n, settings, seed in cases:
        rid, = serve(sched, [(feats, n, settings, seed)])
        got = sched.run()[rid]
        want = gen_alone(model, feats, n, None, settings, seed)
        assert torch.equal(got, want), settings
    # EOS stop: the sequence ends with the first EOS, like generate()
    sched_e = SlotScheduler(model, slots=1, max_len=64, eos_token_ids=eos)
    rid, = serve(sched_e, [(a, 12, {}, 0)])
    got = sched_e.run()[rid]
    want = gen_alone(model, a, 12, eos, {}, 0)
    assert torch.equal(got, want) and got.shape[1] < S + 12 and int(got[0, -1]) == eos[0]
    # three requests back to back through the one slot, cache NaN-filled first: no leak from the previous occupant
    poison(sched)
    ids = serve(sched, cases[:3])
    res = sched.run()
    for rid, (feats, n, settings, seed) in zip(ids, cases[:3]):
        assert torch.equal(res[rid], gen_alone(model, feats, n, None, settings, seed)), settings
    assert sched.engine.captures == 1 and sched.steps > 20


def test_submit_validation():
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    sched = SlotScheduler(model, slots=2, max_len=32)
    t = text_request(cfg, 20, 1)
    with pytest.raises(ValueError):
        sched.submit(t, max_new_tokens=13)                            # 20 + 13 > 32
    with pytest.raises(ValueError):
        sched.submit(t, max_new_tokens=4, do_sample=True, top_p=1.5)
    with pytest.raises(ValueError):
        sched.submit(t, max_new_tokens=4, top_p=float("nan"))
    with pytest.raises(NotImplementedError):
        sched.submit(t, max_new_tokens=4, num_beams=2)
    with pytest.raises(ValueError):
        sched.submit(dict(input_ids=t["input_ids"].repeat(2, 1)), max_new_tokens=4)
    assert sched.pending() == []
    rid = sched.submit(t, max_new_tokens=12)
    assert torch.equal(sched.run()[rid], model.generate(**t, max_new_tokens=12))


# ================================================================================================ 3/4. row isolation and the graph
def _mixed_requests(cfg, n_req, seed, audio=True):
    settings = [{}, dict(do_sample=True, temperature=0.7, top_k=50), dict(do_sample=True, temperature=1.0, top_k=0, top_p=0.9),
                dict(repetition_penalty=1.3), dict(do_sample=True, temperature=0.8, top_p=0.6, repetition_penalty=1.2)]
    rng = np.random.default_rng(seed)
    reqs = []
    for i in range(n_req):
        if audio and i % 3 == 0:
            feats = audio_request(cfg, int(rng.choice([8000, 16000, 30000])), 100 + i)
        else:
            feats = text_request(cfg, int(rng.integers(4, 30)), 200 + i)
        reqs.append((feats, int(rng.integers(2, 24)), settings[i % len(settings)], 300 + i))
    return reqs


def _isolation(model, reqs, eos, slots, max_len):
    from ultravox_b200.serving import SlotScheduler
    busy = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos, sync_every=3)
    poison(busy)
    ids = serve(busy, reqs)
    res = busy.run()
    assert busy.engine.captures == 1
    alone = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos)
    for rid, r in zip(ids, reqs):
        poison(alone)
        a_rid, = serve(alone, [r])
        assert torch.equal(res[rid], alone.run()[a_rid]), rid
    assert alone.engine.captures == 1
    eager = SlotScheduler(model, slots=slots, max_len=max_len, eos_token_ids=eos, sync_every=3, use_graph=False)
    e_ids = serve(eager, reqs)
    e_res = eager.run()
    assert eager.engine.graph is None and eager.engine.captures == 0
    for rid, e_rid in zip(ids, e_ids):
        assert torch.equal(res[rid], e_res[e_rid]), rid
    return res, ids


def test_row_isolation_eight_slots():
    """20 requests (audio and text, mixed prompt lengths, budgets and settings) through 8 slots, admitted as slots free up:
    each equals the same request alone in an 8-slot engine whose other slots idle on NaN-filled cache rows, and generate()."""
    cfg, model = build()
    reqs = _mixed_requests(cfg, 20, 0)
    first = gen_alone(model, reqs[0][0], 24, None, {}, 0)
    S0 = reqs[0][0]["input_ids"].shape[1]
    eos = [int(first[0, S0 + 4])]                         # some requests stop early on it
    res, ids = _isolation(model, reqs, eos, 8, 256)
    stops = 0
    for rid, (feats, n, settings, seed) in zip(ids, reqs):
        S = feats["input_ids"].shape[1]
        stops += res[rid].shape[1] < S + n
        assert res[rid].shape[1] <= S + n
    assert stops >= 1, "no request ended on the EOS id"


def test_row_isolation_at_8b_widths():
    from ultravox_b200.config import PRESETS
    base = PRESETS["v0_5_8b"]
    cfg, model = build("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                       text_config=dict(base["text_config"], num_hidden_layers=2, vocab_size=32000))
    reqs = _mixed_requests(cfg, 10, 1, audio=False)
    _isolation(model, reqs, None, 8, 64)


# ================================================================================================ 5. oracle
def test_served_greedy_request_matches_stepwise_oracle():
    """A greedy audio request in a 4-slot engine next to three sampled text requests, teacher-forced through the fp32 oracle
    with the bar of test_generate_greedy_matches_stepwise_oracle."""
    from oracle import model as om
    from ultravox_b200.serving import SlotScheduler
    cfg, model = build()
    sd, sh = om.state_dict_fp32(model), om.shapes_from_config(cfg)
    a = audio_request(cfg, 16000, 1)
    others = [(text_request(cfg, 7 + 5 * i, 40 + i), 10, dict(do_sample=True, temperature=0.8), 50 + i) for i in range(3)]
    sched = SlotScheduler(model, slots=4, max_len=64)
    ids = serve(sched, others[:2] + [(a, 6, {}, 0)] + others[2:])
    seq = sched.run()[ids[2]]
    n_new = 6
    S = a["input_ids"].shape[1]
    assert seq.shape == (1, S + n_new)
    st = {}
    om.forward(sd, sh, a["input_ids"].cpu(), a["audio_values"].cpu().to(torch.bfloat16).float(), a["audio_token_start_idx"].cpu(),
               a["audio_lens"].cpu(), a["audio_token_len"].cpu(), a["audio_batch_size"].cpu(), last_only=True, stages=st)
    cur = st["inputs_embeds"]
    table = sd["language_model.model.embed_tokens.weight"]
    exact = 0
    for t in range(n_new):
        ref = om.llama_forward(sd, sh, cur, last_only=True).view(-1)
        tok = int(seq[0, S + t])
        assert tok in ref.topk(5).indices.tolist(), t
        assert float(ref.max() - ref[tok]) < 3e-2 * float(ref.abs().max()), t
        exact += int(tok == int(ref.argmax()))
        cur = torch.cat([cur, table[tok][None, None]], dim=1)
    assert exact >= n_new - 2, exact


# ================================================================================================ 6. infer_many
class _ChatTok:
    eos_token = "<|eot_id|>"
    eos_token_id = 1000
    padding_side = "left"
    pad_token_id = 1000
    added_tokens_encoder = {"<|eot_id|>": 1000}
    model_input_names = ["input_ids", "attention_mask"]

    def get_vocab(self):
        return {self.eos_token: self.eos_token_id}

    def convert_tokens_to_ids(self, t):
        return self.added_tokens_encoder[t]

    def __call__(self, parts, add_special_tokens=False, **kw):
        out = []
        for p in parts:
            words = p.replace(self.eos_token, f" {self.eos_token} ").split()
            out.append([self.eos_token_id if w == self.eos_token else (sum(map(ord, w)) * 31 + len(w)) % 1000 for w in words])
        return {"input_ids": out}

    def apply_chat_template(self, messages, add_generation_prompt=True, tokenize=False, chat_template=None, **kw):
        text = " ".join(f"<s> {m['role']} : {m['content']} {self.eos_token}" for m in messages)
        return text + (" <s> assistant :" if add_generation_prompt else "")

    def decode(self, ids, skip_special_tokens=True):
        ids = [int(i) for i in (ids.tolist() if hasattr(ids, "tolist") else ids)]
        return " ".join(f"t{i}" for i in ids if not (skip_special_tokens and i == self.eos_token_id))


def test_infer_many():
    from ultravox_b200.data_proc import VoiceSample
    from ultravox_b200.inference import LocalInference
    from ultravox_b200.processing import MelSpec, UltravoxProcessor
    cfg, model = build()
    tok = _ChatTok()
    proc = UltravoxProcessor(MelSpec(feature_size=80), tok, mel_device="cuda")
    inf = LocalInference(model, proc, tok, conversation_mode=False)
    samples = [VoiceSample.from_prompt_and_raw("Listen to <|audio|> and answer", wave(1, 16000), 16000),
               VoiceSample.from_prompt("plain text question without audio"),
               VoiceSample.from_prompt_and_raw("<|audio|> what", (wave(2, 48000) * 3000).astype(np.int16), 48000),
               VoiceSample.from_prompt("another much longer plain text question for a longer prompt"),
               VoiceSample.from_prompt_and_raw("tell me about <|audio|>", wave(3, 32000), 16000)]
    singles = [inf.infer(s, max_tokens=7) for s in samples]
    many1 = inf.infer_many(samples, max_tokens=7, slots=1)
    assert [(o.text, o.input_tokens, o.output_tokens) for o in many1] == [(o.text, o.input_tokens, o.output_tokens) for o in singles]
    many4 = inf.infer_many(samples, max_tokens=7, slots=4)
    for s, got in zip(samples, many4):
        alone = inf.infer_many([s], max_tokens=7, slots=4)[0]
        assert (got.text, got.input_tokens, got.output_tokens) == (alone.text, alone.input_tokens, alone.output_tokens)
    assert inf.infer_many([], max_tokens=3) == []
    with pytest.raises(ValueError):
        inf.infer_many(samples[:2], max_tokens=7, max_len=10)
    conv = LocalInference(model, proc, tok, conversation_mode=True)
    with pytest.raises(AssertionError):
        conv.infer_many(samples[:1])
