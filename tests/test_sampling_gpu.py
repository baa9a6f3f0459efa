"""Nucleus (top-p) sampling: uvx_sample_top_p, ops.sample(top_p=), DecodeEngine(top_p=) and generate(top_p=), against
transformers' own TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper applied in fp32 on the CPU to the same logits.

A row whose float64 cumulative mass (ascending, over the top-k survivors) comes within MARGIN of 1 - top_p below the maximum
is ambiguous: fp32 summation order alone can move its cut.  Such rows are skipped and counted, and there must be few.  Ties at
the cut are the one intended difference from HF (include/uvx.h): the library keeps or drops a tie group whole."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

MARGIN = 1e-5


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def hf_warp(logits, T, k, p):
    """[R, V] -> the scores HF samples from (filtered entries -inf), fp32 on the CPU."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = TemperatureLogitsWarper(T)(None, logits.float().cpu().clone())
    if k:
        s = TopKLogitsWarper(k)(None, s)
    if p < 1.0:
        s = TopPLogitsWarper(p)(None, s)
    return s


def hf_kept(logits, T, k, p):
    """[R, V] kept mask and the renormalised float64 distribution HF draws from."""
    s = hf_warp(logits, T, k, p)
    return torch.isfinite(s), torch.softmax(s.double(), -1)


def ambiguous(logits, T, k, p):
    """[R] bool: a float64 cumulative mass below the maximum lies within MARGIN of 1 - p."""
    x = logits.double().cpu() / T
    if k:
        x = x.masked_fill(x < x.topk(k, -1).values[:, -1:], -math.inf)
    c = torch.softmax(x, -1).sort(-1).values.cumsum(-1)[:, :-1]
    return ((c - (1.0 - p)).abs() < MARGIN).any(-1)


def grid(n):
    """n uniforms (j + 1/2) / n: every token whose renormalised mass exceeds 1/n covers a grid point and is drawn."""
    return ((torch.arange(n, dtype=torch.float64) + 0.5) / n).float().cuda()


def test_kept_set_and_distribution_small_vocab(ops):
    V, n = 1000, 1 << 16
    u = grid(n)
    g = torch.Generator().manual_seed(0)
    checked = skipped = 0
    for scale in (0.5, 2.0, 8.0):
        row = torch.randn(1, V, generator=g) * scale
        big = row.cuda().expand(n, V).contiguous()
        for T in (0.6, 1.0):
            for k in (0, 50):
                for p in (0.0, 0.5, 0.9, 0.95):
                    if bool(ambiguous(row, T, k, p)[0]):
                        skipped += 1
                        continue
                    kept, probs = hf_kept(row, T, k, p)
                    assert float(probs[0][kept[0]].min()) > 4.0 / n, (scale, T, k, p)    # every kept token is drawn
                    picks = ops.sample(big, T, k, u, top_p=p).cpu()
                    assert set(picks.unique().tolist()) == set(kept[0].nonzero().view(-1).tolist()), (scale, T, k, p)
                    hist = torch.bincount(picks, minlength=V).double() / n
                    assert float((hist - probs[0]).abs().max()) < 0.01, (scale, T, k, p)
                    if p == 0.0:
                        assert set(picks.tolist()) == {int(row.argmax())}
                    checked += 1
    assert skipped <= 2 and checked + skipped == 48, (checked, skipped)


def test_top_p_one_is_uvx_sample_bit_for_bit(ops):
    from ultravox_b200._lib import check, lib
    V, B = 128256, 8
    g = torch.Generator().manual_seed(1)
    lg = (torch.randn(B, V, generator=g) * 3).cuda()
    uu = torch.rand(6, B, generator=g).cuda()
    step = torch.tensor([4], dtype=torch.int32).cuda()
    stream = torch.cuda.current_stream().cuda_stream
    for k in (0, 50):
        for T in (0.6, 1.3):
            ref = torch.empty(B, dtype=torch.int64, device="cuda")
            check(lib().uvx_sample(lg.data_ptr(), B, V, T, k, uu.data_ptr(), step.data_ptr(), uu.stride(0), ref.data_ptr(), stream))
            via = torch.empty_like(ref)
            check(lib().uvx_sample_top_p(lg.data_ptr(), B, V, T, k, 1.0, uu.data_ptr(), step.data_ptr(), uu.stride(0),
                                         via.data_ptr(), stream))
            assert torch.equal(ops.sample(lg, T, k, uu, step, top_p=1.0), ref)
            assert torch.equal(ops.sample(lg, T, k, uu, step), ref)
            assert torch.equal(via, ref)
    out = torch.empty(B, dtype=torch.int64, device="cuda")
    for bad in (1.5, -0.1, float("nan")):                      # the C entry rejects what generate() rejects
        rc = lib().uvx_sample_top_p(lg.data_ptr(), B, V, 1.0, 0, bad, uu.data_ptr(), None, 0, out.data_ptr(), stream)
        assert rc != 0, bad


def _tile_draws(ops, rows, T, k, p, steps, copies):
    """Draws steps * copies samples of each of the R rows: the rows tiled `copies` times, one launch per step-indexed u row."""
    R, V = rows.shape
    big = rows.cuda().repeat(copies, 1)
    g = torch.Generator(device="cuda").manual_seed(7)
    u = torch.rand(steps, R * copies, device="cuda", generator=g)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = []
    for s in range(steps):
        step.fill_(s)
        out.append(ops.sample(big, T, k, u, step, top_p=p).view(copies, R))
    return torch.cat(out).cpu().T                              # [R, steps * copies]


def test_full_vocabulary(ops):
    V, B, T = 128256, 8, 0.6
    g = torch.Generator().manual_seed(3)
    # peaked rows: 40 candidates far above a broad background (about 2 % of the mass), so the nucleus is tens of tokens
    peaked = torch.randn(B, V, generator=g) * 1.5
    for b in range(B):
        peaked[b, torch.randperm(V, generator=g)[:40]] = 9.0 + torch.randn(40, generator=g) * 0.8
    for k in (0, 50):
        amb = ambiguous(peaked, T, k, 0.9)
        assert int(amb.sum()) <= 1
        kept, probs = hf_kept(peaked, T, k, 0.9)
        picks = _tile_draws(ops, peaked, T, k, 0.9, steps=100, copies=128)          # 12800 draws per row, 102400 in all
        for b in range(B):
            if amb[b]:
                continue
            want = set(kept[b].nonzero().view(-1).tolist())
            assert 10 <= len(want) <= 40 and float(probs[b][kept[b]].min()) > 1e-3, (k, b, len(want))
            assert set(picks[b].unique().tolist()) == want, (k, b)
    # flat rows without top-k: the nucleus is most of the vocabulary, ~1e-5 of mass per token, so some token always sits
    # within MARGIN of the cut; every pick lies inside the nucleus widened by MARGIN, which differs from HF's by a few tokens
    flat = torch.randn(B, V, generator=g) * 0.5
    kept, _ = hf_kept(flat, T, 0, 0.9)
    x = flat.double() / T
    order = x.argsort(-1)
    cum = torch.empty_like(x).scatter_(1, order, torch.softmax(x, -1).gather(1, order).cumsum(-1))
    loose = cum > (1.0 - 0.9) - MARGIN
    assert int(kept.sum(-1).min()) > V // 2 and bool((kept <= loose).all()) and int((loose & ~kept).sum(-1).max()) < 10
    picks = _tile_draws(ops, flat, T, 0, 0.9, steps=8, copies=64)
    for b in range(B):
        assert bool(loose[b][picks[b]].all()), b
    # top_p = 0 is the argmax, with or without top-k
    for rows in (peaked, flat):
        for k in (0, 50):
            picks = _tile_draws(ops, rows, T, k, 0.0, steps=4, copies=16)
            assert bool((picks == rows.argmax(-1, keepdim=True)).all())


def test_tie_group_at_the_cut_is_kept_whole(ops):
    """One max (2.0), a tie group of four (1.0), 852 background entries tied at -5.0 and 143 at -inf.  Ascending cumulative
    mass: background 0.239, the group's members 0.352 / 0.465 / 0.579 / 0.692, the max 1."""
    V, n = 1000, 1 << 16
    row = torch.full((1, V), -5.0)
    row[0, ::7] = -math.inf
    group = [100, 200, 300, 400]
    row[0, 10] = 2.0
    row[0, group] = 1.0
    finite = set(torch.isfinite(row[0]).nonzero().view(-1).tolist())
    big = row.cuda().expand(n, V).contiguous()
    u = grid(n)
    cases = {0.5: {10, *group},          # the cut falls inside the group (HF keeps part of it): kept whole
             0.25: {10},                 # the cut falls above the group: dropped whole
             0.7: {10, *group},          # the cut falls between the background and the group
             0.8: finite}                # the cut falls inside the 852-way background tie: all of it is kept
    for p, want in cases.items():
        assert set(ops.sample(big, 1.0, 0, u, top_p=p).unique().tolist()) == want, p
    # HF's sort splits a straddling tie group; where no tie straddles the cut, HF agrees
    assert int(hf_kept(row, 1.0, 0, 0.5)[0].sum()) < 5 and int(hf_kept(row, 1.0, 0, 0.8)[0].sum()) < len(finite)
    assert set(hf_kept(row, 1.0, 0, 0.25)[0][0].nonzero().view(-1).tolist()) == {10}
    assert set(hf_kept(row, 1.0, 0, 0.7)[0][0].nonzero().view(-1).tolist()) == {10, *group}


# ------------------------------------------------------------------------------------------------------------------------
# engine and generate()

def _model(name="micro", enc_layers=None, llm_layers=None, logit_std=3.0):
    """Seeded random model whose lm_head is rescaled so the logits have std `logit_std`: at random init they are nearly flat
    and top-p would keep the whole top-k set, which would test nothing."""
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    kw = {}
    if enc_layers is not None:
        kw = dict(audio_config=dict(PRESETS[name]["audio_config"], encoder_layers=enc_layers),
                  text_config=dict(PRESETS[name]["text_config"], num_hidden_layers=llm_layers))
    cfg = preset(name, **kw)
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, min(cfg.vocab_size, 128000), (1, 12), generator=g).cuda()
    std = float(model(ids, logits_to_keep=1).logits.float().std())
    model.language_model.lm_head.weight.data.mul_(logit_std / std)
    return cfg, model


def _engine_steps_in_hf_kept_set(model, ids, n_steps, T, k, p, penalty):
    """Drives DecodeEngine step by step; every token must lie in the HF kept set of that step's post-penalty logits.
    Returns (steps checked, steps whose kept set is smaller than the top-k set, ambiguous steps)."""
    from ultravox_b200 import ops
    from ultravox_b200.engine import DecodeEngine
    B, S = ids.shape
    g = torch.Generator(device="cuda").manual_seed(5)
    de = DecodeEngine(model, B, S + n_steps + 2, temperature=T, top_k=k, top_p=p, repetition_penalty=penalty, generator=g)
    emb = ops.embed_splice(ids, model.language_model.model.embed_tokens.weight, None, None)
    tok = de.prefill(emb)
    checked = cut = amb = 0
    for t in range(n_steps):
        if t:
            tok = de.step().view(-1)
        lg = de.logits.float().cpu()
        kept, _ = hf_kept(lg, T, k, p)
        a = ambiguous(lg, T, k, p)
        for b in range(B):
            if a[b]:
                amb += 1
                continue
            assert bool(kept[b, int(tok[b])]), (t, b)
            checked += 1
            cut += int(kept[b].sum()) < k
    return checked, cut, amb


def test_generate_top_p_arguments():
    cfg, model = _model()
    ids = torch.randint(0, cfg.vocab_size, (1, 10), generator=torch.Generator().manual_seed(2)).cuda()
    for bad in (1.5, -0.1, float("nan")):
        with pytest.raises(ValueError):
            model.generate(ids, max_new_tokens=2, top_p=bad)
        with pytest.raises(ValueError):
            model.generate(ids, max_new_tokens=2, do_sample=True, top_p=bad)
    greedy = model.generate(ids, max_new_tokens=8)
    assert torch.equal(model.generate(ids, max_new_tokens=8, do_sample=False, top_p=0.5), greedy)


def test_engine_and_generate_micro():
    cfg, model = _model()
    ids = torch.randint(0, cfg.vocab_size, (1, 10), generator=torch.Generator().manual_seed(2)).cuda()
    kw = dict(max_new_tokens=16, do_sample=True, temperature=0.6, top_k=50, repetition_penalty=1.1)

    def gen(seed, **extra):
        return model.generate(ids, generator=torch.Generator(device="cuda").manual_seed(seed), **{**kw, **extra})

    s1, s2 = gen(11, top_p=0.9), gen(11, top_p=0.9)
    assert torch.equal(s1, s2)                                              # reproducible for a seeded generator
    assert torch.equal(gen(11, top_p=0.9, use_graph=False), s1)             # graph replay == eager steps
    assert torch.equal(gen(11, top_p=None), gen(11, top_p=1.0))             # no filter either way
    greedy = model.generate(ids, max_new_tokens=16, repetition_penalty=1.1)
    assert torch.equal(gen(11, top_p=0.0), greedy)                          # top_p = 0 keeps the argmax only
    checked, cut, amb = _engine_steps_in_hf_kept_set(model, ids, 16, 0.6, 50, 0.9, 1.1)
    assert amb <= 1 and checked >= 15 and cut >= checked // 2, (checked, cut, amb)
    # left-padded batch of 2 (kv_start): reproducible, graph == eager, top_p = 0 == greedy
    ids2 = torch.randint(0, cfg.vocab_size, (2, 14), generator=torch.Generator().manual_seed(4)).cuda()
    am = torch.ones(2, 14, dtype=torch.long, device="cuda")
    am[1, :5] = 0
    kw2 = dict(attention_mask=am, max_new_tokens=10, do_sample=True, temperature=0.6, top_k=50)

    def gen2(seed, **extra):
        return model.generate(ids2, generator=torch.Generator(device="cuda").manual_seed(seed), **{**kw2, **extra})

    b1 = gen2(3, top_p=0.9)
    assert b1.shape == (2, 24) and torch.equal(b1, gen2(3, top_p=0.9))
    assert torch.equal(gen2(3, top_p=0.9, use_graph=False), b1)
    assert torch.equal(gen2(3, top_p=0.0), model.generate(ids2, attention_mask=am, max_new_tokens=10))


def test_engine_top_p_cfg2_widths():
    """Llama-3.1-8B widths (d4096, 32q / 8kv heads, ffn 14336, V 128256), 2 layers: each step's token lies in the HF kept set."""
    cfg, model = _model("v0_5_8b", enc_layers=1, llm_layers=2)
    ids = torch.randint(0, 128000, (1, 16), generator=torch.Generator().manual_seed(6)).cuda()
    checked, cut, amb = _engine_steps_in_hf_kept_set(model, ids, 6, 0.6, 50, 0.9, 1.0)
    assert amb <= 1 and checked >= 5 and cut == checked, (checked, cut, amb)
