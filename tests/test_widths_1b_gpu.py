"""Per-op parity at the Llama-3.2-1B + Whisper-tiny widths of BASELINE config 1 (``preset("tiny_1b")``, DESIGN section 5).

The per-op suites run every LLM case at head_dim 128 and the encoder at Whisper-large's 1280 columns.  Config 1 runs other
template instances and shapes: head_dim 64 on the LLM path (``model.py`` fuses RoPE into the q|k|v epilogue only at 128, so
the prefill runs a plain ``ops.linear`` and ``uvx_rope`` at D = 64, then ``attn_wg_kernel<64>`` / ``attn_fwd_kernel<64>``
causal with GQA 32 / 8), the tied LM head at d = 2048, and the 384-wide encoder (LayerNorm with 48 vectors over 32 lanes, conv1
with K = 240 ending inside a 64-wide k-block, 6 heads).  This module calls the same kernels through the same helpers as the
128-wide suites (imported from them, with their bounds) at these widths:

* d 2048, 32 q / 8 kv heads of 64, ffn 8192, V 128256 tied to ``embed_tokens``, llama3 RoPE tables from
  ``ops.llama3_inv_freq(64, ...)``;
* Whisper-tiny: d 384, 6 heads of 64, ffn 1536, 80 mel bins; the projector 3072 -> 8192 (SwiGLU to 4096) -> 2048.

Sections: prefill attention, RoPE and the cache fill, decode (attention over the cache, RoPE + append, GEMV, LM head), long
contexts, the prefill GEMMs, the backward, the Whisper-tiny front end and encoder, and config 1 composed at full depth.

Bounds are the 128-wide suites' own (each helper's module docstring derives them).  Two of them involve the head dimension:

* attention vs the rounding-matched reference, ``MATCH_K`` * (ulp + 2^-11 sum_j p_j |v_j|): the 2^-11 term covers entries of P
  flipping to the neighbouring bf16 value because the kernel's score (a D-term tensor-core dot product) differs from torch's
  fp32 score by a few fp32 ulps.  At D = 64 the dot product has half the terms, so the same bound holds with more margin; the
  bound is not changed;
* the needle patterns of the long-context forms need a scaled log2 score gap > 160 (``NEEDLE_GAP``).  With the 128-wide needle
  value 4 the gap at D = 64 is about (16 * 64 - 5 * 32) / 8 * log2 e ~ 155, too small, so the needle value is 6 here
  (score 2304 against N(0, 48^2), gap ~ 370); ``needle_gap`` asserts it for every planted needle.

Worst values the tests print, measured over the whole module on an H100 80GB HBM3 at a 700 W power limit (wall time 117 s, about 25 s
of it the dispatch child process):

* attention rows vs fp32 softmax 3.6e-3 (bound ``ROW_REL`` 8e-3); vs the rounding-matched reference 2.22 of the unit
  (``MATCH_K`` 8); wgmma vs mma.sync 0 (bit for bit); decode / long-context rows vs fp32 2.7e-3 (3e-3), vs the rounding-matched
  walk 9.6e-4 (1e-3, growing above 1024 tiles);
* RoPE, conv stem, GEMV, LM head and GEMM per-element bounds at most 0.50 of the bound (the final bf16 rounding); LayerNorm
  at 384 columns 0.17 of its fp32 term; log-mel at 80 bins 2.1e-6 abs (2e-3);
* attention backward vs fp32 autograd 2.6e-3 (1e-2);
* config 1 at full depth vs the fp32 oracle: encoder 6.4e-3, projector 1.0e-2, embeds 1.0e-2, last-row logits 2.7e-2 (1.5e-2 /
  2e-2 / 2e-2 / 3e-2); decode steps vs the cacheless forward 2.3e-2 (3e-2).

Dispatch: every kernel or GEMM form a case names is asserted by ``test_dispatch`` (section 0), which profiles the same calls
at the same shapes in a child process and fails when a form is missing or another kernel runs."""
import math

import numpy as np
import pytest
import torch

import test_backward_gpu as BW
import test_decode_gpu as DG
import test_gemm_gpu as G
import test_long_context_gpu as LC
import test_prefill_gpu as P

pytestmark = pytest.mark.gpu
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64

D1B, HQ, HKV, HD, FFN, V = 2048, 32, 8, 64, 8192, 128256
ENC_D, ENC_H, ENC_FFN, MELS = 384, 6, 1536, 80
NEEDLE_64 = 6.0


@pytest.fixture(autouse=True)
def _gpu_state():
    """fp32 references in full fp32 (no TF32); buffers freed between tests."""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def model_1b():
    """The full-depth config-1 model (4 encoder layers, 16 Llama layers, V = 128256 tied) on seeded random weights."""
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    model = UltravoxModel(preset("tiny_1b"), device="cuda").init_random_(seed=42)
    yield model
    del model
    torch.cuda.empty_cache()


def tables_64():
    return P._llama3_tables(HD, "tiny_1b")


# ================================================================================================ 0. dispatch
# Every form a case of this module names, with the kernels it must run.  Inside this module's pytest process the profiler
# loses the kernel records of many windows (all of them, for whole stretches of the run), while a fresh Python process on the
# same machine records every window, before and after the same attention, 131 k-key and GEMM work.  So the calls are
# profiled in a child process of their own, on inputs of the cases' shapes, and every check fails hard: a window without
# the expected records is profiled again up to 3 times, then the test fails.
def _gemm_forms():
    """name -> exact set of ``uvx::`` kernels (``test_gemm_gpu.short`` names)."""
    f = {}
    # M = 20: the tokens on the wgmma N dimension (32-wide) with split-K; M = 201: 2 x 128-row tiles with split-K; M = 804:
    # tensor bound, the norm as its own pass; gate|up on the 128-row SwiGLU image: 1 x 128 tiles
    for M in (20, 201, 804):
        small = {20: [G.swap(20)], 201: [G.wg(2, 128)], 804: []}[M]
        f[f"1b qkv M={M}"] = small + [G.RED] if M < 804 else [G.wg(1, 128, True)]
        for layer in ("o", "down"):
            f[f"1b {layer} M={M}"] = small + [G.RED_NORM] if M < 804 else [G.wg(1, 128), G.NORM]
        f[f"1b gate_up M={M}"] = [G.wg(1, 128)]
    f["1b logits M=20"], f["1b logits M=201"] = [G.wg(1, 128)], [G.wg(2, 128)]
    # Whisper-tiny encoder: M = 50 one 128-row tile (fc2, K = 1536: split-K); M = 1500 / 3000 the staged epilogue, 64-wide
    # tiles for N = 384 at 1500
    for M in (50, 1500, 3000):
        for layer in ("qkv", "out", "fc1", "fc2"):
            if M == 50:
                f[f"tiny {layer} M={M}"] = [G.wg(1, 128)] + ([G.RED] if layer == "fc2" else [])
            else:
                f[f"tiny {layer} M={M}"] = [G.wg(1, 64 if (M == 1500 and layer in ("out", "fc2")) else 128, True)]
    return f


GEMM_FORMS = _gemm_forms()
WG64, FWD64 = "attn_wg_kernel<64, false, false, false>", "attn_fwd_kernel<64, false, false>"
# name -> the one attention kernel it runs (``test_long_context_gpu.assert_kernel``'s rule)
ATTN_FORMS = {"prefill S=201 B=4": WG64, "prefill S=20 B=4": WG64, "prefill on cache Sq=64 past=300": WG64,
              "eligibility cache Sq=16": WG64, "eligibility cache Sq=15": FWD64,
              "eligibility fused Sq=16": WG64, "eligibility fused Sq=15": FWD64,
              "decode B=3 S_max=4160": FWD64, "cache prefill Sq=7": FWD64, "cache prefill Sq=33": WG64,
              "decode S_max=131072": FWD64, "paged bf16": "attn_fwd_kernel<64, true, false>",
              "paged e4m3": "attn_fwd_kernel<64, true, true>", "encoder S=50": WG64, "encoder S=1500": WG64}
# name -> kernels (name prefix, template prefix) that must be among those it runs
OTHER_FORMS = {"layernorm 1500x384": ["layernorm_warp_kernel"],
               "attention bwd D=64": ["attn_bwd_dq_kernel<64,", "attn_bwd_dkv_kernel<64,"]}


def _dispatch_calls():
    """name -> zero-argument call on seeded inputs of the shapes the cases of this module use (run in the child process)."""
    from ultravox_b200 import ops
    calls = {}
    for M in (20, 201, 804):
        x, x8, r = P.rnd(M, D1B, seed=1), P.rnd(M, FFN, seed=2), P.rnd(M, D1B, seed=3)
        nw = P.rnd(D1B, scale=0.5, mean=1.0, seed=4)
        wq, wo, wd = P.rnd(3072, D1B, scale=0.02, seed=5), P.rnd(D1B, D1B, scale=0.02, seed=6), P.rnd(D1B, FFN, scale=0.02, seed=7)
        tw = ops.TiledWeight(P.rnd(2 * FFN, D1B, scale=0.02, seed=8), 128, swiglu=True)

        def norm_call(a, w, M=M, r=r, nw=nw):
            return lambda: ops.linear(a, w, residual=r.clone(), norm=(nw, 1e-5, torch.empty(M, D1B, dtype=BF, device="cuda")))
        calls[f"1b qkv M={M}"] = lambda x=x, w=wq: ops.linear(x, w)
        calls[f"1b o M={M}"] = norm_call(x, wo)
        calls[f"1b down M={M}"] = norm_call(x8, wd)
        calls[f"1b gate_up M={M}"] = lambda x=x, tw=tw: ops.linear_tiled(x, tw, act=ops.ACT_SWIGLU)
    wl = P.rnd(V, D1B, scale=0.02, seed=9)
    for M in (20, 201):
        calls[f"1b logits M={M}"] = lambda x=P.rnd(M, D1B, seed=10): ops.linear(x, wl, out_dtype=F32)
    for M in (50, 1500, 3000):
        for layer, N, K in (("qkv", 3 * ENC_D, ENC_D), ("out", ENC_D, ENC_D), ("fc1", ENC_FFN, ENC_D), ("fc2", ENC_D, ENC_FFN)):
            x, w, b = P.rnd(M, K, seed=11), P.rnd(N, K, scale=0.05, seed=12), P.rnd(N, seed=13)
            res = None if layer in ("qkv", "fc1") else P.rnd(M, N, seed=14)
            act = ops.ACT_GELU if layer == "fc1" else ops.ACT_NONE
            calls[f"tiny {layer} M={M}"] = lambda x=x, w=w, b=b, res=res, act=act: ops.linear(x, w, bias=b, act=act, residual=res)
    # attention
    c = P.AttnCase("fused", 4, 201, HQ, HKV, HD, causal=True, starts=[0, 1, 63, 64], seed=1)
    calls["prefill S=201 B=4"] = c.run
    c20 = P.AttnCase("fused", 4, 20, HQ, HKV, HD, causal=True, starts=[0, 1, 10, 19], seed=2)
    calls["prefill S=20 B=4"] = c20.run
    cc = P.AttnCase("cache", 3, 64, HQ, HKV, HD, causal=True, past=300, starts=[0, 64, 130], seed=3)
    calls["prefill on cache Sq=64 past=300"] = cc.run
    for form in ("cache", "fused"):
        c16, c15 = P.eligibility_cases(form, HD)
        calls[f"eligibility {form} Sq=16"], calls[f"eligibility {form} Sq=15"] = c16.run, c15.run
    qkv1, kc, vc = P.rnd(3, (HQ + 2 * HKV) * HD, seed=4), P.rnd(3, 4160, HKV, HD, seed=5), P.rnd(3, 4160, HKV, HD, seed=6)
    lens = torch.tensor([4160, 65, 1], dtype=torch.int32, device="cuda")
    calls["decode B=3 S_max=4160"] = lambda: DG.cache_attention(qkv1, kc, vc, HQ, 1, 4160, False, lens, None)
    for Sq in (7, 33):
        q = P.rnd(4 * Sq, (HQ + 2 * HKV) * HD, seed=Sq)
        k4, v4 = kc[:1].expand(4, -1, -1, -1).contiguous(), vc[:1].expand(4, -1, -1, -1).contiguous()
        calls[f"cache prefill Sq={Sq}"] = lambda q=q, k4=k4, v4=v4, Sq=Sq: DG.cache_attention(q, k4, v4, HQ, Sq, 137 + Sq, True)
    kl, vl = P.rnd(1, LC.SMAX, HKV, HD, seed=7), P.rnd(1, LC.SMAX, HKV, HD, seed=8)
    ql, ll = P.rnd(1, HQ * HD, seed=9), torch.tensor([LC.SMAX - 3], dtype=torch.int32, device="cuda")
    calls["decode S_max=131072"] = lambda: LC.decode(ql, kl, vl, HQ, ll)
    table = torch.arange(8, dtype=torch.int32, device="cuda").view(2, 4)
    pl = torch.tensor([256, 200], dtype=torch.int32, device="cuda")
    qp = P.rnd(2, HQ * HD, seed=10)
    pk, pv = P.rnd(8, LC.PAGE, HKV, HD, seed=11), P.rnd(8, LC.PAGE, HKV, HD, seed=12)
    pk8, pv8 = LC.quant(pk, 1.0), LC.quant(pv, 1.0)
    sc = torch.tensor([1.0, 1.0], dtype=F32, device="cuda")
    calls["paged bf16"] = lambda: ops.attention_paged(qp, pk, pv, torch.empty(2, HQ * HD, dtype=BF, device="cuda"), HQ, HD ** -0.5,
                                                      table, pl)
    calls["paged e4m3"] = lambda: ops.attention_paged(qp, pk8, pv8, torch.empty(2, HQ * HD, dtype=BF, device="cuda"), HQ,
                                                      HD ** -0.5, table, pl, kv_scale=sc)
    for S in (50, 1500):
        ce = P.AttnCase("enc", 2, S, ENC_H, ENC_H, 64, lens=[S, S // 2], seed=S)
        calls[f"encoder S={S}"] = ce.run
    xl, wln, bln = P.rnd(1500, ENC_D, seed=13), P.rnd(ENC_D, seed=14), P.rnd(ENC_D, seed=15)
    calls["layernorm 1500x384"] = lambda: ops.layernorm(xl, wln, bln, 1e-5)
    A = BW.Attn(B=2, S=201, Hq=HQ, Hkv=HKV, D=HD, causal=True, kv_len=[201, 150])
    qkvb, doutb = BW._inputs(A, 11)
    calls["attention bwd D=64"] = lambda: A.run(qkvb, doutb)
    return calls


def _dispatch_child():
    """Profile every call of ``_dispatch_calls`` (up to 3 windows while a window misses an expected kernel) and print
    {name: [kernel names]} as one JSON line."""
    import json
    want = {**{k: v for k, v in GEMM_FORMS.items()}, **{k: [v] for k, v in ATTN_FORMS.items()}, **OTHER_FORMS}
    out = {}
    for name, fn in _dispatch_calls().items():
        fn()
        for _ in range(3):
            names = LC.kernels_run(fn).splitlines()
            if all(any(w.split("<")[0] in n for n in names) for w in want[name]):
                break
        out[name] = names
    print("DISPATCH " + json.dumps(out))


@pytest.fixture(scope="module")
def dispatch():
    """{name: kernel names} from ``_dispatch_child`` in a process of its own."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", "import test_widths_1b_gpu as W; W._dispatch_child()"], cwd=here,
                       capture_output=True, text=True, timeout=600, env=dict(os.environ, PYTHONPATH=os.pathsep.join(
                           [here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")])))
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("DISPATCH ")]
    assert r.returncode == 0 and lines, (r.returncode, r.stdout[-2000:], r.stderr[-4000:])
    return json.loads(lines[-1][len("DISPATCH "):])


def _mangled(want):
    name, args = want[:-1].split("<")
    args = [a.strip() for a in args.split(",")]
    return f"{name}ILi{args[0]}E" + "".join("Lb1E" if a == "true" else "Lb0E" for a in args[1:]) + "E"


@pytest.mark.parametrize("name", list(GEMM_FORMS) + list(ATTN_FORMS) + list(OTHER_FORMS))
def test_dispatch(dispatch, name):
    """The call a case names runs exactly the kernels it names: GEMMs the exact set of ``uvx::`` kernels, attention the one
    ``attn_`` kernel (demangled or mangled name), LayerNorm / the backward at least the named kernels."""
    names = dispatch[name]
    if name in GEMM_FORMS:
        ran = sorted({G.short(n) for n in names if "uvx::" in n})
        assert ran == sorted(set(GEMM_FORMS[name])), (name, ran)
    elif name in ATTN_FORMS:
        want = ATTN_FORMS[name]
        attn = {n.split("(")[0] for n in names if "attn_" in n}
        assert len(attn) == 1 and any(want in a or _mangled(want) in a for a in attn), (name, want, names)
    else:
        for w in OTHER_FORMS[name]:
            base, _, arg = w.partition("<")
            assert any(w in n or (arg and f"{base}ILi{arg.rstrip(',')}E" in n) or (not arg and base in n) for n in names), (name, w, names)


# ================================================================================================ 1. prefill attention, D = 64
def _prefill_cases_1b():
    """``test_prefill_gpu``'s grid at 32 / 8 heads plus S = 20, the config-1 prompt."""
    cs = {}
    for S in (201, 640, 64, 65, 20):
        ok = [x for x in (0, 1, 63, 64, 65, 128, S - 1) if x < S]
        if len(ok) < 4:
            ok = [0, 1, S // 2, S - 1]
        cs[f"S{S}_B1_plain"] = dict(S=S, B=1, starts=None, lens=None)
        cs[f"S{S}_B1_start{ok[-2]}"] = dict(S=S, B=1, starts=[ok[-2]], lens=None)
        cs[f"S{S}_B1_start{min(63, S - 2)}_len{S - 1}"] = dict(S=S, B=1, starts=[min(63, S - 2)], lens=[S - 1])
        a, b_ = ok[:4], (ok[4:] + ok[:4])[:4]
        cs[f"S{S}_B4_starts{'-'.join(map(str, a))}"] = dict(S=S, B=4, starts=a, lens=None)
        lens = [min(S, max(s + 1, S - d)) for s, d in zip(b_, (3, 0, 1, S // 3))]
        cs[f"S{S}_B4_starts{'-'.join(map(str, b_))}_lens{'-'.join(map(str, lens))}"] = dict(S=S, B=4, starts=b_, lens=lens)
    return cs


PREFILL_CASES = _prefill_cases_1b()


@pytest.mark.parametrize("case", list(PREFILL_CASES))
def test_attention_prefill_d64(case):
    """The 1B prefill (causal GQA 32 / 8, head_dim 64) through ``ops.attention_fused_qkv`` with left padding and a right-side
    ``kv_len``: per row vs fp32, per element vs the rounding-matched reference, masks bit for bit, wgmma == mma.sync."""
    p = PREFILL_CASES[case]
    c = P.AttnCase("fused", p["B"], p["S"], HQ, HKV, HD, causal=True, lens=p["lens"], starts=p["starts"], seed=p["S"] + 7 * p["B"])
    P.check_attention(c, "prefill 1b " + case)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("past", [1, 63, 300, 4000])
@pytest.mark.parametrize("Sq", [64, 70, 201])
def test_attention_prefill_on_cache_d64(Sq, past, B):
    P.prefill_on_cache_case(Sq, past, B, HD, HQ, HKV)


@pytest.mark.parametrize("form", ["cache", "fused"])
def test_attention_eligibility_edge_d64(form):
    """Sq = 16 on ``attn_wg_kernel<64>``, Sq = 15 on ``attn_fwd_kernel<64>`` (``test_dispatch`` pins both on these cases): the
    same rows agree."""
    P.eligibility_edge_case(form, HD)


@pytest.mark.parametrize("form", ["fused", "cache"])
def test_attention_batch_and_head_isolation_d64(form):
    P.isolation_case(form, HQ, HKV, HD)


@pytest.mark.parametrize("kernel", ["wgmma", "mma.sync"])
def test_attention_empty_rows_and_lse_d64(kernel):
    P.empty_rows_case(kernel, HD)


# ================================================================================================ 2. RoPE and the cache fill, D = 64
@pytest.mark.parametrize("B", [1, 3])
def test_rope_offsets_and_positions_d64(B):
    """``ops.rope_`` at head_dim 64 with the 1B tables: pos_offset up to 131071 - S and the left-padded ``positions``."""
    P.rope_case(HQ, HKV, HD, B, tables_64(), "1b")


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("past", [0, 300])
def test_kv_write_fills_the_cache_d64(past, B):
    P.kv_write_case(HQ, HKV, HD, past, B, tables_64())


# ================================================================================================ 3. decode, D = 64
@pytest.mark.parametrize("left_pad", [False, True])
@pytest.mark.parametrize("smax", [210, 4160])
@pytest.mark.parametrize("B", [1, 3, 8, 32])
def test_decode_attention_over_cache_d64(B, smax, left_pad):
    DG.decode_attention_case(HQ, HKV, HD, B, smax, left_pad, "1b")


@pytest.mark.parametrize("left_pad", [False, True])
@pytest.mark.parametrize("Sq", [2, 7, 15, 16, 33])
def test_prefill_attention_on_cache_short_d64(Sq, left_pad):
    DG.prefill_on_cache_case(HQ, HKV, HD, Sq, left_pad, "1b")


def test_rope_kv_append_long_positions_d64(ops):
    """Plain form through ``test_decode_gpu``'s check; then the map form (one row not appended) and the e4m3 map form (power of
    two scales, so the quantizer is exact division) bit for bit against it."""
    DG.rope_kv_append_case(HQ, HKV, HD, "tiny_1b", "1b")
    cos, sin = tables_64()
    B, smax = 8, 210
    rope_pos = torch.tensor([0, 1, 8191, 8192, 65535, 100003, 131070, 131071], dtype=torch.int32, device="cuda")
    slot = torch.tensor([3, 0, 77, 209, 5, 150, 1, 9], dtype=torch.int32, device="cuda")
    qkv0 = P.rnd(B, (HQ + 2 * HKV) * HD, scale=2.0, seed=11)
    kc, vc = torch.full((B, smax, HKV, HD), -3.5, dtype=BF, device="cuda"), torch.full((B, smax, HKV, HD), -3.5, dtype=BF, device="cuda")
    qkv = qkv0.clone()
    ops.rope_kv_append_(qkv, HQ, HKV, HD, cos, sin, rope_pos, kc, vc, slot)
    rows = torch.arange(B, dtype=torch.int32, device="cuda")
    cache_row = rows.clone()
    cache_row[5] = -1
    q2 = qkv0.clone()
    k2, v2 = torch.full_like(kc, -3.5), torch.full_like(vc, -3.5)
    ops.rope_kv_append_map_(q2, HQ, HKV, HD, cos, sin, rope_pos, k2, v2, cache_row, slot)
    assert torch.equal(q2, qkv), "map form: rotated rows differ from the plain form"
    keep = cache_row >= 0
    r, s_ = rows[keep].long(), slot[keep].long()
    assert torch.equal(k2[r, s_], kc[r, s_]) and torch.equal(v2[r, s_], vc[r, s_]), "map form: appended rows differ"
    assert bool((k2[5] == -3.5).all()) and bool((v2[5] == -3.5).all()), "map form: row with cache_row -1 was appended"
    for sk, sv in ((1.0, 1.0), (2.0 ** -3, 2.0 ** 2)):
        q3 = qkv0.clone()
        k8 = torch.full((B, smax, HKV, HD), LC.NAN_BYTE, dtype=torch.uint8, device="cuda").view(LC.E4M3)
        v8 = k8.clone()
        scale = torch.tensor([sk, sv], dtype=F32, device="cuda")
        ops.rope_kv_append_map_(q3, HQ, HKV, HD, cos, sin, rope_pos, k8, v8, cache_row, slot, kv_scale=scale)
        assert torch.equal(q3, qkv)
        assert torch.equal(k8[r, s_].view(torch.uint8), LC.quant(kc[r, s_], sk).view(torch.uint8)), ("fp8 k", sk)
        assert torch.equal(v8[r, s_].view(torch.uint8), LC.quant(vc[r, s_], sv).view(torch.uint8)), ("fp8 v", sv)
        assert bool((k8[5].view(torch.uint8) == LC.NAN_BYTE).all()), "fp8 map form: row with cache_row -1 was appended"


GEMV_1B = {"qkv": (3072, 2048), "o": (2048, 2048), "gate_up": (16384, 2048), "down": (2048, 8192)}


@pytest.mark.parametrize("shape", list(GEMV_1B))
def test_gemv_and_decode_gemm_1b(shape):
    DG.gemv_case(*GEMV_1B[shape], "1b_" + shape)


@pytest.mark.parametrize("case", [("norm", 3072, 2048, (1, 5, 8)), ("norm", 16384, 2048, (2, 8)),
                                  # down_proj: B * 2K * 2 bytes = 192 KiB at B = 6 (fused), 224 KiB at B = 7 (unfused)
                                  ("swiglu", 2048, 8192, (1, 6, 7, 8))])
def test_gemv_fused_prologues_1b(case):
    DG.gemv_prologue_case(case)


def test_lm_head_tied_storage(ops, model_1b):
    """``ops.lm_head`` at d = 2048 over the model's own tied storage (``lm_head.weight`` is ``embed_tokens.weight``), B up to
    32 (slabs of 8 past 8), dense and strided hidden rows: every logit within gamma(8 ceil(d/256) + 5) sum|h w| of fp64;
    argmax == torch.argmax."""
    lm = model_1b.language_model
    w = lm.lm_head.weight
    assert w.data_ptr() == lm.model.embed_tokens.weight.data_ptr() and tuple(w.shape) == (V, D1B)
    hid = P.rnd(32, 5, D1B, seed=2048)
    ref, mag = DG.matvec_f64(hid[:, -1], w)
    bound = DG.gamma(8 * math.ceil(D1B / 256) + 5) * mag
    worst = 0.0
    for B in (1, 2, 7, 8, 9, 12, 32):
        for h in (hid[:B, -1].contiguous(), hid[:B, -1, :]):
            lg = ops.lm_head(h, w)
            worst = max(worst, P.worst_ratio(lg, ref[:B], bound[:B]))
            DG.assert_within(lg, ref[:B], bound[:B], f"lm_head 1b B={B} row stride {h.stride(0)}")
            assert torch.equal(ops.argmax(lg), lg.argmax(-1)), B
    print(f"lm_head d=2048 tied: max err / bound {worst:.3f}")


# ================================================================================================ 4. long context, D = 64
@pytest.mark.parametrize("smax,B", [(32768, 3), (LC.SMAX, 1), (LC.SMAX, 3)])
def test_decode_long_cache_d64(smax, B):
    LC.decode_long_case(HQ, smax, B, "1b", D=HD, needle=NEEDLE_64, check_dispatch=False)


@pytest.mark.parametrize("kind", ["bf16", "fp8-0", "fp8-1", "fp8-2"])
def test_paged_decode_long_table_d64(kind):
    LC.paged_long_case(kind, D=HD, needle=NEEDLE_64, check_dispatch=False)


# ================================================================================================ 5. prefill GEMMs at the 1B shapes
@pytest.mark.parametrize("regime", G.REGIMES)
@pytest.mark.parametrize("M", [20, 201, 804])
@pytest.mark.parametrize("layer", ["qkv", "o", "gate_up", "down"])
def test_llama_1b_prefill_gemms(request, ops, regime, M, layer):
    """The four projections as ``llama_hidden`` calls them at head_dim 64: q|k|v 3072 x 2048 plain (no RoPE epilogue), o 2048 x
    2048 and down 2048 x 8192 with the residual in place and the fused RMSNorm, gate|up 16384 x 2048 on the 128-row SwiGLU
    image with silu(gate) * up in the epilogue."""
    gen = G.Gen(regime, seed=M + 3 * len(layer))
    if layer in ("o", "down"):
        K = D1B if layer == "o" else FFN

        def call(x, w, r, out, nw, xn):
            ops.linear(x, w, residual=r, out=out, norm=(nw, 1e-5, xn))
        G.residual_norm_case(request, ops, gen, M, D1B, K, call, None, f"1b {layer} M={M}")
        print(f"1b {layer} M={M} {regime}: max err / bound {G.RATIOS.get(request.node.name, 0.0):.3f}")
        return
    x, au = gen.mat(M, D1B)
    if layer == "qkv":
        w, wu = gen.mat((HQ + 2 * HKV) * HD, D1B, scale=0.02)
        acc, mag = G.mm_ref(x, w, au, wu)
        (y,) = G.run(ops, lambda: (ops.linear(x, w),), None)
        G.check_plain(request, y, acc, mag, D1B, f"1b qkv M={M}")
    else:
        w, wu = gen.mat(2 * FFN, D1B, scale=0.02)
        acc, mag = G.mm_ref(x, w, au, wu)
        tw = ops.TiledWeight(w, 128, swiglu=True)
        (y,) = G.run(ops, lambda: (ops.linear_tiled(x, tw, act=ops.ACT_SWIGLU),), None)
        G.check_swiglu(request, y, acc, mag, D1B, f"1b gate|up M={M}")
    print(f"1b {layer} M={M} {regime}: max err / bound {G.RATIOS.get(request.node.name, 0.0):.3f}")


@pytest.mark.parametrize("regime", G.REGIMES)
@pytest.mark.parametrize("M", [20, 201])
def test_lm_head_logits_fp32_1b(request, ops, regime, M):
    """All-row fp32 logits of the config-1 prompt (M = 20) and of a 201-row prefill against the V = 128256 head at K = 2048."""
    gen = G.Gen(regime, seed=2048 + M)
    x, au = gen.mat(M, D1B)
    w, wu = gen.mat(V, D1B, scale=0.02)
    acc, mag = G.mm_ref(x, w, au, wu)
    (y,) = G.run(ops, lambda: (ops.linear(x, w, out_dtype=F32),), None)
    G.check_plain(request, y, acc, mag, D1B, f"1b logits M={M}")
    print(f"1b logits M={M} {regime}: max err / bound {G.RATIOS.get(request.node.name, 0.0):.3f}")


# ================================================================================================ 6. backward, D = 64 causal GQA
BWD_CASES = {
    "llm1b_4x201": dict(B=4, S=201, Hq=HQ, Hkv=HKV, D=HD, causal=True),
    "llm1b_201_kv150": dict(B=2, S=201, Hq=HQ, Hkv=HKV, D=HD, causal=True, kv_len=[201, 150]),
    "llm1b_640_kv333": dict(B=2, S=640, Hq=HQ, Hkv=HKV, D=HD, causal=True, kv_len=[640, 333]),
}


@pytest.mark.parametrize("case", list(BWD_CASES))
def test_attention_bwd_d64_vs_fp32(case):
    BW.bwd_vs_fp32_case(BW.Attn(**BWD_CASES[case]), case)


@pytest.mark.parametrize("case", list(BWD_CASES))
def test_attention_bwd_d64_masks_exact(case):
    BW.bwd_masks_case(BW.Attn(**BWD_CASES[case]), case)


@pytest.mark.parametrize("pos_offset", [0, 37])
def test_rope_bwd_llama3_d64(pos_offset):
    BW.rope_bwd_case(pos_offset, HQ, HKV, HD, "tiny_1b")


@pytest.mark.parametrize("rows,cols", [(201, D1B), (402, D1B)])
def test_rmsnorm_bwd_1b(rows, cols):
    BW.rmsnorm_bwd_case(rows, cols, 1e-5)


def test_swiglu_bwd_1b():
    BW.swiglu_bwd_case(201, FFN, True)


# ================================================================================================ 7. Whisper-tiny front end and encoder
def test_logmel_80_bins():
    """80 mel bins: silence alone and beside noise, a sub-window clip, a full-scale square wave, DC, and a 1 s clip beside a 30 s
    one (its frames inside the clip equal the clip alone; the frames past its end are one constant)."""
    from ultravox_b200 import ops
    rng = np.random.default_rng(80)
    t = np.arange(16000)
    square = np.where((t // 50) % 2 == 0, 1.0, -1.0).astype(np.float32)
    noise = rng.standard_normal(16000).astype(np.float32)
    for waves in ([np.zeros(16000, np.float32)], [noise, np.zeros(9000, np.float32)]):
        got, ref, padded = P._logmel_check(waves, MELS)
        assert np.all(ref[-1] == -1.5) and np.abs(got[-1] + 1.5).max() <= 1e-6
        assert bool((ops.logmel(torch.from_numpy(padded).cuda(), MELS, want_f32=False, want_tm=True)[-1, 1:-1] == -1.5).all())
    P._logmel_check([noise, rng.standard_normal(300).astype(np.float32)], MELS)
    P._logmel_check([square], MELS)
    P._logmel_check([np.ones(16000, np.float32)], MELS)
    one_s, long_ = (0.3 * rng.standard_normal(16000)).astype(np.float32), rng.standard_normal(480000).astype(np.float32)
    both, ref, _ = P._logmel_check([long_, one_s], MELS)
    alone, _, _ = P._logmel_check([one_s], MELS)
    assert both.shape[2] == 3000 and alone.shape[2] == 100
    d = np.abs(both[1][:, :99] - alone[0][:, :99]).max()       # frame t reads samples up to 160 t + 200 <= 16000
    print(f"logmel 80: 1 s clip in a 30 s batch vs alone: max abs {d:.3e}")
    assert d < 2e-3, d
    tail = both[1][:, 102:]
    assert np.all(tail == tail[0, 0]), "the frames past the clip's end are one constant"


@pytest.mark.parametrize("T", [100, 99, 3000, 2999])
@pytest.mark.parametrize("layer", ["conv1", "conv2"])
def test_conv_stem_tiny(layer, T):
    """conv1 80 -> 384 (implicit-GEMM K = 240, ending inside a 64-wide k-block, into the guard-padded buffer) and conv2 384 ->
    384 stride 2 with the positional embedding, per element, the frames where the padding enters named."""
    if layer == "conv1":
        P.conv_case(MELS, ENC_D, 1, T, 2, False, f"tiny conv1_T{T}")
    else:
        P.conv_case(ENC_D, ENC_D, 2, T, 2, True, f"tiny conv2_T{T}")


ENC_TINY = {"S50_B1": dict(S=50, B=1, lens=None, block=0), "S50_B3_lens": dict(S=50, B=3, lens=[50, 1, 33], block=0),
            "S1500_B1": dict(S=1500, B=1, lens=None, block=0), "S1500_B3_lens": dict(S=1500, B=3, lens=[1500, 563, 0], block=0),
            "S1500_B2_stream100": dict(S=1500, B=2, lens=[1500, 250], block=100),
            "S50_B2_stream25": dict(S=50, B=2, lens=[50, 37], block=25)}


@pytest.mark.parametrize("case", list(ENC_TINY))
def test_attention_encoder_tiny(case):
    """Whisper-tiny's encoder attention (6 heads of 64, non-causal) at S = 50 (1 s) and 1500 (30 s), with key lengths and the
    block-causal streaming mask."""
    p = ENC_TINY[case]
    c = P.AttnCase("enc", p["B"], p["S"], ENC_H, ENC_H, 64, lens=p["lens"], block=p["block"], seed=p["S"] + p["B"] + p["block"])
    P.check_attention(c, "encoder tiny " + case)


@pytest.mark.parametrize("regime", G.REGIMES)
@pytest.mark.parametrize("M", [50, 1500, 3000])
@pytest.mark.parametrize("layer,N,K", [("qkv", 3 * ENC_D, ENC_D), ("out", ENC_D, ENC_D), ("fc1", ENC_FFN, ENC_D),
                                       ("fc2", ENC_D, ENC_FFN)])
def test_whisper_tiny_encoder_gemms(request, ops, regime, M, layer, N, K):
    """The encoder linears at K = 384 (six k-blocks) and 1536: q|k|v + bias, out / fc2 + bias + residual, fc1 + bias + GELU."""
    gen = G.Gen(regime, seed=N + K + M)
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.05)
    b = gen.bias(N, wu)
    acc, mag = G.mm_ref(x, w, au, wu)
    if layer in ("qkv", "fc1"):
        act = ops.ACT_GELU if layer == "fc1" else ops.ACT_NONE
        (y,) = G.run(ops, lambda: (ops.linear(x, w, bias=b, act=act),), None)
        G.check_plain(request, y, acc, mag, K, f"tiny {layer}", bias=b, gelu=layer == "fc1")
    else:
        r = gen.res(M, N, au, wu)
        (y,) = G.run(ops, lambda: (ops.linear(x, w, bias=b, residual=r),), None)
        G.check_plain(request, y, acc, mag, K, f"tiny {layer}", bias=b, res=r)
    print(f"tiny {layer} M={M} {regime}: max err / bound {G.RATIOS.get(request.node.name, 0.0):.3f}")


@pytest.mark.parametrize("rows", [50, 1500, 3000])
def test_layernorm_384(rows):
    """``layernorm_warp_kernel`` at 384 columns (48 vectors over 32 lanes: lanes hold 2 or 1), dense, strided and with rows of
    mean 30."""
    P.layernorm_case(rows, ENC_D)


@pytest.mark.parametrize("M", [7, 188])
def test_projector_tiny(ops, M):
    """StackAudioFrames(8) + ln_pre at C = 384 (T = 50 -> 7 rows, the last one holding 2 frames and 6 zero frames), linear_1
    3072 -> 8192, SwiGLU (value first) to 4096, ln_mid at 4096, linear_2 4096 -> 2048: each stage against fp64 of the
    stage's own bf16 input."""
    k, C = 8, ENC_D
    T = 8 * M - 6
    enc, w_pre = P.rnd(1, T, C, seed=M), P.rnd(k * C, scale=0.3, mean=1.0, seed=2)
    st = torch.nn.functional.pad(enc.to(F64), (0, 0, 0, M * k - T)).reshape(1, M, k * C)
    ref, _, xn = P.rmsnorm_hf(st, w_pre, 1e-6)
    y = ops.stack_rmsnorm(enc, w_pre, k, 1e-6)
    assert y.shape == ref.shape
    P.assert_two_roundings(y, ref, xn, w_pre.to(F64)[None, None].expand_as(xn), f"tiny stack_rmsnorm M={M}")
    assert int(torch.count_nonzero(y[0, -1, 2 * C:])) == 0, "the six zero frames of the last stacked row"
    x = y.view(M, k * C)
    for name, N, K, xin in (("linear_1", 2 * 4096, k * C, x), ("linear_2", D1B, 4096, None)):
        if xin is None:
            h = P.rnd(M, 2 * 4096, scale=2.0, seed=M + 5)
            a, g = h[:, :4096].to(F64), h[:, 4096:].to(F64)
            act = g * torch.sigmoid(g)
            sref = (act.to(BF).to(F64) * a).to(BF)
            sw = ops.swiglu(h, gate_first=False)
            P.assert_two_roundings(sw, sref, act, a, f"tiny projector swiglu M={M}")
            w_mid = P.rnd(4096, scale=0.3, mean=1.0, seed=7)
            mref, _, mxn = P.rmsnorm_hf(sw.to(F64), w_mid, 1e-6)
            xin = ops.rmsnorm(sw, w_mid, 1e-6)
            P.assert_two_roundings(xin, mref, mxn, w_mid.to(F64)[None].expand_as(mxn), f"tiny ln_mid M={M}")
        w = P.rnd(N, K, scale=0.02, seed=N + K)
        got = ops.linear(xin, w)
        ref64 = xin.to(F64) @ w.to(F64).T
        mag = xin.to(F64).abs() @ w.to(F64).abs().T
        bound = G.bf16_ulp(ref64) + G.gamma_p(4 * math.ceil(K / 16) + G.S_MAX + 3) * mag
        r = P.worst_ratio(got, ref64, bound)
        print(f"tiny projector {name} M={M}: max err / bound {r:.3f}")
        P.assert_within(got, ref64, bound, f"tiny projector {name} M={M}")


# ================================================================================================ 8. config 1 composed
def test_cfg1_every_stage_vs_oracle(model_1b):
    """The full-depth config-1 model on a 1 s clip (20 prompt rows, 7 audio rows) against the fp32 oracle stage by stage: mel,
    encoder, projector, spliced rows bit for bit, last-row logits (SURVEY section 7's bounds, as the cfg2 width test)."""
    from oracle import logmel as ol, model as om
    from test_cfg_widths_gpu import prompt, rel
    from ultravox_b200 import ops
    model = model_1b
    cfg = model.config
    sd, sh = om.state_dict_fp32(model), om.shapes_from_config(cfg)
    padded, batch = prompt(cfg, [16000])
    assert batch["input_ids"].shape == (1, 20) and batch["audio_token_len"].tolist() == [7]
    mel_ref = torch.from_numpy(ol.log_mel(padded, MELS))
    mel = ops.logmel(torch.from_numpy(padded).cuda(), MELS)
    assert tuple(mel.shape) == (1, MELS, 100) and float((mel.cpu() - mel_ref).abs().max()) < 2e-3
    st = {}
    ref_logits, _ = om.forward(sd, sh, batch["input_ids"], mel.cpu().to(BF).float(), batch["audio_token_start_idx"],
                               batch["audio_lens"], batch["audio_token_len"], batch["audio_batch_size"], last_only=True, stages=st)
    enc = model.encode_audio(ops.mel_to_timemajor(mel), batch["audio_lens"])
    assert tuple(enc.shape) == (1, 50, ENC_D)
    r_enc = rel(enc, st["encoder"])
    aud = model.project_audio(enc)
    assert tuple(aud.shape) == (1, 7, D1B)
    r_proj = rel(aud, st["projector"])
    emb = model._prepare_audio_embeds(batch["input_ids"].cuda(), mel, batch["audio_token_start_idx"], batch["audio_lens"],
                                      batch["audio_token_len"], batch["audio_batch_size"])
    table = model.language_model.model.embed_tokens.weight
    ids = batch["input_ids"][0].cuda()
    assert torch.equal(emb[0, 8:15], aud[0, :7])
    assert torch.equal(emb[0, :8], table[ids[:8]]) and torch.equal(emb[0, 15:], table[ids[15:]])
    r_emb = rel(emb, st["inputs_embeds"])
    out = model(audio_values=mel, logits_to_keep=1, **{k: v.cuda() for k, v in batch.items()})
    got = out.logits.view(1, 1, -1).cpu()
    r_log = rel(got, ref_logits)
    print(f"cfg1 full depth: encoder {r_enc:.3e} projector {r_proj:.3e} embeds {r_emb:.3e} last-row logits {r_log:.3e}")
    assert r_enc < 1.5e-2 and r_proj < 2e-2 and r_emb < 2e-2 and r_log < 3e-2
    assert int(ref_logits.view(-1).argmax()) in got.view(-1).topk(5).indices.tolist()
    # 8 greedy tokens against the oracle re-forwarding each prefix, teacher-forced with the CUDA tokens
    n_new = 8
    kw = {k: v.cuda() for k, v in batch.items()}
    seq = model.generate(audio_values=mel, max_new_tokens=n_new, **kw)
    S = batch["input_ids"].shape[1]
    assert seq.shape == (1, S + n_new)
    cur = st["inputs_embeds"]
    table32 = sd["language_model.model.embed_tokens.weight"]
    for t in range(n_new):
        ref = om.llama_forward(sd, sh, cur, last_only=True).view(-1)
        tok = int(seq[0, S + t])
        assert tok in ref.topk(5).indices.tolist(), t
        assert float(ref.max() - ref[tok]) < 3e-2 * float(ref.abs().max()), t
        cur = torch.cat([cur, table32[tok][None, None]], dim=1)


@pytest.mark.parametrize("pads", [[9], [0, 17, 70]])
def test_cfg1_decode_graph_matches_eager(model_1b, pads):
    """``DecodeEngine`` on the full-depth 1B model with left-padded prompts (B = 1: the matrix-vector step, B = 3: the
    tensor-core GEMM step): 6 steps with and without the CUDA graph give the same tokens and logits bit for bit, and each step's
    logits are within rel 3e-2 of the cacheless forward over the same sequence.  ``test_decode_gpu``'s 1e-2 is for one layer;
    through 16 layers the two bf16 paths (matrix-vector / decode-form GEMMs against prefill GEMMs) each drift from exact math by
    what the full-depth logits bound of SURVEY section 7 allows (3e-2; the prefill measured 2.7e-2 against the fp32 oracle)."""
    model = model_1b
    B, S, n = len(pads), 80, 6
    g = torch.Generator().manual_seed(17)
    ids = torch.randint(0, V, (B, S), generator=g).cuda()
    am = torch.ones(B, S, dtype=torch.int64, device="cuda")
    for b, p in enumerate(pads):
        am[b, :p] = 0
        ids[b, :p] = 0
    toks_e, lg_e = DG._engine_run(model, ids, am, n, use_graph=False)
    toks_g, lg_g = DG._engine_run(model, ids, am, n, use_graph=True)
    assert torch.equal(toks_e, toks_g)
    for t in range(n):
        assert torch.equal(lg_e[t], lg_g[t]), ("graph != eager", t)
    worst = 0.0
    for t in range(n):
        seq = torch.cat([ids, toks_e[:, :t + 1]], 1)
        am_t = torch.cat([am, torch.ones(B, t + 1, dtype=am.dtype, device="cuda")], 1)
        pos = (am_t.cumsum(-1) - 1).clamp_min(0)
        ref = model(seq, attention_mask=am_t, position_ids=pos, logits_to_keep=1).logits.view(B, -1)
        for b in range(B):
            e = DG.rel(lg_e[t][b], ref[b])
            worst = max(worst, e)
            assert e < 3e-2, (pads, t, b, e)
    print(f"cfg1 decode pads={pads}: max rel vs cacheless forward {worst:.3e}")


def test_cfg1_lm_head_is_embed_storage(model_1b):
    """``lm_head.weight`` shares ``embed_tokens``' storage after ``init_random_``, after ``load_state_dict`` of a checkpoint
    without ``lm_head.weight`` (new values arrive in both) and after ``tie_weights()``."""
    lm = model_1b.language_model

    def tied():
        return lm.lm_head.weight.data_ptr() == lm.model.embed_tokens.weight.data_ptr()
    assert tied(), "after init_random_"
    sd = {k: v for k, v in model_1b.state_dict().items() if k != "language_model.lm_head.weight"}
    key = "language_model.model.embed_tokens.weight"
    original = sd[key].clone()
    new = original.clone()
    new[:4] = 0.5
    try:
        model_1b.load_state_dict(dict(sd, **{key: new}))
        assert tied(), "after load_state_dict without lm_head.weight"
        assert bool((lm.lm_head.weight[:4] == 0.5).all()) and torch.equal(lm.lm_head.weight, new)
        model_1b.tie_weights()
        assert tied(), "after tie_weights()"
    finally:                                     # the module's other tests share this model: give it its weights back
        model_1b.load_state_dict(dict(sd, **{key: original}))
    assert tied() and torch.equal(lm.lm_head.weight, original)
