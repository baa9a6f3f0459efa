"""Per-op parity of the decode-step kernels at the widths, batch sizes and cache lengths generation runs (DESIGN a13).

``DecodeEngine._step`` replays one CUDA graph over a handful of kernels; each is called here through ``ops`` on seeded bf16
inputs and compared with plain fp32 / fp64 math of the same operation, at the Llama-3.1-8B (d 4096, 32 / 8 heads of 128,
ffn 14336, V 128256) and 70B (d 8192, 64 / 8 heads, ffn 28672) widths:

* attention over the static KV cache (``attn_fwd_kernel``): one query per stream over S_max keys with per-row ``kv_len`` and
  left-padding ``kv_start``, and the prefill-on-a-cache form (2 <= Sq <= 33, causal shift > 0) on both attention kernels -
  against fp32 softmax, against a reference that copies the kernel's roundings, and with bit-level mask checks;
* the matrix-vector linears (``gemv_kernel``) with their RMSNorm / SwiGLU prologues and shared-memory fallbacks, and the decode
  form of the tensor-core GEMM that runs from two streams on;
* the LM head at V = 128256 (slab loop for B > 8, strided hidden rows) and greedy argmax (ties, unaligned rows, all -inf rows);
* RoPE + KV-cache append at positions up to 131071 with cache slots that differ from the RoPE positions;
* one decode step composed at 8B widths: graph == eager, and cache decode against the cacheless forward.

Bounds: ``rel`` is a Frobenius-norm relative error; "ulp" is the spacing of bf16 at the reference value; u = 2^-24.  The
matrix-vector bounds follow from the kernels' fp32 summation order (n sequential roundings): |got - exact| <= n u / (1 - n u)
* sum |x w|."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
U32 = 2.0 ** -24

W8B = dict(d=4096, Hq=32, Hkv=8, ffn=14336)
W70B = dict(d=8192, Hq=64, Hkv=8, ffn=28672)
HD = 128
V_LLM = 128256


@pytest.fixture(autouse=True, scope="module")
def _no_tf32():
    """The fp32 references run on the GPU: keep their matmuls in full fp32."""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def rnd(*shape, scale=1.0, seed=0):
    """Seeded bf16 normal values generated on the GPU (the 70B weights are 0.5 G elements)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF)


def bf16_ulp(ref: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 (8 significant bits) at |ref| (0 at ref == 0)."""
    _, e = torch.frexp(ref)
    ulp = torch.ldexp(torch.ones_like(ref), (e - 8).to(torch.int32))
    return torch.where(ref == 0, torch.zeros_like(ulp), ulp)


def assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError(f"{what}: {int(bad.sum())} entries out of bound; first at flat {i}: got "
                             f"{float(got.reshape(-1)[i])!r} ref {float(ref.reshape(-1)[i])!r} bound {float(bound.reshape(-1)[i])!r}")


def gamma(n):
    return n * U32 / (1 - n * U32)


def matvec_f64(x, w, r=None, chunk=8192):
    """x [B, K] @ w[N, K].T in fp64 (+ r) and sum_k |x w| (+ |r|), over chunks of w's rows."""
    xd = x.to(F64)
    xa = xd.abs()
    ref, mag = [], []
    for n0 in range(0, w.shape[0], chunk):
        wd = w[n0:n0 + chunk].to(F64)
        ref.append(xd @ wd.T)
        mag.append(xa @ wd.abs().T)
    ref, mag = torch.cat(ref, 1), torch.cat(mag, 1)
    if r is not None:
        ref, mag = ref + r.to(F64), mag + r.to(F64).abs()
    return ref, mag


# ================================================================================================ 1. attention over the KV cache
def cache_attention(qkv, kc, vc, Hq, Sq, Skv, causal, lens=None, start=None):
    """The engine's call (engine.py ``_step``; model.py ``llama_hidden`` with a cache): q from the fused q|k|v rows [B*Sq, W],
    k / v from the caches [B, S_max, Hkv, D], output [B*Sq, Hq*D]."""
    from ultravox_b200 import ops
    B, smax, Hkv, D = kc.shape
    rs, cs = qkv.stride(0), smax * Hkv * D
    out = torch.empty(B * Sq, Hq * D, dtype=BF, device="cuda")
    return ops.attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), out, B, Hq, Hkv, Sq, Skv, D,
                         (rs, Sq * rs, Hkv * D, cs, Hkv * D, cs, Hq * D, Sq * Hq * D), D ** -0.5, causal, lens, 0, start)


def attention_refs(qkv, kc, vc, Hq, Sq, Skv, causal, lens, start):
    """(fp32 softmax(q k^T scale) v, rounding-matched reference) over the keys in [start, min(Skv, lens)), causal with shift
    Skv - Sq.  The matched one walks the kernel's 64-key tiles with a running max, rounds P to bf16 before P.V, sums l in fp32
    on the unrounded P and rounds the output once (tiles wholly masked for a row leave its state unchanged, so walking every
    tile from 0 is the kernel's walk from floor(kv_start / 64) * 64)."""
    B, smax, Hkv, D = kc.shape
    G = Hq // Hkv
    q = qkv.view(B, Sq, Hq + 2 * Hkv, D)[:, :, :Hq].float().reshape(B, Sq, Hkv, G, D).permute(0, 2, 3, 1, 4)   # [B, Hkv, G, Sq, D]
    k = kc[:, :Skv].float().permute(0, 2, 1, 3)[:, :, None]                                                   # [B, Hkv, 1, Skv, D]
    v = vc[:, :Skv].float().permute(0, 2, 1, 3)[:, :, None]
    j = torch.arange(Skv, device="cuda")
    end = torch.full((B,), Skv, device="cuda") if lens is None else lens.clamp(max=Skv)
    beg = torch.zeros(B, dtype=torch.int32, device="cuda") if start is None else start
    ok = (j[None] >= beg[:, None]) & (j[None] < end[:, None])                                                 # [B, Skv]
    ok = ok[:, None, None, None, :].expand(B, 1, 1, Sq, Skv)
    if causal:
        i = torch.arange(Sq, device="cuda")[:, None]
        ok = ok & (j[None] <= i + (Skv - Sq))
    s = q @ k.transpose(-1, -2)                                                                               # unscaled, fp32
    s = s.masked_fill(~ok, float("-inf"))
    scale = torch.tensor(D ** -0.5, dtype=torch.float32)
    ref = (torch.softmax(s * scale, -1).nan_to_num(0.0) @ v)
    sl2 = float(scale * torch.tensor(1.4426950408889634, dtype=torch.float32))
    m = torch.full(s.shape[:-1], float("-inf"), device="cuda")
    l = torch.zeros_like(m)
    o = torch.zeros(*s.shape[:-1], D, device="cuda")
    for t0 in range(0, Skv, 64):
        st = s[..., t0:t0 + 64]
        m_new = torch.maximum(m, st.amax(-1))
        mref = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
        corr = torch.exp2((m - mref) * sl2)
        m = m_new
        p = torch.exp2((st - mref[..., None]) * sl2)
        l = l * corr + p.sum(-1)
        o = o * corr[..., None] + p.to(BF).float() @ v[..., t0:t0 + 64, :]
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    matched = (o * inv[..., None]).to(BF)

    def flat(t):
        return t.permute(0, 3, 1, 2, 4).reshape(B * Sq, Hq * D)
    return flat(ref), flat(matched)


def poison_outside(kc, vc, start, end):
    """Copies of the caches with every row outside [start_b, end_b) set to NaN / +Inf / -Inf."""
    kp, vp = kc.clone(), vc.clone()
    smax = kc.shape[1]
    vals = torch.tensor([float("nan"), float("inf"), float("-inf")], device="cuda").to(BF)
    pos = torch.arange(smax, device="cuda")
    for b in range(kc.shape[0]):
        out = (pos < int(start[b])) | (pos >= int(end[b]))
        kp[b, out] = vals[pos[out] % 3][:, None, None].expand(-1, kc.shape[2], kc.shape[3])
        vp[b, out] = vals[(pos[out] + 1) % 3][:, None, None].expand(-1, kc.shape[2], kc.shape[3])
    return kp, vp


def check_attention(qkv, kc, vc, Hq, Sq, Skv, causal, lens, start, what):
    """fp32 and rounding-matched bounds per batch row, determinism, and the masked cache rows changing no bit."""
    B = kc.shape[0]
    out = cache_attention(qkv, kc, vc, Hq, Sq, Skv, causal, lens, start)
    assert torch.equal(out, cache_attention(qkv, kc, vc, Hq, Sq, Skv, causal, lens, start)), (what, "two runs differ")
    ref, matched = attention_refs(qkv, kc, vc, Hq, Sq, Skv, causal, lens, start)
    r32 = [rel(out[b * Sq:(b + 1) * Sq], ref[b * Sq:(b + 1) * Sq].to(BF)) for b in range(B)]
    rm = [rel(out[b * Sq:(b + 1) * Sq], matched[b * Sq:(b + 1) * Sq]) for b in range(B)]
    print(f"{what}: vs fp32 max rel {max(r32):.3e}, vs rounding-matched max rel {max(rm):.3e}")
    assert max(r32) < 3e-3, (what, "vs fp32", r32)
    assert max(rm) < 1e-3, (what, "vs rounding-matched", rm)     # 4.4e-4 measured at most (H100 80GB HBM3, 700 W, every case)
    beg = torch.zeros(B, dtype=torch.int32, device="cuda") if start is None else start
    end = torch.full((B,), Skv, dtype=torch.int32, device="cuda") if lens is None else lens.clamp(max=Skv)
    kp, vp = poison_outside(kc, vc, beg, end)
    assert torch.equal(cache_attention(qkv, kp, vp, Hq, Sq, Skv, causal, lens, start), out), (what, "reads a masked cache row")
    return out


DECODE_LENS = (1, 63, 64, 65, 201, -1, 0)          # -1 / 0: S_max - 1 / S_max
PAD_STARTS = (0, 5, 64, 130)


@pytest.mark.parametrize("left_pad", [False, True])
@pytest.mark.parametrize("smax", [210, 4160])
@pytest.mark.parametrize("B", [1, 3, 8, 32])
@pytest.mark.parametrize("width", ["8b", "70b"])
def test_decode_attention_over_cache(width, B, smax, left_pad):
    Wd = W8B if width == "8b" else W70B
    decode_attention_case(Wd["Hq"], Wd["Hkv"], HD, B, smax, left_pad, width)


def decode_attention_case(Hq, Hkv, D, B, smax, left_pad, width):
    """One query per stream (Sq = 1, non-causal, kv_len = lens) over the whole static cache on ``attn_fwd_kernel``; B = 32 is
    8 prompts x 4 beams.  Then bit-exact: a row whose one visible key is kv_len - 1 returns that key's V row, kv_start = kv_len
    returns zeros, and another row's cache changes no output of this row."""
    off = {1: 5, 3: 2, 8: 0, 32: 3}[B] + (smax == 4160)
    L = [smax + x if x <= 0 else x for x in DECODE_LENS]
    lens = [L[(b + off) % len(L)] for b in range(B)]
    starts = [PAD_STARTS[b % 4] if left_pad else 0 for b in range(B)]
    if left_pad:
        lens = [min(smax, s + n) for s, n in zip(starts, lens)]
    lens_t = torch.tensor(lens, dtype=torch.int32, device="cuda")
    start_t = torch.tensor(starts, dtype=torch.int32, device="cuda") if left_pad else None
    seed = 100 * B + smax
    qkv = rnd(B, (Hq + 2 * Hkv) * D, seed=seed)
    kc, vc = rnd(B, smax, Hkv, D, seed=seed + 1), rnd(B, smax, Hkv, D, seed=seed + 2)
    what = f"decode {width} B={B} S_max={smax} lens={lens} starts={starts}"
    out = check_attention(qkv, kc, vc, Hq, 1, smax, False, lens_t, start_t, what)
    # one visible key (kv_start = kv_len - 1): P = 1, the output is that key's V row exactly
    one = cache_attention(qkv, kc, vc, Hq, 1, smax, False, lens_t, lens_t - 1)
    last_v = vc[torch.arange(B, device="cuda"), (lens_t - 1).long()]                       # [B, Hkv, D]
    assert torch.equal(one, last_v.repeat_interleave(Hq // Hkv, 1).reshape(B, Hq * D)), what
    # no visible key (kv_start = kv_len): zeros
    assert int(torch.count_nonzero(cache_attention(qkv, kc, vc, Hq, 1, smax, False, lens_t, lens_t.clone()))) == 0, what
    # batch isolation: a new cache for the last row moves no bit of the others, and does move the last row
    if B >= 2:
        k2, v2 = kc.clone(), vc.clone()
        k2[-1], v2[-1] = rnd(smax, Hkv, D, seed=seed + 3), rnd(smax, Hkv, D, seed=seed + 4)
        o2 = cache_attention(qkv, k2, v2, Hq, 1, smax, False, lens_t, start_t)
        assert torch.equal(o2[:-1], out[:-1]), (what, "row isolation")
        assert not torch.equal(o2[-1], out[-1]), what


@pytest.mark.parametrize("left_pad", [False, True])
@pytest.mark.parametrize("Sq", [2, 7, 15, 16, 33])
@pytest.mark.parametrize("width", ["8b", "70b"])
def test_prefill_attention_on_cache(width, Sq, left_pad):
    Wd = W8B if width == "8b" else W70B
    prefill_on_cache_case(Wd["Hq"], Wd["Hkv"], HD, Sq, left_pad, width)


def prefill_on_cache_case(Hq, Hkv, D, Sq, left_pad, width):
    """A short prompt or conversation turn prefilled on top of a cache (model.py ``llama_hidden``): causal with past = 137 keys
    before the Sq queries (shift = Skv - Sq > 0), kv_start in {0, 5, 64, 130}.  Sq < 16 runs on the mma.sync kernel, Sq >= 16 on
    the wgmma kernel and once more on the mma.sync kernel."""
    from ultravox_b200 import _lib
    B, past, smax = 4, 137, 210
    Skv = past + Sq
    start_t = torch.tensor(PAD_STARTS, dtype=torch.int32, device="cuda") if left_pad else None
    seed = 7 * Sq + 1000 * left_pad
    qkv = rnd(B * Sq, (Hq + 2 * Hkv) * D, seed=seed)
    kc, vc = rnd(B, smax, Hkv, D, seed=seed + 1), rnd(B, smax, Hkv, D, seed=seed + 2)
    what = f"cache prefill {width} Sq={Sq} past={past} starts={PAD_STARTS if left_pad else None}"
    out = check_attention(qkv, kc, vc, Hq, Sq, Skv, True, None, start_t, what)
    if Sq >= 16:
        _lib.lib().uvx_debug_attn_tc(0)
        try:
            out_mma = check_attention(qkv, kc, vc, Hq, Sq, Skv, True, None, start_t, what + " (mma.sync)")
        finally:
            _lib.lib().uvx_debug_attn_tc(-1)
        assert rel(out, out_mma) < 3e-3
    # causality, bit-exact: key past + i0 reaches no query before i0 and does reach query i0
    i0 = Sq // 2
    k2, v2 = kc.clone(), vc.clone()
    k2[:, past + i0], v2[:, past + i0] = rnd(B, Hkv, D, seed=seed + 3), rnd(B, Hkv, D, seed=seed + 4)
    o2 = cache_attention(qkv, k2, v2, Hq, Sq, Skv, True, None, start_t).view(B, Sq, -1)
    o1 = out.view(B, Sq, -1)
    assert torch.equal(o2[:, :i0], o1[:, :i0]), (what, "a query sees a later key")
    assert not torch.equal(o2[:, i0], o1[:, i0]), what


# ================================================================================================ 2. matrix-vector linears
GEMV_SHAPES = {
    # 8B: q|k|v, o_proj, gate|up, down_proj
    "8b_qkv": (6144, 4096), "8b_o": (4096, 4096), "8b_gate_up": (28672, 4096), "8b_down": (4096, 14336),
    # 70B
    "70b_qkv": (10240, 8192), "70b_o": (8192, 8192), "70b_gate_up": (57344, 8192), "70b_down": (8192, 28672),
    # tails: N not a multiple of the CTA's 8 rows; K / 8 = 161 vectors is not a multiple of the 32 lanes
    "tail_n": (1000, 4096), "tail_k": (6144, 1288), "tail_nk": (1000, 1288),
}


def strided(t, pad_front, pad_back):
    """The same values as a column view of a wider buffer (row stride = cols + pad_front + pad_back)."""
    buf = torch.full((t.shape[0], t.shape[1] + pad_front + pad_back), float("nan"), dtype=t.dtype, device=t.device)
    buf[:, pad_front:pad_front + t.shape[1]] = t
    return buf[:, pad_front:pad_front + t.shape[1]]


@pytest.mark.parametrize("shape", list(GEMV_SHAPES))
def test_gemv_and_decode_gemm_at_width(shape):
    gemv_case(*GEMV_SHAPES[shape], shape)


def gemv_case(N, K, shape):
    """``ops.gemv`` at B in {1, 2, 5, 8} with a residual, x / residual / out as strided views: fp32 output within
    gamma(8 ceil(K/256) + 6) sum|x w| of fp64 (8 FMAs per lane per 256 columns, a 5-level shuffle tree, the residual add), bf16
    output within that plus one ulp and rel < 1e-3; the same bits as dense operands.  K = 28672 at B = 8 takes the slab loop (3
    slabs).  Then, for the eight 8B / 70B projections, the decode form of the tensor-core GEMM (``ops.linear``, 2+ streams) at
    B in {2, 3, 8}, plain and with a residual: rel < 1e-3 against fp32 math and the same bits from run to run."""
    from ultravox_b200 import ops
    w = rnd(N, K, scale=0.02, seed=N + K)
    x8, r8 = rnd(8, K, seed=1), rnd(8, N, scale=0.5, seed=2)
    ref8, mag8 = matvec_f64(x8, w, r8)
    n_fp32 = 8 * math.ceil(K / 256) + 6
    for B in (1, 2, 5, 8):
        x, r, ref, mag = x8[:B], r8[:B], ref8[:B], mag8[:B]
        xs, rs = strided(x, 64, 64), strided(r, 8, 3)
        for dt in (torch.float32, BF):
            ob = torch.full((B, N + 40), -7.0, dtype=dt, device="cuda")
            got = ops.gemv(xs, w, residual=rs, out=ob[:, 24:24 + N])
            assert torch.equal(ob[:, :24], torch.full_like(ob[:, :24], -7.0)) and torch.equal(ob[:, 24 + N:], torch.full_like(ob[:, 24 + N:], -7.0))
            bound = gamma(n_fp32) * mag
            if dt == BF:
                bound = bound + bf16_ulp(ref)
                assert rel(got, ref.to(BF)) < 1e-3, (shape, B, rel(got, ref.to(BF)))
            assert_within(got, ref, bound, f"gemv {shape} B={B} {dt}")
            assert torch.equal(got, ops.gemv(x, w, residual=r, out_dtype=dt)), (shape, B, dt, "strided != dense")
    # decode form of the tensor-core GEMM (its ABI takes N % 64 == 0: every projection of both widths)
    if N % 64:
        return
    wf = w.float()
    for B in (2, 3, 8):
        x, r = x8[:B], r8[:B]
        plain = x.float() @ wf.T
        for res in (None, r):
            got = ops.linear(x, w, residual=res)
            want = plain if res is None else plain + res.float()
            e = rel(got, want.to(BF))
            assert e < 1e-3, (shape, B, res is not None, e)
            assert torch.equal(got, ops.linear(x, w, residual=res)), (shape, B, "two runs differ")


def rmsnorm_hf(x, w, eps):
    """LlamaRMSNorm in HF's rounding order, fp64 arithmetic: x * rsqrt(mean(x^2) + eps) rounded to bf16, times the weight,
    rounded to bf16."""
    xd = x.to(F64)
    xn = (xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)).to(BF)
    return (w.to(F64) * xn.to(F64)).to(BF)


def swiglu_hf(gu):
    """LlamaMLP's act_fn(gate) * up on bf16 tensors: silu(gate) rounded to bf16, the product rounded to bf16."""
    K = gu.shape[1] // 2
    g, u = gu[:, :K].to(F64), gu[:, K:].to(F64)
    return ((g * torch.sigmoid(g)).to(BF).to(F64) * u).to(BF)


@pytest.mark.parametrize("case", [
    # RMSNorm prologue: q|k|v and gate|up of both widths
    ("norm", 6144, 4096, (1, 5, 8)), ("norm", 28672, 4096, (2, 8)), ("norm", 10240, 8192, (1, 8)), ("norm", 57344, 8192, (3,)),
    # SwiGLU prologue: down_proj; each side of ops.gemv's shared-memory switch (B * 2K * 2 bytes > 200 KiB -> unfused)
    ("swiglu", 4096, 14336, (1, 7, 8)), ("swiglu", 8192, 28672, (1, 3, 4, 8))])
def test_gemv_fused_prologues_at_width(case):
    gemv_prologue_case(case)


def gemv_prologue_case(case):
    """``gemv(norm=)`` / ``gemv(swiglu=True)`` against fp64 LlamaRMSNorm / act(gate) * up in HF's rounding order followed by
    the matmul (rel < 1e-3), and bit-identical to the separate kernels they replace."""
    from ultravox_b200 import ops
    kind, N, K, Bs = case
    w = rnd(N, K, scale=0.02, seed=N + 3 * K)
    nw = rnd(K, scale=0.3, seed=5).float().add(1.0).to(BF)
    xw = 2 * K if kind == "swiglu" else K
    xall, rall = rnd(max(Bs), xw, scale=3.0, seed=6), rnd(max(Bs), N, seed=7)
    for B in Bs:
        x, r = xall[:B], rall[:B]
        if kind == "norm":
            got = ops.gemv(x, w, residual=r, norm=(nw, 1e-5))
            act = rmsnorm_hf(x, nw, 1e-5)
            unfused = ops.gemv(ops.rmsnorm(x, nw, 1e-5), w, residual=r)
        else:
            got = ops.gemv(x, w, residual=r, swiglu=True)
            act = swiglu_hf(x)
            unfused = ops.gemv(ops.swiglu(x, gate_first=True), w, residual=r)
        ref, _ = matvec_f64(act, w, r)
        e = rel(got, ref.to(BF))
        print(f"gemv {kind} N={N} K={K} B={B}: rel {e:.3e}")
        assert e < 1e-3, (case, B, e)
        assert torch.equal(got, unfused), (case, B, "fused != unfused")


# ================================================================================================ 4. LM head and argmax
@pytest.mark.parametrize("d", [4096, 8192])
def test_lm_head_full_vocab(d):
    """V = 128256 at B in {1, 2, 7, 8, 9, 12, 32} (B > 8 runs in slabs of 8), on a dense h and on ``hid[:, -1, :]`` of a
    [B, 5, d] tensor (row stride 5 d): every logit within gamma(8 ceil(d/256) + 5) sum|h w| of fp64; argmax == torch.argmax."""
    from ultravox_b200 import ops
    w = rnd(V_LLM, d, scale=0.02, seed=d)
    hid = rnd(32, 5, d, seed=d + 1)
    ref, mag = matvec_f64(hid[:, -1], w)
    bound = gamma(8 * math.ceil(d / 256) + 5) * mag
    for B in (1, 2, 7, 8, 9, 12, 32):
        for h in (hid[:B, -1].contiguous(), hid[:B, -1, :]):
            lg = ops.lm_head(h, w)
            assert_within(lg, ref[:B], bound[:B], f"lm_head d={d} B={B} row stride {h.stride(0)}")
            assert torch.equal(ops.argmax(lg), lg.argmax(-1)), (d, B)


def _tie_rows(V, B=64, seed=0):
    """[B, V] fp32 rows with planted exact maxima at indices owned by different elements of a float4, threads, warps and
    passes of argmax_kernel's 1024-thread stride, at 0 and V - 1; and rows that are all -inf or nearly so."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, V, generator=g)
    M = 10.0
    plants = [
        [0], [V - 1], [0, V - 1], [V - 2, V - 1],
        [4 * 7 + 1, 4 * 7 + 2],                      # one float4
        [4 * 7 + 3, 4 * 8],                          # neighbouring threads
        [4 * 1000, 4 * 3075],                        # warp 31 (float4 1000) before warp 0 (float4 3075 = thread 3, pass 3)
        [4 * 33, 4 * 1],                             # warps 1 and 0
        [4 * 31 + 2, 4 * 32],                        # last lane of warp 0, first of warp 1
        [5, 5 + 4096, 5 + 8192],                     # one thread, three passes
        [4 * 1023 + 3, 4 * 1024],                    # last thread's first float4, first thread's second
        [V // 2, V // 2 + 1, V // 3],
    ]
    for b in range(B):
        if b < len(plants):
            idx = [i for i in plants[b] if i < V]
        else:
            idx = torch.randint(0, V, (1 + b % 5,), generator=g).tolist()
        x[b, idx] = M
    x[40] = float("-inf")                            # all -inf: torch returns 0
    x[41] = float("-inf")
    x[41, V - 1] = -1e30
    x[42] = float("-inf")
    x[42, [3, V - 3]] = -5.0
    x[43] = torch.where(x[43] > 1.0, x[43], torch.full_like(x[43], float("-inf")))
    return x.cuda()


@pytest.mark.parametrize("V", [V_LLM, 32001, 7])
def test_argmax_ties_and_edges(V):
    """Equal to torch.argmax (first maximal index) on 64 rows with planted exact ties, rows that are all -inf, and V = 32001,
    where the rows whose start is not 16-byte aligned (b * V % 4 != 0) take the scalar path.  A row that is all -inf used to
    come back as INT64_MAX (aligned rows, V % 4 == 0) or as the first index of the scalar tail (V = 32001: 32000)."""
    from ultravox_b200 import ops
    x = _tie_rows(V)
    got = ops.argmax(x)
    want = x.argmax(-1)
    bad = torch.nonzero(got != want).view(-1).tolist()
    assert not bad, [(b, int(got[b]), int(want[b])) for b in bad[:8]]
    assert int(got[40]) == 0
    # a row that does not start on a 16-byte boundary
    if V % 4:
        sub = x.view(-1)[1:1 + 3 * V].view(3, V)
        assert sub.data_ptr() % 16 != 0
        assert torch.equal(ops.argmax(sub), sub.argmax(-1))


# ================================================================================================ 5. RoPE + cache append
@pytest.mark.parametrize("width", ["8b", "70b"])
def test_rope_kv_append_long_positions(width):
    Wd = W8B if width == "8b" else W70B
    rope_kv_append_case(Wd["Hq"], Wd["Hkv"], HD, "v0_5_8b", width)


def rope_kv_append_case(Hq, Hkv, D, name, width):
    """B = 8 streams at RoPE positions up to 131071 (llama3 scaling) written to cache slots that differ from them (left
    padding): q and k within one ulp of the fp64 rotation with the same fp32 tables (+ 2^-23 (|x1 c| + |x2 s|), the fp32
    rounding of the two products when they cancel); the cache row is the rotated k and the raw v bit for bit; every other
    slot keeps its sentinel; ``rope_`` with ``positions=`` + ``kv_append`` give the same bits."""
    from ultravox_b200 import ops
    from ultravox_b200.config import PRESETS
    tc = PRESETS[name]["text_config"]
    B, smax = 8, 210
    inv = ops.llama3_inv_freq(D, tc["rope_theta"], tc["rope_scaling"])
    cos, sin = ops.rope_tables(inv, 131072, "cuda")
    rope_pos = torch.tensor([0, 1, 8191, 8192, 65535, 100003, 131070, 131071], dtype=torch.int32, device="cuda")
    slot = torch.tensor([3, 0, 77, 209, 5, 150, 1, 9], dtype=torch.int32, device="cuda")
    qkv0 = rnd(B, (Hq + 2 * Hkv) * D, scale=2.0, seed=11)
    sentinel = -3.5
    kc = torch.full((B, smax, Hkv, D), sentinel, dtype=BF, device="cuda")
    vc = kc.clone()
    qkv = qkv0.clone()
    ops.rope_kv_append_(qkv, Hq, Hkv, D, cos, sin, rope_pos, kc, vc, slot)
    nr = (Hq + Hkv) * D
    h = qkv0[:, :nr].to(F64).view(B, Hq + Hkv, D)
    c, s = cos[rope_pos.long()].to(F64)[:, None], sin[rope_pos.long()].to(F64)[:, None]
    x1, x2 = h[..., :D // 2], h[..., D // 2:]
    ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).view(B, nr)
    cancel = torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], -1).view(B, nr)
    assert_within(qkv[:, :nr], ref, bf16_ulp(ref) + 2.0 ** -23 * cancel, f"rope {width}")
    assert torch.equal(qkv[:, nr:], qkv0[:, nr:]), "v section changed"
    rows = torch.arange(B, device="cuda")
    assert torch.equal(kc[rows, slot.long()].view(B, -1), qkv[:, Hq * D:nr]), "cache k != rotated k"
    assert torch.equal(vc[rows, slot.long()].view(B, -1), qkv0[:, nr:]), "cache v != raw v"
    other = torch.ones(B, smax, dtype=torch.bool, device="cuda")
    other[rows, slot.long()] = False
    assert bool((kc[other] == sentinel).all()) and bool((vc[other] == sentinel).all()), "a slot other than positions[b] changed"
    q2 = qkv0.clone()
    k2, v2 = torch.full_like(kc, sentinel), torch.full_like(vc, sentinel)
    ops.rope_(q2, Hq, Hkv, D, cos, sin, rows_per_seq=1, positions=rope_pos)
    ops.kv_append(q2, k2, v2, slot, Hq, Hkv, D)
    assert torch.equal(q2, qkv) and torch.equal(k2, kc) and torch.equal(v2, vc)


# ================================================================================================ 6. one decode step composed at width
def _engine_run(model, ids, am, n_steps, use_graph):
    """generate()'s sequence (prefill with the mask-derived positions, DecodeEngine.begin with kv_start) stepped n times:
    (tokens [B, n + 1], the logits of every step)."""
    from ultravox_b200.engine import DecodeEngine
    B, S = ids.shape
    kv_start, _ = model._pad_bounds(am)
    pos = (am.cumsum(-1) - 1).clamp_min(0)
    cache = model.new_cache(B, S + n_steps + 2)
    out = model(ids, attention_mask=am, past_key_values=cache, logits_to_keep=1, position_ids=pos)
    eng = DecodeEngine(model, B, cache.capacity, use_graph=use_graph, cache=cache)
    toks = [eng.begin(ids, out.logits.view(B, -1), kv_start).clone()]
    logits = []
    for _ in range(n_steps):
        eng.step()
        logits.append(eng.logits.clone())
        toks.append(eng.token.view(-1).clone())
    return torch.stack(toks, 1), logits


@pytest.fixture(scope="module")
def model_8b_one_layer():
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=1, vocab_size=32000))
    return UltravoxModel(cfg, device="cuda").init_random_(seed=42)


@pytest.mark.parametrize("pads", [[9], [0, 17, 70]])
def test_decode_step_composed_at_width(model_8b_one_layer, pads):
    """One Llama layer at 8B widths (vocab 32000), left-padded prompts of 80 positions: B = 1 runs the matrix-vector step, B = 3
    the tensor-core GEMM step.  6 steps with and without the CUDA graph give the same logits bit for bit; each step's logits are
    within rel 1e-2 of the cacheless forward over the same sequence (teacher-forced with the engine's tokens, attention mask
    and mask-derived positions)."""
    model = model_8b_one_layer
    B, S, n = len(pads), 80, 6
    g = torch.Generator().manual_seed(17)
    ids = torch.randint(0, 32000, (B, S), generator=g).cuda()
    am = torch.ones(B, S, dtype=torch.int64, device="cuda")
    for b, p in enumerate(pads):
        am[b, :p] = 0
        ids[b, :p] = 0
    toks_e, lg_e = _engine_run(model, ids, am, n, use_graph=False)
    toks_g, lg_g = _engine_run(model, ids, am, n, use_graph=True)
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
            e = rel(lg_e[t][b], ref[b])
            worst = max(worst, e)
            assert e < 1e-2, (pads, t, b, e)       # 5.5e-3 measured at most (H100 80GB HBM3, 700 W)
    print(f"composed decode step pads={pads}: max rel vs cacheless forward {worst:.3e}")
