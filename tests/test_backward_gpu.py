"""Per-op parity of the adapter-training backward kernels at the widths and masks training runs (DESIGN a14).

Each kernel is called through ``ops`` / ``losses`` on bf16 inputs and compared with plain fp32 / fp64 math of the same operation,
at the shapes ``autograd.py`` passes when training Whisper-large + Llama-3.1-8B adapters:

* attention backward (and the forward log-sum-exp it reads): the encoder form (non-causal, head_dim 64, 20 heads, S = 1500,
  per-clip ``kv_len``) and the LLM form (causal GQA, head_dim 128, right padding), against fp32 autograd, against a reference
  that rounds P and dS to bf16 where the kernel does, and with exact (bit-level) mask, causality and batch-isolation checks;
* RMSNorm (plain and the ln_pre stack mode with dx), LayerNorm, GELU, SwiGLU and RoPE backwards at width;
* cross entropy and KL distillation at V = 128256, strided logits included;
* AdamW as a step function, transpose and splice_inverse;
* one encoder-LoRA training step at width with ragged clips, against the fp32 CPU oracle's autograd.

Bounds: ``rel`` is a Frobenius-norm relative error; "ulp" is the spacing of bf16 at the reference value.  Where a bound carries an
fp32 term it is the rounding of the kernel's fp32 arithmetic on operands that cancel (e.g. softmax(s) - softmax(t)), which the
bf16 ulp of a near-zero result cannot absorb."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64


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


def rnd(*shape, scale=1.0, seed=0, mean=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g, dtype=torch.float32) * scale + mean).to(BF).cuda()


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


# ================================================================================================ 1. attention backward
class Attn:
    """One forward (with lse) + backward through the fused-qkv wrappers; ``block`` > 0 builds the argument struct directly
    (``uvx_attention_bwd`` accepts a block-causal mask although training does not use one)."""

    def __init__(self, B, S, Hq, Hkv, D, causal, kv_len=None, block=0):
        self.B, self.S, self.Hq, self.Hkv, self.D, self.causal, self.block = B, S, Hq, Hkv, D, causal, block
        self.kv_len = None if kv_len is None else torch.tensor(kv_len, dtype=torch.int32, device="cuda")
        self.lens = list(kv_len) if kv_len is not None else [S] * B
        self.scale = D ** -0.5
        self.W = (Hq + 2 * Hkv) * D

    def run(self, qkv, dout):
        from ultravox_b200 import ops
        B, S, Hq, Hkv, D = self.B, self.S, self.Hq, self.Hkv, self.D
        out = torch.empty(B * S, Hq * D, dtype=BF, device="cuda")
        lse = torch.empty(B * Hq * S, dtype=torch.float32, device="cuda")
        if self.block == 0:
            ops.attention_fused_qkv_train(qkv, B, S, Hq, Hkv, D, self.scale, self.causal, out, lse, self.kv_len)
            dqkv = ops.attention_fused_qkv_bwd(qkv, out, dout, lse, B, S, Hq, Hkv, D, self.scale, self.causal, kv_len=self.kv_len)
            return out, lse.view(B, Hq, S), dqkv
        from ultravox_b200._lib import AttnArgs, check, lib
        rs, base = qkv.stride(0), qkv.data_ptr()
        a = AttnArgs()
        a.q, a.k, a.v, a.o = base, base + 2 * Hq * D, base + 2 * (Hq + Hkv) * D, out.data_ptr()
        a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, S, S, D
        (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = (rs, S * rs, rs, S * rs, rs, S * rs, Hq * D, S * Hq * D)
        a.kv_len = self.kv_len.data_ptr() if self.kv_len is not None else None
        a.causal, a.block, a.scale, a.lse = int(self.causal), self.block, self.scale, lse.data_ptr()
        st = torch.cuda.current_stream().cuda_stream
        check(lib().uvx_attention(C.byref(a), st), "uvx_attention")
        dqkv = torch.empty_like(qkv)
        delta = torch.empty(B * Hq * S, dtype=torch.float32, device="cuda")
        db = dqkv.data_ptr()
        check(lib().uvx_attention_bwd(C.byref(a), out.data_ptr(), dout.data_ptr(), db, db + 2 * Hq * D, db + 2 * (Hq + Hkv) * D,
                                      rs, S * rs, rs, S * rs, rs, S * rs, delta.data_ptr(), st), "uvx_attention_bwd")
        return out, lse.view(B, Hq, S), dqkv

    def allowed(self):
        """[B, 1, S(query), S(key)] visibility mask."""
        S = self.S
        i = torch.arange(S, device="cuda")[:, None]
        j = torch.arange(S, device="cuda")[None, :]
        lens = torch.tensor(self.lens, device="cuda")[:, None, None, None]
        m = (j[None, None] < lens)
        if self.causal:
            m = m & (j <= i)
        if self.block:
            m = m & (j // self.block <= i // self.block)
        return m

    def split(self, t):
        """[B*S, W] -> q [B, Hq, S, D], k / v [B, Hkv, S, D]."""
        B, S, Hq, Hkv, D = self.B, self.S, self.Hq, self.Hkv, self.D
        t = t.view(B, S, Hq + 2 * Hkv, D)
        return t[:, :, :Hq].transpose(1, 2), t[:, :, Hq:Hq + Hkv].transpose(1, 2), t[:, :, Hq + Hkv:].transpose(1, 2)

    def autograd_ref(self, qkv, dout):
        """fp32 attention + torch.autograd: (out, lse, dqkv) in fp32."""
        B, S, Hq, Hkv, D = self.B, self.S, self.Hq, self.Hkv, self.D
        t = qkv.float().requires_grad_(True)
        q, k, v = self.split(t)
        grp = Hq // Hkv
        s = (q @ k.repeat_interleave(grp, 1).transpose(-1, -2)) * self.scale
        s = s.masked_fill(~self.allowed(), float("-inf"))
        lse = torch.logsumexp(s, -1)
        o = torch.softmax(s, -1) @ v.repeat_interleave(grp, 1)
        o = o.transpose(1, 2).reshape(B * S, Hq * D)
        o.backward(dout.float())
        return o.detach(), lse.detach(), t.grad

    def matched_ref(self, qkv, out, lse, dout):
        """The kernel's own formulation in fp32 from ITS lse and output: P and dS rounded to bf16 before the products that
        consume them as mma operands (attention_bwd.cu), sums over the query heads of a group in fp32."""
        B, S, Hq, Hkv, D = self.B, self.S, self.Hq, self.Hkv, self.D
        grp = Hq // Hkv
        q, k, v = (x.float() for x in self.split(qkv))
        k2, v2 = k.repeat_interleave(grp, 1), v.repeat_interleave(grp, 1)
        do = dout.float().view(B, S, Hq, D).transpose(1, 2)
        o = out.float().view(B, S, Hq, D).transpose(1, 2)
        s = (q @ k2.transpose(-1, -2)) * self.scale
        p = torch.exp(s - lse[..., None]).masked_fill(~self.allowed(), 0.0)
        del s
        delta = (do * o).sum(-1, keepdim=True)
        ds = p * ((do @ v2.transpose(-1, -2)) - delta) * self.scale
        pb, dsb = p.to(BF).float(), ds.to(BF).float()
        del p, ds
        dv = (pb.transpose(-1, -2) @ do).view(B, Hkv, grp, S, D).sum(2)
        dk = (dsb.transpose(-1, -2) @ q).view(B, Hkv, grp, S, D).sum(2)
        dq = dsb @ k2
        g = torch.cat([dq, dk, dv], 1).transpose(1, 2).reshape(B * S, self.W)
        return g

    def sections(self):
        qd, kd = self.Hq * self.D, self.Hkv * self.D
        return {"dQ": slice(0, qd), "dK": slice(qd, qd + kd), "dV": slice(qd + kd, qd + 2 * kd)}

    def per_batch_rel(self, got, ref):
        """{(name, b): rel} over the dQ / dK / dV sections of each batch element.  An element whose exact gradient is ~0 (a clip
        with one key: P = 1, dS = 0) is measured against 1 % of the section's mean per-element norm instead."""
        out = {}
        for name, sl in self.sections().items():
            g, r = got[:, sl].double().reshape(self.B, -1), ref[:, sl].double().reshape(self.B, -1)
            floor = 1e-2 * float(r.norm()) / math.sqrt(self.B)
            for b in range(self.B):
                out[(name, b)] = float((g[b] - r[b]).norm()) / max(float(r[b].norm()), floor, 1e-30)
        return out


ATTN_CASES = {
    # encoder (Whisper-large): non-causal, head_dim 64, 20 heads, per-clip key lengths
    "enc_1500_kv563": dict(B=2, S=1500, Hq=20, Hkv=20, D=64, causal=False, kv_len=[1500, 563]),
    "enc_600_kv250_1": dict(B=3, S=600, Hq=20, Hkv=20, D=64, causal=False, kv_len=[600, 250, 1]),
    "enc_77": dict(B=1, S=77, Hq=20, Hkv=20, D=64, causal=False),
    # LLM (Llama-3.1-8B / 70B head layout): causal GQA, head_dim 128, right padding
    "llm_bench_4x201": dict(B=4, S=201, Hq=32, Hkv=8, D=128, causal=True),
    "llm_201_kv150": dict(B=2, S=201, Hq=32, Hkv=8, D=128, causal=True, kv_len=[201, 150]),
    "llm_640_kv333": dict(B=2, S=640, Hq=32, Hkv=8, D=128, causal=True, kv_len=[640, 333]),
    "llm_group8_130": dict(B=1, S=130, Hq=64, Hkv=8, D=128, causal=True),
    # ABI: block-causal with key lengths
    "block100_kv170": dict(B=2, S=300, Hq=4, Hkv=4, D=64, causal=False, kv_len=[300, 170], block=100),
}


def _inputs(A, seed):
    return rnd(A.B * A.S, A.W, seed=seed), rnd(A.B * A.S, A.Hq * A.D, seed=seed + 1)


@pytest.mark.parametrize("case", list(ATTN_CASES))
def test_attention_bwd_vs_fp32(case):
    bwd_vs_fp32_case(Attn(**ATTN_CASES[case]), case)


def bwd_vs_fp32_case(A, case):
    """Forward out / lse, then dQ, dK, dV per batch element against fp32 autograd (rel < 1e-2) and against the rounding-matched
    fp32 reference (rel < 1e-3)."""
    qkv, dout = _inputs(A, 11)
    out, lse, dqkv = A.run(qkv, dout)
    ref_o, ref_lse, ref_g = A.autograd_ref(qkv, dout)
    for b in range(A.B):
        rows = slice(b * A.S, (b + 1) * A.S)
        assert rel(out[rows], ref_o[rows].to(BF)) < 3e-3, (case, b, rel(out[rows], ref_o[rows].to(BF)))
    assert torch.allclose(lse, ref_lse, atol=2e-3, rtol=1e-3), (case, float((lse - ref_lse).abs().max()))
    r_auto = A.per_batch_rel(dqkv, ref_g)
    del ref_g
    r_match = A.per_batch_rel(dqkv, A.matched_ref(qkv, out, lse, dout).to(BF))
    print(f"{case}: vs fp32 autograd max rel {max(r_auto.values()):.3e}, vs rounding-matched max rel {max(r_match.values()):.3e}")
    bad = {k: v for k, v in r_auto.items() if not v < 1e-2}
    assert not bad, (case, "vs fp32 autograd", bad)
    bad = {k: v for k, v in r_match.items() if not v < 1e-3}       # 1.7e-4 measured at most (H100, every case here)
    assert not bad, (case, "vs rounding-matched", bad)


@pytest.mark.parametrize("case", list(ATTN_CASES))
def test_attention_bwd_masks_exact(case):
    bwd_masks_case(Attn(**ATTN_CASES[case]), case)


def bwd_masks_case(A, case):
    """Bit-level mask checks: what the mask hides cannot move a single bit, what it shows must move something."""
    B, S, sec = A.B, A.S, A.sections()
    kv = slice(sec["dK"].start, sec["dV"].stop)                 # the k | v columns of the fused layout (and of dqkv)
    qkv, dout = _inputs(A, 21)
    out, lse, dqkv = A.run(qkv, dout)
    # determinism: the kernels are atomic-free
    out2, lse2, dqkv2 = A.run(qkv, dout)
    assert torch.equal(out, out2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2), case
    g = torch.Generator().manual_seed(5)

    def fresh(n, w):
        return (torch.randn(n, w, generator=g) * 2).to(BF).cuda()

    # keys at or past kv_len: zero gradient, and their k / v values change nothing at all
    if A.kv_len is not None:
        q2 = qkv.clone()
        for b, L in enumerate(A.lens):
            rows = slice(b * S + L, (b + 1) * S)
            assert int(torch.count_nonzero(dqkv[rows, kv])) == 0, (case, b, "dK/dV must be 0 past kv_len")
            q2[rows, kv] = fresh(S - L, kv.stop - kv.start)
        o_, l_, d_ = A.run(q2, dout)
        assert torch.equal(o_, out) and torch.equal(l_, lse), (case, "forward reads keys past kv_len")
        assert torch.equal(d_, dqkv), (case, "backward reads keys past kv_len")
    # the last visible key is not masked: dV there is P^T dO != 0, and its k / v reach dQ
    for b, L in enumerate(A.lens):
        row = b * S + L - 1
        assert int(torch.count_nonzero(dqkv[row, sec["dV"]])) > 0, (case, b, "dV of the last visible key is 0")
        if L >= 2:
            q2 = qkv.clone()
            q2[row, kv] = fresh(1, kv.stop - kv.start)
            _, _, d_ = A.run(q2, dout)
            rows = slice(b * S, (b + 1) * S)
            assert not torch.equal(d_[rows, sec["dQ"]], dqkv[rows, sec["dQ"]]), (case, b, "key kv_len-1 does not reach dQ")
    # causality: key j reaches no query i < j; query i reaches no key j > i
    if A.causal:
        j = S // 2 + 3
        q2 = qkv.clone()
        q2[j, kv] = fresh(1, kv.stop - kv.start)
        o_, l_, d_ = A.run(q2, dout)
        assert torch.equal(o_[:j], out[:j]) and torch.equal(l_[0, :, :j], lse[0, :, :j]), (case, "forward: key j seen before j")
        assert torch.equal(d_[:j, sec["dQ"]], dqkv[:j, sec["dQ"]]), (case, "dQ rows i < j depend on key j")
        assert not torch.equal(d_[j:S, sec["dQ"]], dqkv[j:S, sec["dQ"]]), case
        i = S // 2 - 5
        q2, do2 = qkv.clone(), dout.clone()
        q2[i, sec["dQ"]] = fresh(1, A.Hq * A.D)
        do2[i] = fresh(1, A.Hq * A.D)
        _, _, d_ = A.run(q2, do2)
        assert torch.equal(d_[i + 1:S, kv], dqkv[i + 1:S, kv]), (case, "dK/dV rows j > i depend on query i")
        assert not torch.equal(d_[:i + 1, kv], dqkv[:i + 1, kv]), case
    # batch isolation: every row of element 1 changes, element 0 does not move
    if B >= 2:
        q2, do2 = qkv.clone(), dout.clone()
        q2[S:2 * S] = fresh(S, A.W)
        do2[S:2 * S] = fresh(S, A.Hq * A.D)
        o_, l_, d_ = A.run(q2, do2)
        assert torch.equal(o_[:S], out[:S]) and torch.equal(l_[0], lse[0]) and torch.equal(d_[:S], dqkv[:S]), case


# ================================================================================================ 2. norm backwards at width
@pytest.mark.parametrize("T2", [1500, 77])
def test_rmsnorm_bwd_stack_mode_dx(T2):
    """ln_pre backward exactly as projector_backward(want_d_enc=True) calls it: 8 x 1280 = 10240 columns (the kernel's widest),
    the clip's last stacked row partial (1500 % 8 = 4, 77 % 8 = 5); dx in the stacked layout."""
    from ultravox_b200 import ops
    N, dE, k = 2, 1280, 8
    rows_a = -(-T2 // k)
    enc, w, dy = rnd(N, T2, dE, seed=1), rnd(k * dE, scale=0.5, mean=1.0, seed=2), rnd(N * rows_a, k * dE, seed=3)
    ef, wf = enc.to(F64).requires_grad_(True), w.to(F64).requires_grad_(True)
    st = F.pad(ef, (0, 0, 0, rows_a * k - T2)).reshape(N * rows_a, k * dE)
    (wf * (st * torch.rsqrt(st.pow(2).mean(-1, keepdim=True) + 1e-6))).backward(dy.to(F64))
    dw = torch.zeros(k * dE, device="cuda")
    d_st = ops.rmsnorm_bwd(dy, enc, w, 1e-6, want_dx=True, dw=dw, stack=(rows_a, T2 * dE))
    assert d_st.shape == (N * rows_a, k * dE)
    dx = d_st.view(N, rows_a * k, dE)[:, :T2]
    assert rel(dx, ef.grad.to(BF)) < 2e-3, rel(dx, ef.grad.to(BF))
    tail = slice((rows_a - 1) * k, T2)                       # the frames of each clip's partial last row
    assert rel(dx[:, tail], ef.grad[:, tail].to(BF)) < 2e-3, rel(dx[:, tail], ef.grad[:, tail].to(BF))
    assert rel(dw, wf.grad) < 1e-3, rel(dw, wf.grad)


@pytest.mark.parametrize("rows,cols,eps", [(402, 4096, 1e-5), (201, 8192, 1e-5), (376, 2048, 1e-6)])
def test_rmsnorm_bwd_plain_width(rows, cols, eps):
    rmsnorm_bwd_case(rows, cols, eps)


def rmsnorm_bwd_case(rows, cols, eps):
    """The LLM's norms (4096 at B*S = 402, 8192 for 70B widths) and the v0_5_8b projector's ln_mid (2048 over N*rows_a = 376,
    eps 1e-6), with the residual gradient, and dw accumulated (+=) into a pre-filled buffer."""
    from ultravox_b200 import ops
    x, w, dy, dres = rnd(rows, cols, seed=1), rnd(cols, scale=0.5, mean=1.0, seed=2), rnd(rows, cols, seed=3), rnd(rows, cols, seed=4)
    xf, wf = x.to(F64).requires_grad_(True), w.to(F64).requires_grad_(True)
    (wf * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))).backward(dy.to(F64))
    dw0 = torch.randn(cols, generator=torch.Generator().manual_seed(5)).cuda() * float(wf.grad.abs().mean())
    dw = dw0.clone()
    dx = ops.rmsnorm_bwd(dy, x, w, eps, dres=dres, dw=dw)
    ref = (xf.grad + dres.to(F64)).to(BF)
    assert rel(dx, ref) < 2e-3, rel(dx, ref)
    assert rel(dw, dw0.to(F64) + wf.grad) < 1e-3, rel(dw, dw0.to(F64) + wf.grad)


@pytest.mark.parametrize("rows,cols,mean,with_dres", [(3000, 1280, 0.0, True), (3000, 1280, 0.0, False), (3000, 1280, 30.0, True),
                                                       (257, 2048, 0.0, True)])
def test_layernorm_bwd_width(rows, cols, mean, with_dres):
    """Whisper-large's encoder LayerNorms (2 clips x 1500 frames x 1280), a large common offset (mean 30, std 0.5: the mean
    must be removed before the variance), and 2048 columns, the kernel's maximum."""
    from ultravox_b200 import ops
    std = 0.5 if mean else 1.0
    x, w, dy = rnd(rows, cols, scale=std, mean=mean, seed=1), rnd(cols, scale=0.5, mean=1.0, seed=2), rnd(rows, cols, seed=3)
    b = rnd(cols, seed=4)
    dres = rnd(rows, cols, seed=5) if with_dres else None
    xf = x.to(F64).requires_grad_(True)
    F.layer_norm(xf, (cols,), w.to(F64), b.to(F64), 1e-5).backward(dy.to(F64))
    ref = xf.grad + (dres.to(F64) if with_dres else 0)
    dx = ops.layernorm_bwd(dy, x, w, 1e-5, dres=dres)
    assert rel(dx, ref.to(BF)) < 2e-3, rel(dx, ref.to(BF))


# ================================================================================================ 3. elementwise backwards vs fp64
def test_gelu_bwd_every_bf16_in_range():
    """Every bf16 value in [-12, 12] (both zeros included): |got - ref| <= 1 ulp(ref) + 1e-6 |dy|."""
    from ultravox_b200 import ops
    bits = torch.arange(0, 0x8000, dtype=torch.int32).to(torch.int16)
    pos = bits.view(BF)
    pos = pos[(pos.float() <= 12.0) & torch.isfinite(pos.float())]
    x = torch.cat([pos, -pos])                                 # -pos of +0 is -0
    pad = (-x.numel()) % 8
    x = torch.cat([x, torch.zeros(pad, dtype=BF)]).cuda()
    assert bool((x.float() == 0).any()) and bool(torch.signbit(x.float()).logical_and(x.float() == 0).any())
    dy = rnd(x.numel(), seed=3)
    got = ops.gelu_bwd(x, dy)
    xd = x.to(F64)
    ref = dy.to(F64) * (0.5 * (1 + torch.erf(xd / math.sqrt(2))) + xd * torch.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi))
    assert_within(got, ref, bf16_ulp(ref) + 1e-6 * dy.to(F64).abs(), "gelu_bwd")


@pytest.mark.parametrize("rows,H,gate_first", [(201, 14336, True), (376, 2048, False)])
def test_swiglu_bwd_width(rows, H, gate_first):
    swiglu_bwd_case(rows, H, gate_first)


def swiglu_bwd_case(rows, H, gate_first):
    """LLM MLP (H = 14336, gate | up) and projector (H = 2048, up | gate), gates in [-40, 40] so the sigmoid saturates."""
    from ultravox_b200 import ops
    g = torch.Generator().manual_seed(1)
    gate = (torch.rand(rows, H, generator=g) * 80 - 40)
    lin = torch.randn(rows, H, generator=g) * 2
    x = (torch.cat([gate, lin], 1) if gate_first else torch.cat([lin, gate], 1)).to(BF).cuda()
    d = rnd(rows, H, seed=2)
    got = ops.swiglu_bwd(x, d, gate_first)
    xd, dd = x.to(F64), d.to(F64)
    gt, ln = (xd[:, :H], xd[:, H:]) if gate_first else (xd[:, H:], xd[:, :H])
    sg = torch.sigmoid(gt)
    d_lin, d_gate = dd * gt * sg, dd * ln * sg * (1 + gt * (1 - sg))
    ref = torch.cat([d_gate, d_lin], 1) if gate_first else torch.cat([d_lin, d_gate], 1)
    assert_within(got, ref, bf16_ulp(ref) + 1e-6 * dd.abs().repeat(1, 2), "swiglu_bwd")


@pytest.mark.parametrize("pos_offset", [0, 37])
def test_rope_bwd_llama3_d128(pos_offset):
    rope_bwd_case(pos_offset, 32, 8, 128, "v0_5_8b")


def rope_bwd_case(pos_offset, Hq, Hkv, D, name):
    """The rope of preset ``name`` (theta, llama3 scaling) at head_dim D, Hq / Hkv heads, B = 2 sequences of 201 rows: the explicit
    transposed rotation per (position, frequency); the v section is not touched."""
    from ultravox_b200 import ops
    from ultravox_b200.config import PRESETS
    tc = PRESETS[name]["text_config"]
    S, B = 201, 2
    inv = ops.llama3_inv_freq(D, tc["rope_theta"], tc["rope_scaling"])
    cos, sin = ops.rope_tables(inv, 256, "cuda")
    x = rnd(B * S, (Hq + 2 * Hkv) * D, seed=1)
    got = ops.rope_bwd_(x.clone(), Hq, Hkv, D, cos, sin, rows_per_seq=S, pos_offset=pos_offset)
    pos = pos_offset + torch.arange(B * S, device="cuda") % S
    c, s = cos[pos].to(F64)[:, None], sin[pos].to(F64)[:, None]
    nr = (Hq + Hkv) * D
    h = x[:, :nr].to(F64).view(B * S, Hq + Hkv, D)
    x1, x2 = h[..., :D // 2], h[..., D // 2:]
    ref = torch.cat([x1 * c + x2 * s, x2 * c - x1 * s], -1).view(B * S, nr)
    assert rel(got[:, :nr], ref.to(BF)) < 1e-3, rel(got[:, :nr], ref.to(BF))
    assert torch.equal(got[:, nr:], x[:, nr:])


# ================================================================================================ 4. losses at V = 128256
V_LLM = 128256


def _ce_inputs(R=37, seed=1):
    g = torch.Generator().manual_seed(seed)
    lg = torch.randn(R, V_LLM, generator=g)
    lg[R // 2:] *= 20.0                                        # half the rows std 1, half std 20
    lab = torch.randint(0, V_LLM, (R,), generator=g)
    lab[1], lab[2] = 0, V_LLM - 1
    lab[[3, 11, 25]] = -100
    return lg.cuda(), lab.cuda()


@pytest.mark.parametrize("shift", [False, True])
def test_ce_loss_and_bwd_full_vocab(shift):
    """loss within 1e-5 max(1, |ref|), row_lse within 1e-5 relative, dlogits within 1 bf16 ulp of the fp64 gradient
    (+ 1e-30 for entries below fp32's range); grad_scale 0.5."""
    from ultravox_b200.losses import causal_lm_loss, causal_lm_loss_bwd
    R, gs = 37, 0.5
    lg, lab = _ce_inputs(R)
    lf = lg.to(F64).requires_grad_(True)
    if shift:
        ref = F.cross_entropy(lf[:-1], lab[1:], ignore_index=-100)
    else:
        ref = F.cross_entropy(lf, lab, ignore_index=-100)
    (ref * gs).backward()
    keep = {}
    loss = causal_lm_loss(lg[None] if shift else lg, lab[None] if shift else lab, keep=keep, shift=shift)
    assert abs(float(loss) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref))), (float(loss), float(ref))
    lse_ref = torch.logsumexp(lg.to(F64), -1)
    assert_within(keep["row_lse"], lse_ref, 1e-5 * lse_ref.abs(), "row_lse")
    d = causal_lm_loss_bwd(keep, grad_scale=gs).view(R, V_LLM)
    assert_within(d, lf.grad, bf16_ulp(lf.grad) + 1e-30, "ce dlogits")


def test_ce_all_ignored_is_nan_with_zero_gradient():
    from ultravox_b200.losses import causal_lm_loss, causal_lm_loss_bwd
    lg = torch.randn(4, V_LLM, generator=torch.Generator().manual_seed(2)).cuda()
    lab = torch.full((4,), -100, dtype=torch.int64, device="cuda")
    ref = F.cross_entropy(lg, lab, ignore_index=-100)
    keep = {}
    loss = causal_lm_loss(lg, lab, keep=keep, shift=False)
    assert math.isnan(float(loss)) and math.isnan(float(ref)) and float(keep["loss2"][1]) == 0.0
    assert int(torch.count_nonzero(causal_lm_loss_bwd(keep, grad_scale=0.5))) == 0


def _kl_ref(s, t, is_eot, T, eot_w, gs):
    s, t = s.to(F64), t.to(F64)
    R = s.shape[0]
    w = torch.full((R,), 1.0 / R, dtype=F64)
    w[is_eot] += eot_w / int(is_eot.sum())
    w = w.cuda()
    ls, lt = F.log_softmax(s / T, -1), F.log_softmax(t / T, -1)
    ps, pt = ls.exp(), lt.exp()
    loss = float((w * (pt * (lt - ls)).sum(-1)).sum())
    scale = (w * gs / T)[:, None]
    # |fp32 rounding of the kernel's softmax(s/T) - softmax(t/T)| <= 2^-15 (ps + pt): a 100th of a bf16 ulp unless they cancel
    return loss, scale * (ps - pt), scale * (ps + pt) * 2.0 ** -15


def test_kl_loss_and_bwd_full_vocab():
    from ultravox_b200.losses import kl_distill_loss, kl_distill_loss_bwd
    R, T, gs = 11, 2.0, 0.5
    g = torch.Generator().manual_seed(1)
    s, t = (torch.randn(R, V_LLM, generator=g) * 3).cuda(), (torch.randn(R, V_LLM, generator=g) * 3).cuda()
    is_eot = torch.zeros(R, dtype=torch.bool)
    is_eot[[4, 10]] = True
    ref_loss, ref_d, cancel = _kl_ref(s, t, is_eot, T, 1.0, gs)
    keep = {}
    loss = float(kl_distill_loss(s, t, is_eot, T, 1.0, keep=keep))
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)
    d = kl_distill_loss_bwd(keep, grad_scale=gs)
    assert_within(d, ref_d, bf16_ulp(ref_d) + cancel + 1e-30, "kl dlogits")


def test_losses_on_strided_logits():
    """Student, teacher and CE logits as column views of wider buffers (the teacher with a different row stride than the
    student): the same answer as on dense copies; a teacher of another shape is refused."""
    from ultravox_b200.losses import causal_lm_loss, causal_lm_loss_bwd, kl_distill_loss, kl_distill_loss_bwd
    R, T, gs = 9, 2.0, 0.5
    g = torch.Generator().manual_seed(3)
    sbuf = (torch.randn(R, V_LLM + 64, generator=g) * 3).cuda()
    tbuf = (torch.randn(R, V_LLM + 128, generator=g) * 3).cuda()
    s, t = sbuf[:, :V_LLM], tbuf[:, 64:64 + V_LLM]
    is_eot = torch.zeros(R, dtype=torch.bool)
    is_eot[[3, 8]] = True
    ref_loss, ref_d, cancel = _kl_ref(s, t, is_eot, T, 1.0, gs)
    keep = {}
    loss = float(kl_distill_loss(s, t, is_eot, T, 1.0, keep=keep))
    d = kl_distill_loss_bwd(keep, grad_scale=gs)
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)
    assert_within(d, ref_d, bf16_ulp(ref_d) + cancel + 1e-30, "kl dlogits (strided)")
    keep2 = {}
    assert loss == float(kl_distill_loss(s.contiguous(), t.contiguous(), is_eot, T, 1.0, keep=keep2))
    assert torch.equal(d, kl_distill_loss_bwd(keep2, grad_scale=gs))
    with pytest.raises(ValueError):
        kl_distill_loss(s, tbuf[:R - 1, :V_LLM], is_eot, T, 1.0)
    lab = torch.randint(0, V_LLM, (R,), generator=g).cuda()
    for view in (s, sbuf[:, 1:1 + V_LLM]):                   # row stride V + 64; and a start that breaks 16-byte alignment
        k, dense = {}, {}
        loss = float(causal_lm_loss(view, lab, keep=k, shift=False))
        assert loss == float(causal_lm_loss(view.contiguous(), lab, keep=dense, shift=False))
        assert torch.equal(causal_lm_loss_bwd(k, grad_scale=gs), causal_lm_loss_bwd(dense, grad_scale=gs))
        ref = float(F.cross_entropy(view.to(F64), lab))
        assert abs(loss - ref) <= 1e-5 * max(1.0, abs(ref)), (loss, ref)


# ================================================================================================ 5. optimizer and glue
def test_adamw_step_function():
    """20 consecutive steps and one at step 10 000 on n = 1 000 003, each against fp64 arithmetic from the kernel's own previous
    state: p within 1 bf16 ulp, m and v within 1e-6 of the magnitude of their two terms."""
    from ultravox_b200 import ops
    n, lr, (b1, b2), eps, wd, gs = 1_000_003, 1e-3, (0.9, 0.95), 1e-8, 0.01, 0.5
    g0 = torch.Generator().manual_seed(1)
    p = (torch.randn(n, generator=g0) * 0.02).to(BF).cuda()
    m = (torch.randn(n, generator=g0) * 1e-3).cuda()
    v = (torch.randn(n, generator=g0) * 1e-3).pow(2).cuda()
    for step in list(range(1, 21)) + [10_000]:
        grad = (torch.randn(n, generator=g0) * 0.1).cuda()
        p0, m0, v0 = p.to(F64), m.to(F64), v.to(F64)
        ops.adamw_(p, grad, m, v, step, lr, (b1, b2), eps, wd, gs)
        gi = grad.to(F64) * gs
        mt, vt = b1 * m0, (1 - b1) * gi
        m_ref, v_ref = mt + vt, b2 * v0 + (1 - b2) * gi * gi
        assert_within(m, m_ref, 1e-6 * (mt.abs() + vt.abs()) + 1e-30, f"m step {step}")
        assert_within(v, v_ref, 1e-6 * v_ref + 1e-30, f"v step {step}")
        upd = (lr / (1 - b1 ** step)) * (m_ref / (v_ref.sqrt() / math.sqrt(1 - b2 ** step) + eps))
        p_ref = p0 * (1 - lr * wd) - upd
        assert_within(p, p_ref, bf16_ulp(p_ref) + 1e-6 * (p0.abs() + upd.abs()), f"p step {step}")


@pytest.mark.parametrize("R,Cc", [(3000, 1280), (376, 64), (201, 4096)])
def test_transpose_bit_exact(R, Cc):
    from ultravox_b200 import ops
    x = rnd(R, Cc, seed=R)
    t = ops.transpose(x)
    Rp = -(-R // 8) * 8
    assert t.shape == (Cc, Rp) and torch.equal(t[:, :R], x.T) and int(torch.count_nonzero(t[:, R:])) == 0


def test_splice_inverse_multi_clip():
    """Three clips over two of three sequences, text rows between them, and audio rows that are never spliced (-1)."""
    from ultravox_b200 import ops
    B, S, n_audio = 3, 40, 42
    src = torch.full((B * S,), -1, dtype=torch.int32)
    row = 0
    for b, start, n in ((0, 5, 12), (0, 25, 7), (2, 3, 20)):
        src[b * S + start:b * S + start + n] = torch.arange(row, row + n, dtype=torch.int32)
        row += n
    want = torch.full((n_audio,), -1, dtype=torch.int32)
    for p_, r in enumerate(src.tolist()):
        if r >= 0:
            want[r] = p_
    assert torch.equal(ops.splice_inverse(src.cuda(), n_audio).cpu(), want)


def test_backward_wrappers_take_strided_gradients():
    """Non-contiguous dy / dres (rmsnorm_bwd), dout (swiglu_bwd, attention_fused_qkv_bwd): the same bits as dense inputs."""
    from ultravox_b200 import ops
    rows, cols = 201, 4096
    x, w = rnd(rows, cols, seed=1), rnd(cols, seed=2)
    dyb, drb = rnd(rows, cols + 64, seed=3), rnd(rows, cols + 64, seed=4)
    dy, dres = dyb[:, 32:32 + cols], drb[:, :cols]
    dw1, dw2 = torch.zeros(cols, device="cuda"), torch.zeros(cols, device="cuda")
    a = ops.rmsnorm_bwd(dy, x, w, 1e-5, dres=dres, dw=dw1)
    b = ops.rmsnorm_bwd(dy.contiguous(), x, w, 1e-5, dres=dres.contiguous(), dw=dw2)
    assert torch.equal(a, b) and rel(dw1, dw2) < 1e-6
    H = 2048
    xs, db = rnd(rows, 2 * H, seed=5), rnd(rows, H + 64, seed=6)
    assert torch.equal(ops.swiglu_bwd(xs, db[:, 64:], True), ops.swiglu_bwd(xs, db[:, 64:].contiguous(), True))
    A = Attn(B=2, S=130, Hq=8, Hkv=2, D=128, causal=True, kv_len=[130, 77])
    qkv = rnd(A.B * A.S, A.W, seed=7)
    dbuf = rnd(A.B * A.S, A.Hq * A.D + 128, seed=8)
    out, _, d_dense = A.run(qkv, dbuf[:, 128:].contiguous())
    _, _, d_strided = A.run(qkv, dbuf[:, 128:])
    assert torch.equal(d_dense, d_strided)


# ================================================================================================ 6. composed: encoder LoRA at width
def test_encoder_lora_at_width_ragged_clips():
    """Encoder LoRA r = 8 trained through AdapterTrainer on one Whisper-large encoder layer + one Llama-3.1-8B layer (vocab
    32000), clips of 30 s and 11.25 s (key lengths 1500 / 563): adapter and linear_2 gradients against the fp32 CPU oracle's
    autograd with the adapters merged as W + s B A."""
    from oracle import logmel as ol, model as om
    from ultravox_b200 import ops
    from ultravox_b200.autograd import EncoderLora
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    from ultravox_b200.training import AdapterTrainer
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=1, vocab_size=32000))
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    waves = [np.random.default_rng(1000 + i).standard_normal(n).astype(np.float32) for i, n in enumerate([16000 * 30, 180_000])]
    padded, frames = ol.pad_batch(waves)
    assert [(int(f) - 1) // 2 + 1 for f in frames] == [1500, 563]
    g = torch.Generator().manual_seed(7)
    tok = [int(-(-int(f) // 16)) for f in frames]
    S = 8 + max(tok) + 5
    ids = torch.randint(0, cfg.vocab_size, (2, S), generator=g)
    labels = ids.clone()
    labels[:, :-5] = -100
    batch = dict(input_ids=ids, audio_token_start_idx=torch.tensor([8, 8]), audio_lens=torch.tensor([int(f) for f in frames]),
                 audio_token_len=torch.tensor(tok, dtype=torch.int32), audio_batch_size=torch.ones(2, dtype=torch.int64), labels=labels)
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    lora = EncoderLora(model, r=8, alpha=8.0, seed=3)
    r = lora.r
    gen = torch.Generator().manual_seed(9)
    with torch.no_grad():
        lora.Bq[:, :, :r] = (torch.randn(lora.L, lora.d, r, generator=gen) * 0.05).to(BF).cuda()
        lora.Bk[:, :, r:2 * r] = (torch.randn(lora.L, lora.d, r, generator=gen) * 0.05).to(BF).cuda()
    sd0 = om.state_dict_fp32(model)
    tr = AdapterTrainer(model, lr=1e-3, encoder_lora=lora)
    loss = tr.forward_backward(audio_values=mel, **batch)
    sd = dict(sd0)
    l2 = "multi_modal_projector.linear_2.weight"
    sd[l2] = sd0[l2].clone().requires_grad_(True)
    Aq = lora.A[0, :r].float().cpu().requires_grad_(True)
    Ak = lora.A[0, r:2 * r].float().cpu().requires_grad_(True)
    Bq = lora.Bq[0, :, :r].float().cpu().requires_grad_(True)
    Bk = lora.Bk[0, :, r:2 * r].float().cpu().requires_grad_(True)
    p = "audio_tower.layers.0.self_attn."
    sd[p + "q_proj.weight"] = sd0[p + "q_proj.weight"] + lora.scaling * (Bq @ Aq)
    sd[p + "k_proj.weight"] = sd0[p + "k_proj.weight"] + lora.scaling * (Bk @ Ak)
    _, ref_loss = om.forward(sd, om.shapes_from_config(cfg), batch["input_ids"], mel.cpu().to(BF).float(),
                             batch["audio_token_start_idx"], batch["audio_lens"], batch["audio_token_len"], batch["audio_batch_size"],
                             labels=labels)
    ref_loss.backward()
    assert abs(float(loss) - float(ref_loss)) < 3e-2 * max(1.0, abs(float(ref_loss)))
    for name, got, want in (("Aq", lora.gA[0, :r], Aq.grad), ("Ak", lora.gA[0, r:2 * r], Ak.grad), ("Bq", lora.gBq[0, :, :r], Bq.grad),
                            ("Bk", lora.gBk[0, :, r:2 * r], Bk.grad), ("linear_2", tr.grad_view("linear_2"), sd[l2].grad)):
        got = got.float().cpu()
        cos = float(F.cosine_similarity(got.double().flatten(), want.double().flatten(), dim=0))
        rl = rel(got, want)
        print(f"encoder LoRA at width: {name} rel {rl:.3e} cos {cos:.5f}")
        assert cos > 0.995 and rl < 8e-2, (name, cos, rl)
