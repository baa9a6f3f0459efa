"""Per-op parity of the prefill / encoder forward kernels at the widths, lengths and masks inference runs (DESIGN section 5).

Every kernel between the waveform and the first logits is called through ``ops`` (or ``_lib.AttnArgs`` where ``ops`` has no
door) on seeded bf16 inputs and compared with plain fp32 / fp64 math of the same operation, at the Whisper-large-v3 (d 1280,
20 heads of 64, 128 mel, T = 3000 -> 1500), Llama-3.1-8B (d 4096, 32 / 8 heads of 128, ffn 14336, V 128256) and Llama-3.3-70B
(64 / 8 heads of 128) widths:

* attention forward on the wgmma kernel (``attn_wg_kernel``) - the encoder form (key lengths, block-causal streaming mask), the
  causal prefill with left padding and a right-side key length, and the prefill on a KV cache with ``model.py``'s strides -
  per query row against fp32 softmax, per element against a reference that copies the kernel's roundings, bit-level mask /
  batch / head isolation checks, and the same call on the mma.sync kernel (``attn_fwd_kernel``);
* RoPE (``pos_offset``, explicit ``positions`` of a left-padded batch) and the prefill cache fill (``uvx_kv_write``);
* the conv stem (per element, the frames where the padding enters named) and the log-mel (silence, sub-window, full-scale and
  mixed-length batches);
* LayerNorm, RMSNorm, StackAudioFrames + RMSNorm, SwiGLU and embed + splice at width with the strides the model passes.

Bounds ("ulp" is the spacing of bf16 at the reference value, u = 2^-24, gamma(n) = n u / (1 - n u); the observed maxima were
measured on an H100 80GB HBM3 at a 700 W power limit and stand next to each bound):

* attention vs fp32 softmax: the relative error of each (batch, head, query) row of D outputs is below ``ROW_REL``.  The output
  is rounded to bf16 (2^-9 per element) and P is rounded to bf16 before P V (2^-9 per key, averaging out over the keys), so a
  row with few visible keys is the worst case;
* attention vs the rounding-matched reference: per element within ``MATCH_K`` * (ulp + 2^-11 sum_j p_j |v_j|).  The reference
  rounds P where the kernel does, so what is left is the final rounding flipping (1 ulp) and entries of P flipping to the next
  bf16 (each 2^-8 p_j |v_j|) where exp2f and the tensor-core summation order differ from torch's by an fp32 ulp;
* masks, batch and head isolation: bit-identical outputs; rows that see no key are exactly zero and their ``lse`` is -inf;
* RoPE: one ulp + 2^-23 (|x1 c| + |x2 s|) of the fp64 rotation with the same fp32 tables (the kernel rounds each product and
  the sum to fp32, then the result to bf16); observed 0.50 of the bound;
* conv stem: ulp + 1.13 gamma(3 Cin + 2) sum |x w| (fp32 accumulation in any order; GELU's slope is below 1.13) + 2^-20 of
  the terms the epilogue adds in fp32; observed 0.50 of the bound (conv1), 0.38 (conv2);
* LayerNorm: half an ulp + ``LN_F32`` * (|x - mean| rstd |w| + |b|) + 2^-23 |mean| rstd |w|: the kernel is two-pass in fp32,
  so beyond the final rounding only the fp32 rounding of the arithmetic and of the mean itself (half an fp32 ulp of |mean|,
  which x - mean inherits whatever its size) is left; observed 0.21 of the fp32 term; a one-pass variance
  E[x^2] - mean^2 is outside it at mean 30;
* RMSNorm / SwiGLU: HF rounds twice (the normalised value, then the product); where the kernel's fp32 intermediate lands on the
  other side of a bf16 boundary the result moves by that ulp times the second factor - allowed on at most 1e-3 of the entries (observed at most 4.2e-5);
* log-mel: DESIGN section 5's 2e-3 abs / 1e-4 rms against the float64 oracle (observed 1.7e-5 / 1.9e-7); the bf16 image is the fp32 result rounded;
* embed + splice, cache fill: bit-exact."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
U32 = 2.0 ** -24

ROW_REL = 8e-3      # observed at most 3.85e-3 (every attention case here), 5.36e-3 with the edge value rows x1024
MATCH_K = 8.0       # observed at most 3.18
LN_F32 = 2.0 ** -20


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
    """Seeded bf16 normal values generated on the GPU."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale + mean).to(BF)


def bf16_ulp(ref: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 (8 significant bits) at |ref| (0 at ref == 0)."""
    _, e = torch.frexp(ref)
    ulp = torch.ldexp(torch.ones_like(ref), (e - 8).to(torch.int32))
    return torch.where(ref == 0, torch.zeros_like(ulp), ulp)


def assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError(f"{what}: {int(bad.sum())} entries out of bound; first at flat {i}: got "
                             f"{float(got.reshape(-1)[i])!r} ref {float(ref.reshape(-1)[i])!r} bound {float(bound.reshape(-1)[i])!r}")


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound over the entries with a non-zero bound (what a run prints next to its bound)."""
    err = (got.double() - ref.double()).abs()
    ok = bound > 0
    return float((err[ok] / bound[ok]).max()) if bool(ok.any()) else 0.0


def gamma(n):
    return n * U32 / (1 - n * U32)


def i32(v):
    return None if v is None else torch.tensor(list(v), dtype=torch.int32, device="cuda")


# ================================================================================================ 1. attention forward
class AttnCase:
    """One attention call in one of the three forms inference uses, with its inputs.

    ``enc``: ``ops.attention_encoder_tc`` over the fused [B*S, 3*H*64] projection; ``fused``: ``ops.attention_fused_qkv`` over
    [B*S, (Hq + 2 Hkv) D]; ``cache``: ``ops.attention`` with q from the fused rows and k / v from caches [B, S_max, Hkv, D],
    Skv = past + Sq < S_max (model.py ``llama_hidden`` with a cache).  ``lens`` / ``starts`` are kv_len / kv_start per batch
    element (None = not passed)."""

    def __init__(self, form, B, Sq, Hq, Hkv, D, causal=False, past=0, lens=None, starts=None, block=0, seed=0):
        assert form in ("enc", "fused", "cache") and (past == 0 or form == "cache")
        self.form, self.B, self.Sq, self.Hq, self.Hkv, self.D = form, B, Sq, Hq, Hkv, D
        self.causal, self.past, self.lens, self.starts, self.block = causal, past, lens, starts, block
        self.Skv = past + Sq
        self.rows = self.Skv + 37 if form == "cache" else self.Skv        # key rows that exist in memory (S_max for a cache)
        self.scale = D ** -0.5
        self.W = (Hq + 2 * Hkv) * D
        self.lens_t, self.starts_t = i32(lens), i32(starts)
        self.end = [self.Skv if lens is None else max(0, min(self.Skv, lens[b])) for b in range(B)]
        self.beg = [0 if starts is None else min(max(starts[b], 0), self.end[b]) for b in range(B)]
        st = {"qkv": rnd(B * Sq, self.W, seed=seed)}
        if form == "cache":
            st["kc"], st["vc"] = rnd(B, self.rows, Hkv, D, seed=seed + 1), rnd(B, self.rows, Hkv, D, seed=seed + 2)
        self.st = st

    def clone(self, st=None):
        return {k: v.clone() for k, v in (st or self.st).items()}

    def qkv_views(self, st):
        """q [B, Sq, Hq, D], k / v [B, rows, Hkv, D] as views into the storage."""
        t = st["qkv"].view(self.B, self.Sq, self.Hq + 2 * self.Hkv, self.D)
        if self.form == "cache":
            return t[:, :, :self.Hq], st["kc"], st["vc"]
        return t[:, :, :self.Hq], t[:, :, self.Hq:self.Hq + self.Hkv], t[:, :, self.Hq + self.Hkv:]

    def run(self, st=None, lse=False):
        """-> out [B, Sq, Hq, D] (and lse [B, Hq, Sq] through the argument struct, which is the only door to it)."""
        from ultravox_b200 import ops
        st = st or self.st
        B, Sq, Hq, Hkv, D, qkv = self.B, self.Sq, self.Hq, self.Hkv, self.D, st["qkv"]
        out = torch.full((B * Sq, Hq * D), 7.0, dtype=BF, device="cuda")
        if lse:
            return self._raw(st, out)
        if self.form == "enc":
            assert not self.causal and Hq == Hkv and D == 64
            ops.attention_encoder_tc(qkv, B, Sq, Hq, self.scale, self.lens_t, self.block, out=out)
        elif self.form == "fused":
            ops.attention_fused_qkv(qkv, B, Sq, Hq, Hkv, D, self.scale, self.causal, self.lens_t, self.block, out=out, kv_start=self.starts_t)
        else:
            rs, cs = qkv.stride(0), self.rows * Hkv * D
            ops.attention(qkv.data_ptr(), st["kc"].data_ptr(), st["vc"].data_ptr(), out, B, Hq, Hkv, Sq, self.Skv, D,
                          (rs, Sq * rs, Hkv * D, cs, Hkv * D, cs, Hq * D, Sq * Hq * D), self.scale, self.causal, self.lens_t, self.block,
                          self.starts_t)
        return out.view(B, Sq, Hq, D)

    def _raw(self, st, out):
        from ultravox_b200._lib import AttnArgs, check, lib
        B, Sq, Hq, Hkv, D, qkv = self.B, self.Sq, self.Hq, self.Hkv, self.D, st["qkv"]
        rs, base = qkv.stride(0), qkv.data_ptr()
        a = AttnArgs()
        a.q, a.o = base, out.data_ptr()
        a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, Sq, self.Skv, D
        if self.form == "cache":
            cs = self.rows * Hkv * D
            a.k, a.v = st["kc"].data_ptr(), st["vc"].data_ptr()
            strides = (rs, Sq * rs, Hkv * D, cs, Hkv * D, cs, Hq * D, Sq * Hq * D)
        else:
            a.k, a.v = base + 2 * Hq * D, base + 2 * (Hq + Hkv) * D
            strides = (rs, Sq * rs, rs, Sq * rs, rs, Sq * rs, Hq * D, Sq * Hq * D)
        (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = strides
        a.kv_len = None if self.lens_t is None else self.lens_t.data_ptr()
        a.kv_start = None if self.starts_t is None else self.starts_t.data_ptr()
        a.causal, a.block, a.scale = int(self.causal), self.block, self.scale
        lse = torch.full((B, Hq, Sq), 7.0, dtype=torch.float32, device="cuda")
        a.lse = lse.data_ptr()
        check(lib().uvx_attention(C.byref(a), torch.cuda.current_stream().cuda_stream), "uvx_attention")
        return out.view(B, Sq, Hq, D), lse

    def mask(self, b):
        """[Sq, Skv] bool: query i of batch element b sees key j."""
        i = torch.arange(self.Sq, device="cuda")[:, None]
        j = torch.arange(self.Skv, device="cuda")[None, :]
        m = (j >= self.beg[b]) & (j < self.end[b]) & (i >= 0)
        if self.causal:
            m = m & (j <= i + (self.Skv - self.Sq))
        if self.block > 0:
            m = m & (j // self.block <= i // self.block)
        return m

    def refs(self, st, b, matched=True):
        """For batch element b: (a) fp32 softmax(q k^T scale) v, (b) the rounding-matched reference (bf16) and sum_j p_j |v_j|,
        each [Sq, Hq, D].  (b) walks the kernel's 64-key tiles with a running max, rounds P to bf16 before P V, sums l on the
        unrounded P and rounds the output once; a tile wholly masked for a row leaves that row's state unchanged, so walking
        every tile from 0 is the kernel's walk over the tiles it loads."""
        Sq, Skv, Hq, Hkv, D = self.Sq, self.Skv, self.Hq, self.Hkv, self.D
        G = Hq // Hkv
        q, k, v = self.qkv_views(st)
        q = q[b].float().permute(1, 0, 2).reshape(Hkv, G, Sq, D)
        k = k[b, :Skv].float().permute(1, 0, 2)[:, None]                       # [Hkv, 1, Skv, D]
        v = v[b, :Skv].float().permute(1, 0, 2)[:, None]
        ok = self.mask(b)
        s = (q @ k.transpose(-1, -2)).masked_fill(~ok, float("-inf"))          # unscaled, fp32
        scale = torch.tensor(self.scale, dtype=torch.float32)
        p = torch.softmax(s * scale, -1).nan_to_num(0.0)

        def flat(t):
            return t.permute(2, 0, 1, 3).reshape(Sq, Hq, D)
        ref, mag = flat(p @ v), flat(p @ v.abs())
        del p
        if not matched:
            return ref, None, mag
        sl2 = float(scale * torch.tensor(1.4426950408889634, dtype=torch.float32))
        m = torch.full(s.shape[:-1], float("-inf"), device="cuda")
        l = torch.zeros_like(m)
        o = torch.zeros(*s.shape[:-1], D, device="cuda")
        for t0 in range(0, Skv, 64):
            stile = s[..., t0:t0 + 64]
            m_new = torch.maximum(m, stile.amax(-1))
            mref = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
            corr = torch.exp2((m - mref) * sl2)
            m = m_new
            pt = torch.exp2((stile - mref[..., None]) * sl2)
            l = l * corr + pt.sum(-1)
            o = o * corr[..., None] + pt.to(BF).float() @ v[..., t0:t0 + 64, :]
        inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
        return ref, flat((o * inv[..., None]).to(BF)), mag

    def outside(self, b):
        """[rows] bool: key rows of batch element b that no query may read (left padding, kv_len on, the cache tail)."""
        j = torch.arange(self.rows, device="cuda")
        return (j < self.beg[b]) | (j >= self.end[b])

    def poisoned(self, kind):
        """A copy of the inputs with every key / value row outside the visible set replaced: ``finite`` +-1e30, ``nonfinite``
        NaN / +Inf / -Inf."""
        st = self.clone()
        _, k, v = self.qkv_views(st)
        vals = torch.tensor([1e30, -1e30, 3e38] if kind == "finite" else [float("nan"), float("inf"), float("-inf")], device="cuda").to(BF)
        j = torch.arange(self.rows, device="cuda")
        for b in range(self.B):
            out = self.outside(b)
            k[b, out] = vals[j[out] % 3][:, None, None].expand(-1, self.Hkv, self.D)
            v[b, out] = vals[(j[out] + 1) % 3][:, None, None].expand(-1, self.Hkv, self.D)
        return st

    def beacons(self):
        """A copy of the inputs whose first and last visible value rows (and, under a block mask, the first and last key of the
        block holding the last visible key) are 1024 times larger: a kernel that drops one of them is off by far more than the
        fp32 bound in every row that sees it."""
        st = self.clone()
        _, _, v = self.qkv_views(st)
        for b in range(self.B):
            if self.end[b] > self.beg[b]:
                keys = {self.beg[b], self.end[b] - 1}
                if self.block > 0:
                    e = self.end[b] - 1
                    keys |= {max(self.beg[b], e // self.block * self.block), max(self.beg[b], e // self.block * self.block - 1)}
                for key in keys:
                    v[b, key] = v[b, key] * 1024
        return st


def row_rel(got, ref):
    """[Sq, Hq] relative error of each output row of D values (rows whose reference is 0 give 0 where got is 0, inf otherwise)."""
    num = (got.double() - ref.double()).norm(dim=-1)
    den = ref.double().norm(dim=-1)
    return torch.where(den > 0, num / den.clamp_min(1e-300), torch.where(num > 0, torch.full_like(num, float("inf")), num))


def compare_with_refs(c, st, out, what, matched=True):
    """Per-row error vs fp32 softmax and per-element error vs the rounding-matched reference, per batch element; rows that see
    no key are exactly zero.  Returns the observed maxima (row rel, matched ratio)."""
    w32 = wm = 0.0
    for b in range(c.B):
        ref, mt, mag = c.refs(st, b, matched)
        seen = c.mask(b).any(-1)                                              # [Sq]
        assert int(torch.count_nonzero(out[b][~seen])) == 0, (what, b, "a query that sees no key must give exactly 0")
        rr = row_rel(out[b], ref)
        w32 = max(w32, float(rr.max()))
        if not bool((rr < ROW_REL).all()):
            i, h = [int(x) for x in torch.nonzero(~(rr < ROW_REL))[0]]
            raise AssertionError(f"{what}: batch {b} query {i} head {h}: row rel {float(rr[i, h]):.3e} vs fp32 softmax (bound {ROW_REL})")
        if matched:
            unit = bf16_ulp(mt.double()) + 2.0 ** -11 * mag.double()
            wm = max(wm, worst_ratio(out[b], mt, unit))
            assert_within(out[b], mt.double(), MATCH_K * unit, f"{what}: batch {b} vs rounding-matched")
    return w32, wm


def check_attention(c, what, both_kernels=True):
    from ultravox_b200 import _lib
    out = c.run()
    assert torch.equal(out, c.run()), (what, "two runs differ")
    w32, wm = compare_with_refs(c, c.st, out, what)
    # what the mask hides cannot move a bit
    for kind in ("finite", "nonfinite"):
        assert torch.equal(c.run(c.poisoned(kind)), out), (what, f"reads a masked key / value row ({kind} garbage)")
    # what the mask shows at its edges must arrive
    stb = c.beacons()
    wb, _ = compare_with_refs(c, stb, c.run(stb), what + " (edge keys x1024)", matched=False)
    wk = 0.0
    if both_kernels:
        _lib.lib().uvx_debug_attn_tc(0)
        try:
            out_mma = c.run()
            assert torch.equal(c.run(c.poisoned("nonfinite")), out_mma), (what, "mma.sync reads a masked key / value row")
        finally:
            _lib.lib().uvx_debug_attn_tc(-1)
        for b in range(c.B):
            seen = c.mask(b).any(-1)
            assert int(torch.count_nonzero(out_mma[b][~seen])) == 0, (what, b, "mma.sync: a query that sees no key must give 0")
            rr = row_rel(out[b][seen], out_mma[b][seen].float())
            wk = max(wk, float(rr.max()) if rr.numel() else 0.0)
        assert wk < ROW_REL, (what, "wgmma vs mma.sync per row", wk)      # observed 0: the two kernels agree bit for bit today
    print(f"{what}: row rel vs fp32 {w32:.3e} (edge keys x1024 {wb:.3e}), matched ratio {wm:.2f}, wgmma vs mma.sync row rel {wk:.3e}")
    return out


def _enc_cases():
    cs = {}
    for S, B, lens in [(1500, 1, None), (1500, 3, [1499, 1500, 1]), (1500, 3, [63, 64, 65]), (1500, 3, [1500, 0, 777]),
                       (750, 1, None), (750, 3, [750, 65, 749]), (77, 1, None), (77, 3, [77, 1, 64]), (64, 1, None), (64, 3, [64, 63, 1]),
                       (63, 1, None), (63, 3, [63, 62, 1]), (16, 1, None), (16, 3, [16, 1, 15])]:
        cs[f"S{S}_B{B}_" + ("full" if lens is None else "len" + "-".join(map(str, lens)))] = dict(S=S, B=B, lens=lens)
    return cs


ENC_CASES = _enc_cases()


@pytest.mark.parametrize("case", list(ENC_CASES))
def test_attention_encoder(case):
    """Whisper-large's encoder attention (20 heads of 64, non-causal) through ``ops.attention_encoder_tc``: S = 1500 down to one
    16-query tile, per-clip key lengths at 1, 63 / 64 / 65, S - 1 and S (at S = 1500 keys 1498 and 1499 differ in visibility
    between clips) and a clip with no key at all."""
    p = ENC_CASES[case]
    c = AttnCase("enc", p["B"], p["S"], 20, 20, 64, lens=p["lens"], seed=p["S"] + p["B"])
    check_attention(c, "encoder " + case)


STREAM_LENS = {100: [1500, 250], 64: [1473, 640], 50: [1500, 49], 25: [1238, 1475], 1500: [1500, 700]}


@pytest.mark.parametrize("block", list(STREAM_LENS))
def test_attention_encoder_streaming(block):
    """The block-causal streaming mask (query i sees keys j with j / block <= i / block) at S = 1500, B = 2, with block sizes
    that fall inside 64-key tiles at 64-query tile boundaries (100, 50, 25), on them (64) and one block for the whole clip; one
    clip's key length ends inside a block, the other's on a block edge."""
    c = AttnCase("enc", 2, 1500, 20, 20, 64, lens=STREAM_LENS[block], block=block, seed=block)
    check_attention(c, f"encoder streaming block={block} lens={STREAM_LENS[block]}")


def _prefill_cases():
    cs = {}
    for heads, (Hq, Hkv) in (("8b", (32, 8)), ("70b", (64, 8))):
        for S in (201, 640, 64, 65):
            if heads == "70b" and S == 640:
                continue
            ok = [x for x in (0, 1, 63, 64, 65, 128, S - 1) if x < S]
            # B = 1: no padding; one start alone; one start with a right-side kv_len
            cs[f"{heads}_S{S}_B1_plain"] = dict(Hq=Hq, Hkv=Hkv, S=S, B=1, starts=None, lens=None)
            if heads == "8b":
                cs[f"{heads}_S{S}_B1_start{ok[-2]}"] = dict(Hq=Hq, Hkv=Hkv, S=S, B=1, starts=[ok[-2]], lens=None)
                cs[f"{heads}_S{S}_B1_start{min(63, S - 2)}_len{S - 1}"] = dict(Hq=Hq, Hkv=Hkv, S=S, B=1, starts=[min(63, S - 2)], lens=[S - 1])
            # B = 4: the starts in two groups of four, alone and with kv_len < S
            a, b_ = ok[:4], (ok[4:] + ok[:4])[:4]
            cs[f"{heads}_S{S}_B4_starts{'-'.join(map(str, a))}"] = dict(Hq=Hq, Hkv=Hkv, S=S, B=4, starts=a, lens=None)
            lens = [min(S, max(s + 1, S - d)) for s, d in zip(b_, (3, 0, 1, S // 3))]
            cs[f"{heads}_S{S}_B4_starts{'-'.join(map(str, b_))}_lens{'-'.join(map(str, lens))}"] = dict(Hq=Hq, Hkv=Hkv, S=S, B=4, starts=b_, lens=lens)
    return cs


PREFILL_CASES = _prefill_cases()


@pytest.mark.parametrize("case", list(PREFILL_CASES))
def test_attention_prefill(case):
    """The Llama prefill (causal GQA, head_dim 128, 32 / 8 and 64 / 8 heads) through ``ops.attention_fused_qkv`` as model.py
    ``llama_hidden`` calls it without a cache: left padding ``kv_start`` at 0, 1, 63, 64, 65, 128 and S - 1, alone and together
    with a right-side ``kv_len`` < S.  Queries inside the left padding see no key and give exactly zero."""
    p = PREFILL_CASES[case]
    c = AttnCase("fused", p["B"], p["S"], p["Hq"], p["Hkv"], 128, causal=True, lens=p["lens"], starts=p["starts"], seed=p["S"] + 7 * p["B"])
    check_attention(c, "prefill " + case)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("past", [1, 63, 300, 4000])
@pytest.mark.parametrize("Sq", [64, 70, 201])
def test_attention_prefill_on_cache(Sq, past, B):
    """A conversation turn prefilled on a KV cache (model.py ``llama_hidden`` with a cache): Sq new queries over past + Sq keys
    read from caches [B, S_max, Hkv, D] with S_max = Skv + 37, causal with shift = past > 0; at B = 3 each row has its own
    ``kv_start`` (up to past) and ``kv_len`` (up to Skv).  The cache tail [Skv, S_max) holds NaN / Inf in the poisoned runs."""
    Skv = past + Sq
    Hq, Hkv = (64, 8) if (Sq, past) == (70, 300) else (32, 8)
    starts = None if B == 1 else [0, min(past, 64), min(past, 130)]
    lens = None if B == 1 else [Skv, Skv - 1, Skv - Sq // 2]
    c = AttnCase("cache", B, Sq, Hq, Hkv, 128, causal=True, past=past, lens=lens, starts=starts, seed=Sq + past + B)
    out = check_attention(c, f"cache prefill Sq={Sq} past={past} B={B} heads={Hq}/{Hkv} starts={starts} lens={lens}")
    # causality, bit-exact: key past + i0 reaches no query before i0 and does reach query i0
    i0 = Sq // 3
    st = c.clone()
    st["kc"][:, past + i0], st["vc"][:, past + i0] = rnd(B, Hkv, 128, seed=3), rnd(B, Hkv, 128, seed=4)
    o2 = c.run(st)
    assert torch.equal(o2[:, :i0], out[:, :i0]), "a query sees a later key"
    assert not torch.equal(o2[0, i0], out[0, i0])


@pytest.mark.parametrize("form", ["cache", "fused"])
def test_attention_eligibility_edge(form):
    """The two sides of ``attn_wg_eligible``: Sq = 16 runs on the wgmma kernel, Sq = 15 on the mma.sync kernel.  With the same
    data (the first 15 queries, the same keys: causal, so query i sees the same keys in both calls) the two agree per row, and
    the Sq = 15 side passes the same reference, mask and edge-key checks."""
    B, Hq, Hkv, D = 3, 32, 8, 128
    past = 137 if form == "cache" else 0
    c16 = AttnCase(form, B, 16, Hq, Hkv, D, causal=True, past=past, starts=[0, 5, 2 if form == "fused" else 64],
                   lens=[past + 16, past + 15, past + 9], seed=16)
    c15 = AttnCase(form, B, 15, Hq, Hkv, D, causal=True, past=past, starts=c16.starts, lens=c16.lens, seed=16)
    c15.st["qkv"] = c16.st["qkv"].view(B, 16, -1)[:, :15].reshape(B * 15, -1).contiguous()
    if form == "cache":
        c15.st["kc"], c15.st["vc"] = c16.st["kc"][:, :c15.rows].contiguous(), c16.st["vc"][:, :c15.rows].contiguous()
    o16 = check_attention(c16, f"eligibility {form} Sq=16")
    o15 = check_attention(c15, f"eligibility {form} Sq=15", both_kernels=False)
    worst = 0.0
    for b in range(B):
        seen = c15.mask(b).any(-1)
        assert torch.equal(seen, c16.mask(b).any(-1)[:15])
        worst = max(worst, float(row_rel(o15[b][seen], o16[b, :15][seen].float()).max()))
    print(f"eligibility {form}: Sq=15 (mma.sync) vs Sq=16 (wgmma) row rel {worst:.3e}")
    assert worst < ROW_REL, worst


@pytest.mark.parametrize("form,Hq,Hkv", [("enc", 20, 20), ("fused", 32, 8), ("fused", 64, 8), ("cache", 32, 8)])
def test_attention_batch_and_head_isolation(form, Hq, Hkv):
    """New q / k / v for batch element b change only element b's output bits; new k / v for KV head g change the query heads of
    group g, every one of them, and no other head."""
    D = 64 if form == "enc" else 128
    B, Sq = 3, 140
    past = 75 if form == "cache" else 0
    c = AttnCase(form, B, Sq, Hq, Hkv, D, causal=form != "enc", past=past, lens=[past + 140, past + 101, past + 90],
                 starts=None if form == "enc" else [0, 3, 64 if form == "fused" else 70], seed=5)
    out = c.run()
    G = Hq // Hkv
    for b in range(B):
        st = c.clone()
        q, k, v = c.qkv_views(st)
        q[b], k[b], v[b] = rnd(*q[b].shape, seed=10 + b), rnd(*k[b].shape, seed=20 + b), rnd(*v[b].shape, seed=30 + b)
        o2 = c.run(st)
        for b2 in range(B):
            assert torch.equal(o2[b2], out[b2]) == (b2 != b), (form, "batch isolation", b, b2)
    for g in (0, Hkv // 2, Hkv - 1):
        st = c.clone()
        _, k, v = c.qkv_views(st)
        k[:, :, g], v[:, :, g] = rnd(B, c.rows, D, seed=40 + g), rnd(B, c.rows, D, seed=50 + g)
        o2 = c.run(st)
        for h in range(Hq):
            assert torch.equal(o2[:, :, h], out[:, :, h]) == (h // G != g), (form, "head isolation", g, h)


@pytest.mark.parametrize("kernel", ["wgmma", "mma.sync"])
def test_attention_empty_rows_and_lse(kernel):
    """Rows that see no key - queries inside the left padding (causal) and every query of a sequence with kv_len == 0 - write an
    output of exactly 0 and lse = -inf (log of an empty sum), on both kernels; every other row's lse is the log-sum-exp of its
    scaled visible scores."""
    from ultravox_b200 import _lib
    c = AttnCase("fused", 4, 130, 32, 8, 128, causal=True, starts=[0, 64, 129, 17], lens=[130, 130, 130, 0], seed=9)
    _lib.lib().uvx_debug_attn_tc(0 if kernel == "mma.sync" else -1)
    try:
        out, lse = c.run(lse=True)
    finally:
        _lib.lib().uvx_debug_attn_tc(-1)
    q, k, _ = c.qkv_views(c.st)
    for b in range(c.B):
        m = c.mask(b)
        seen = m.any(-1)
        assert int(seen.sum()) == [130, 66, 1, 0][b]
        assert int(torch.count_nonzero(out[b][~seen])) == 0, (b, "output of an empty row")
        assert bool((lse[b][:, ~seen] == float("-inf")).all()), (b, "lse of an empty row", lse[b][:, ~seen])
        s = (q[b].float().permute(1, 0, 2) @ k[b].float().permute(1, 0, 2).repeat_interleave(4, 0).transpose(-1, -2)) * c.scale
        want = torch.logsumexp(s.masked_fill(~m, float("-inf")), -1)
        assert torch.allclose(lse[b][:, seen], want[:, seen], atol=2e-3, rtol=1e-3), (b, float((lse[b][:, seen] - want[:, seen]).abs().max()))


# ================================================================================================ 2. RoPE and the prefill cache fill
def _llama3_tables():
    from ultravox_b200 import ops
    from ultravox_b200.config import PRESETS
    tc = PRESETS["v0_5_8b"]["text_config"]
    inv = ops.llama3_inv_freq(128, tc["rope_theta"], tc["rope_scaling"])
    return ops.rope_tables(inv, 131072, "cuda")


def rope_ref(qkv0, Hq, Hkv, D, cos, sin, pos):
    """fp64 rotation of the q and k heads of bf16 rows [R, W] with the fp32 tables at pos [R]; (ref, bound) over the first
    (Hq + Hkv) D columns: one ulp + 2^-23 (|x1 c| + |x2 s|)."""
    R, nr = qkv0.shape[0], (Hq + Hkv) * D
    h = qkv0[:, :nr].to(F64).view(R, Hq + Hkv, D)
    c, s = cos[pos.long()].to(F64)[:, None], sin[pos.long()].to(F64)[:, None]
    x1, x2 = h[..., :D // 2], h[..., D // 2:]
    ref = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).view(R, nr)
    cancel = torch.cat([(x1 * c).abs() + (x2 * s).abs(), (x2 * c).abs() + (x1 * s).abs()], -1).view(R, nr)
    return ref, bf16_ulp(ref) + 2.0 ** -23 * cancel


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("heads", ["8b", "70b"])
def test_rope_offsets_and_positions(heads, B):
    """``ops.rope_`` (the yardstick of the fused-RoPE GEMM epilogues) at head_dim 128 with the llama3-scaled tables, S = 201, on
    rows that are a column view of a wider buffer: ``pos_offset`` in {0, 37, 8191, 131071 - S} (row r of every sequence is at
    pos_offset + r % S), and the explicit ``positions`` of a left-padded batch as ``generate`` derives them from the attention
    mask, (cumsum(mask) - 1).clamp_min(0): a pad row is at position 0, where cos = 1 and sin = 0, so it comes back bit for bit.
    The V section and the buffer outside the view keep their bits; one sequence's rows do not depend on another's."""
    from ultravox_b200 import ops
    Hq, Hkv = (32, 8) if heads == "8b" else (64, 8)
    D, S = 128, 201
    W, nr = (Hq + 2 * Hkv) * D, (Hq + Hkv) * D
    cos, sin = _llama3_tables()
    buf0 = rnd(B * S, W + 16, scale=2.0, seed=B + Hq)
    worst = 0.0
    for off in (0, 37, 8191, 131071 - S):
        buf = buf0.clone()
        ops.rope_(buf[:, 8:8 + W], Hq, Hkv, D, cos, sin, rows_per_seq=S, pos_offset=off)
        pos = off + torch.arange(B * S, device="cuda") % S
        ref, bound = rope_ref(buf0[:, 8:8 + W], Hq, Hkv, D, cos, sin, pos)
        worst = max(worst, worst_ratio(buf[:, 8:8 + nr], ref, bound))
        assert_within(buf[:, 8:8 + nr], ref, bound, f"rope {heads} B={B} pos_offset={off}")
        assert torch.equal(buf[:, 8 + nr:], buf0[:, 8 + nr:]) and torch.equal(buf[:, :8], buf0[:, :8]), "V section / outside the view changed"
    print(f"rope {heads} B={B}: max err / bound {worst:.3f}")
    # left-padded batch
    pads = [0, 64, 200][:B]
    am = torch.ones(B, S, dtype=torch.int64, device="cuda")
    for b, p in enumerate(pads):
        am[b, :p] = 0
    positions = (am.cumsum(-1) - 1).clamp_min(0).to(torch.int32).reshape(-1).contiguous()
    buf = buf0.clone()
    ops.rope_(buf[:, 8:8 + W], Hq, Hkv, D, cos, sin, rows_per_seq=S, pos_offset=999, positions=positions)   # positions win over pos_offset
    ref, bound = rope_ref(buf0[:, 8:8 + W], Hq, Hkv, D, cos, sin, positions)
    assert_within(buf[:, 8:8 + nr], ref, bound, f"rope {heads} B={B} positions")
    assert torch.equal(buf[:, 8 + nr:], buf0[:, 8 + nr:]) and torch.equal(buf[:, :8], buf0[:, :8])
    for b, p in enumerate(pads):
        assert torch.equal(buf[b * S:b * S + p + 1], buf0[b * S:b * S + p + 1]), (b, "pad rows and the first token are at position 0: unchanged")
        if p + 1 < S:
            assert not torch.equal(buf[b * S + p + 1, 8:8 + nr], buf0[b * S + p + 1, 8:8 + nr])
    if B > 1:
        b2 = buf0.clone()
        b2[S:2 * S] = rnd(S, W + 16, seed=77)
        ops.rope_(b2[:, 8:8 + W], Hq, Hkv, D, cos, sin, rows_per_seq=S, positions=positions)
        assert torch.equal(b2[:S], buf[:S]) and torch.equal(b2[2 * S:], buf[2 * S:]) and not torch.equal(b2[S:2 * S], buf[S:2 * S])


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("past", [0, 300])
@pytest.mark.parametrize("heads", ["8b", "70b"])
def test_kv_write_fills_the_cache(heads, past, B):
    """``ops.rope_`` then ``ops.kv_write`` in model.py's order, S = 201 rows per sequence into caches [B, S_max, Hkv, 128] with
    S_max = past + S + 11 filled with a position-dependent sentinel: cache rows [past, past + S) are the rotated K section and
    the raw V section bit for bit, and every other cache element keeps its sentinel."""
    from ultravox_b200 import ops
    Hq, Hkv = (32, 8) if heads == "8b" else (64, 8)
    D, S = 128, 201
    smax = past + S + 11
    cos, sin = _llama3_tables()
    qkv0 = rnd(B * S, (Hq + 2 * Hkv) * D, seed=past + B)
    qkv = qkv0.clone()
    ops.rope_(qkv, Hq, Hkv, D, cos, sin, rows_per_seq=S, pos_offset=past)
    sent = ((torch.arange(B * smax * Hkv * D, device="cuda") % 251).float() - 125.0).to(BF).view(B, smax, Hkv, D)
    kc, vc = sent.clone(), (-sent).clone()
    ops.kv_write(qkv, kc, vc, B, S, past, Hq, Hkv, D)
    t = qkv.view(B, S, Hq + 2 * Hkv, D)
    assert torch.equal(kc[:, past:past + S], t[:, :, Hq:Hq + Hkv]), "cache K != rotated K section"
    assert torch.equal(vc[:, past:past + S], t[:, :, Hq + Hkv:]), "cache V != V section"
    assert torch.equal(t[:, :, Hq + Hkv:], qkv0.view(B, S, -1, D)[:, :, Hq + Hkv:]), "RoPE touched V"
    assert not torch.equal(t[:, 1:, Hq:Hq + Hkv], qkv0.view(B, S, -1, D)[:, 1:, Hq:Hq + Hkv])
    for cch, s0 in ((kc, sent), (vc, -sent)):
        assert torch.equal(cch[:, :past], s0[:, :past]) and torch.equal(cch[:, past + S:], s0[:, past + S:]), "a row outside [past, past + S) changed"


# ================================================================================================ 3. encoder front end
@pytest.mark.parametrize("with_pos", [False, True])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("layer", ["conv1_T3000", "conv2_T3000", "conv2_T2999"])
def test_conv_stem_per_element(layer, B, with_pos):
    """Whisper-large's conv stem through ``ops.conv1d_k3``: conv1 (128 -> 1280, stride 1, into a guard-padded buffer as
    ``encode_audio`` calls it) and conv2 (1280 -> 1280, stride 2, T = 3000 and the odd T = 2999 whose last output frame reads
    the trailing guard row), per element against fp64 conv1d + exact-erf GELU (+ pos).  The frames where the padding enters
    (0, 1, Tout - 2, Tout - 1) are asserted on their own; guard rows of the output are not written; clip b does not depend on
    clip b'."""
    from ultravox_b200 import ops
    Cin, Cout, stride, T = {"conv1_T3000": (128, 1280, 1, 3000), "conv2_T3000": (1280, 1280, 2, 3000), "conv2_T2999": (1280, 1280, 2, 2999)}[layer]
    Tout = (T + stride - 1) // stride
    guard = stride == 1
    x = rnd(B, T, Cin, seed=1)
    w = rnd(Cout, Cin, 3, scale=0.03, seed=2)
    bias = rnd(Cout, scale=0.5, seed=3)
    pos = rnd(Tout, Cout, seed=4) if with_pos else None
    x_tm = torch.zeros(B, T + 2, Cin, dtype=BF, device="cuda")
    x_tm[:, 1:T + 1] = x
    w_r = w.permute(0, 2, 1).reshape(Cout, 3 * Cin).contiguous()

    def run(xt):
        out = torch.full((B, Tout + 2 * guard, Cout), -3.0, dtype=BF, device="cuda")
        ops.conv1d_k3(xt, w_r, bias, stride, out, out_guard=guard, pos=pos)
        if guard:
            assert bool((out[:, 0] == -3.0).all()) and bool((out[:, Tout + 1] == -3.0).all()), "a guard row of the output was written"
            return out[:, 1:Tout + 1]
        return out
    got = run(x_tm)
    xd, wd = x.to(F64).transpose(1, 2), w.to(F64)
    pre = F.conv1d(xd, wd, bias.to(F64), stride=stride, padding=1).transpose(1, 2)                 # [B, Tout, Cout]
    mag = F.conv1d(xd.abs(), wd.abs(), bias.to(F64).abs(), stride=stride, padding=1).transpose(1, 2)
    assert pre.shape[1] == Tout
    act = 0.5 * pre * (1.0 + torch.erf(pre / math.sqrt(2.0)))
    ref = act + (pos.to(F64) if with_pos else 0.0)
    bound = bf16_ulp(ref) + 1.13 * gamma(3 * Cin + 2) * mag + 2.0 ** -20 * (act.abs() + (pos.to(F64).abs() if with_pos else 0.0))
    print(f"conv {layer} B={B} pos={with_pos}: max err / bound {worst_ratio(got, ref, bound):.3f}, rel {rel(got, ref.to(BF)):.3e}")
    for name, t in (("frame 0", 0), ("frame 1", 1), ("frame Tout-2", Tout - 2), ("frame Tout-1", Tout - 1)):
        assert_within(got[:, t], ref[:, t], bound[:, t], f"conv {layer} B={B} {name}")
    assert_within(got, ref, bound, f"conv {layer} B={B}")
    assert rel(got, ref.to(BF)) < 1e-3
    if B > 1:
        x2 = x_tm.clone()
        x2[1, 1:T + 1] = rnd(T, Cin, seed=9)
        got2 = run(x2)
        assert torch.equal(got2[0], got[0]) and not torch.equal(got2[1], got[1]), "clip 0 depends on clip 1"


def _logmel_check(waves, n_mels=128):
    """``ops.logmel`` on the zero-padded batch vs the float64 oracle at DESIGN section 5's tolerance; the bf16 time-major image
    is the fp32 result rounded, between two zero guard rows.  -> (got [B, n_mels, T] fp32 numpy, oracle, padded)."""
    from oracle import logmel as om
    from ultravox_b200 import ops
    padded, _ = om.pad_batch(waves)
    ref = om.log_mel(padded, n_mels)
    got_t, tm = ops.logmel(torch.from_numpy(padded).cuda(), n_mels, want_f32=True, want_tm=True)
    got = got_t.cpu().numpy()
    assert got.shape == ref.shape
    err = np.abs(got - ref)
    print(f"logmel B={len(waves)} L={padded.shape[1]}: max abs {err.max():.3e}, rms {np.sqrt((err ** 2).mean()):.3e}")
    assert err.max() < 2e-3, err.max()
    assert np.sqrt((err ** 2).mean()) < 1e-4
    T = padded.shape[1] // 160
    assert torch.equal(tm[:, 1:T + 1], got_t.transpose(1, 2).to(BF)), "bf16 image != rounded fp32 result"
    assert int(torch.count_nonzero(tm[:, 0])) == 0 and int(torch.count_nonzero(tm[:, T + 1])) == 0, "guard rows"
    assert torch.equal(ops.logmel(torch.from_numpy(padded).cuda(), n_mels, want_f32=False, want_tm=True), tm)
    return got, ref, padded


def test_logmel_silence():
    """An all-zero clip, alone and beside a noise clip: every mel power is 0, log10 clamps at 1e-10 (= -10), which is the
    clip's own maximum, so every value is (-10 + 4) / 4 = -1.5, the oracle's constant (the bf16 image holds -1.5 exactly)."""
    from ultravox_b200 import ops
    noise = np.random.default_rng(1).standard_normal(16000).astype(np.float32)
    for waves in ([np.zeros(16000, np.float32)], [noise, np.zeros(9000, np.float32)]):
        got, ref, padded = _logmel_check(waves)
        assert np.all(ref[-1] == -1.5)
        assert np.abs(got[-1] + 1.5).max() <= 1e-6, np.abs(got[-1] + 1.5).max()      # log10f(1e-10f) is -10 to within an fp32 ulp
        tm = ops.logmel(torch.from_numpy(padded).cuda(), 128, want_f32=False, want_tm=True)
        assert bool((tm[-1, 1:-1] == -1.5).all())


def test_logmel_short_full_scale_and_dc():
    """A 300-sample clip (shorter than one 400-sample window) padded to a 1 s batch; a full-scale +-1.0 square wave; DC at 1.0."""
    rng = np.random.default_rng(2)
    t = np.arange(16000)
    square = np.where((t // 50) % 2 == 0, 1.0, -1.0).astype(np.float32)
    _logmel_check([rng.standard_normal(16000).astype(np.float32), rng.standard_normal(300).astype(np.float32)])
    _logmel_check([square])
    _logmel_check([np.ones(16000, np.float32)])
    _logmel_check([square, np.ones(12345, np.float32), (0.25 * square[:8000]).astype(np.float32)])


def test_logmel_short_clip_beside_30s():
    """A 0.5 s clip batched with a 30 s clip (T = 3000): the frames whose window lies inside the short clip (t <= 48: frame t
    covers samples [160 t - 200, 160 t + 200), and 49 would read past 8000, where the batch holds zeros and the lone clip its
    reflection) equal what the clip gives alone at the 2e-3 tolerance; the frames wholly past its end (t >= 52) hold the
    oracle's padding value max(-10, clipmax - 8) mapped by (x + 4) / 4, all the same number."""
    rng = np.random.default_rng(3)
    short, long_ = (0.3 * rng.standard_normal(8000)).astype(np.float32), rng.standard_normal(480000).astype(np.float32)
    both, ref, _ = _logmel_check([long_, short])
    alone, _, _ = _logmel_check([short])
    assert both.shape[2] == 3000 and alone.shape[2] == 50
    d = np.abs(both[1][:, :49] - alone[0][:, :49]).max()
    print(f"logmel short clip in a 30 s batch vs alone: max abs {d:.3e}")
    assert d < 2e-3, d
    tail = both[1][:, 52:]
    assert np.all(tail == tail[0, 0]), "the frames past the clip's end are one constant"
    assert abs(float(tail[0, 0]) - float(ref[1][0, 52])) < 1e-5 and np.all(ref[1][:, 52:] == ref[1][0, 52])


# ================================================================================================ 4. row kernels at width
def _layernorm_rows(rows, cols, seed):
    """Rows of std 1 around 0, rows of std 0.5 around 30 (the mean must be removed before the variance) and constant rows."""
    x = rnd(rows, cols, seed=seed)
    x[1::7] = rnd(x[1::7].shape[0], cols, scale=0.5, mean=30.0, seed=seed + 1)
    const = torch.tensor([2.0, -0.5, 0.0, 64.0], device="cuda").to(BF)
    x[3::97] = const[torch.arange(x[3::97].shape[0], device="cuda") % 4][:, None]
    return x


@pytest.mark.parametrize("rows,cols", [(1500, 1280), (3000, 1280), (201, 4096)])
def test_layernorm_per_element(rows, cols):
    """Whisper-large's LayerNorms (1 and 2 clips of 1500 frames x 1280: the warp-per-row kernel) and the block kernel
    (cols > 2048), on a dense input, on a strided view (row stride cols + 64) and with ``out=`` a separate buffer: per element
    within half an ulp + the fp32 term of the module docstring of fp64.  A constant row (variance 0) gives the bias exactly."""
    from ultravox_b200 import ops
    x = _layernorm_rows(rows, cols, seed=cols)
    w, b = rnd(cols, scale=0.5, mean=1.0, seed=2), rnd(cols, seed=3)
    xd = x.to(F64)
    mean = xd.mean(-1, keepdim=True)
    xn = (xd - mean) * torch.rsqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5)
    ref = xn * w.to(F64) + b.to(F64)
    rstd = torch.rsqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5)
    fp32 = LN_F32 * (xn.abs() * w.to(F64).abs() + b.to(F64).abs()) + 2.0 ** -23 * mean.abs() * rstd * w.to(F64).abs()
    bound = 0.5 * bf16_ulp(ref) + fp32
    wide = torch.full((rows, cols + 64), float("nan"), dtype=BF, device="cuda")
    wide[:, 32:32 + cols] = x
    outbuf = torch.full((rows + 2, cols), -3.0, dtype=BF, device="cuda")
    y = ops.layernorm(x, w, b, 1e-5)
    ratio = float((((y.double() - ref).abs() - 0.5 * bf16_ulp(ref)).clamp_min(0) / fp32.clamp_min(1e-30)).max())
    print(f"layernorm {rows}x{cols}: max (err - ulp/2) / fp32 term = {ratio:.3f}")
    assert_within(y, ref, bound, f"layernorm {rows}x{cols}")
    assert torch.equal(ops.layernorm(wide[:, 32:32 + cols], w, b, 1e-5), y), "strided view != dense"
    assert ops.layernorm(x, w, b, 1e-5, out=outbuf[1:rows + 1]).data_ptr() == outbuf[1].data_ptr()
    assert torch.equal(outbuf[1:rows + 1], y) and bool((outbuf[0] == -3.0).all()) and bool((outbuf[rows + 1] == -3.0).all())
    const_rows = torch.arange(3, rows, 97, device="cuda")
    assert torch.equal(y[const_rows], b[None].expand(const_rows.numel(), cols)), "a constant row must give the bias exactly"


def rmsnorm_hf(xd, w, eps):
    """LlamaRMSNorm in HF's rounding order on fp64 rows: (ref bf16, the bf16-rounded normalised value, its fp64 value)."""
    xn = xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    xb = xn.to(BF)
    return (w.to(F64) * xb.to(F64)).to(BF), xb, xn


def assert_two_roundings(got, ref, first, second, what):
    """HF's two roundings: ``got`` equals ``ref`` except where the kernel's fp32 value of ``first`` (fp64 here) lands on the other
    side of a bf16 boundary - then it is off by at most ulp(first) |second| + ulp(ref), on at most 1e-3 of the entries."""
    bound = bf16_ulp(first) * second.abs() + bf16_ulp(ref.double())
    assert_within(got, ref.double(), bound, what)
    frac = float((got != ref).float().mean())
    print(f"{what}: {frac:.2e} of the entries differ from the fp64 two-rounding reference")
    assert frac < 1e-3, (what, frac)


@pytest.mark.parametrize("rows,cols", [(201, 4096), (804, 4096), (201, 8192)])
def test_rmsnorm_per_element(rows, cols):
    """The Llama norms at 4096 (B*S = 201, 804) and 8192, eps 1e-5, LlamaRMSNorm rounding, dense and on a strided view.  An
    all-zero row gives zeros (0 * rsqrt(eps))."""
    from ultravox_b200 import ops
    x, w = rnd(rows, cols, scale=3.0, seed=cols), rnd(cols, scale=0.3, mean=1.0, seed=1)
    x[5] = 0
    ref, _, xn = rmsnorm_hf(x.to(F64), w, 1e-5)
    y = ops.rmsnorm(x, w, 1e-5)
    assert_two_roundings(y, ref, xn, w.to(F64)[None].expand_as(xn), f"rmsnorm {rows}x{cols}")
    assert int(torch.count_nonzero(y[5])) == 0 and bool(torch.isfinite(y.float()).all())
    wide = torch.full((rows, cols + 16), float("nan"), dtype=BF, device="cuda")
    wide[:, 8:8 + cols] = x
    assert torch.equal(ops.rmsnorm(wide[:, 8:8 + cols], w, 1e-5), y)


@pytest.mark.parametrize("T", [1500, 1499, 1, 7, 8, 9])
def test_stack_rmsnorm_tail(T):
    """StackAudioFrames(8) + ln_pre over [2, T, 1280] (10240 columns): the frames past T in a clip's last stacked row read as
    zeros - not as the next clip's frames, which is what lies there in memory - so those columns come out exactly 0."""
    from ultravox_b200 import ops
    N, Cc, k = 2, 1280, 8
    enc, w = rnd(N, T, Cc, seed=T), rnd(k * Cc, scale=0.3, mean=1.0, seed=2)
    rows = -(-T // k)
    st = F.pad(enc.to(F64), (0, 0, 0, rows * k - T)).reshape(N, rows, k * Cc)
    ref, _, xn = rmsnorm_hf(st, w, 1e-6)
    y = ops.stack_rmsnorm(enc, w, k, 1e-6)
    assert y.shape == ref.shape
    assert_two_roundings(y, ref, xn, w.to(F64)[None, None].expand_as(xn), f"stack_rmsnorm T={T}")
    if T % k:
        assert int(torch.count_nonzero(y[:, -1, (T % k) * Cc:])) == 0, "the padded tail of the last stacked row"
        assert int(torch.count_nonzero(y[:, -1, :(T % k) * Cc])) > 0


@pytest.mark.parametrize("rows,H,gate_first", [(201, 14336, True), (804, 14336, True), (376, 2048, False), (188, 4096, False)])
def test_swiglu_per_element(rows, H, gate_first):
    """LlamaMLP's act_fn(gate) * up at ffn 14336 (gate first) and the projector's SwiGLU (value first) at its widths, dense and
    on a strided view: silu(gate) rounded to bf16, the product rounded to bf16."""
    from ultravox_b200 import ops
    x = rnd(rows, 2 * H, scale=2.0, seed=H + rows)
    a, g = x[:, :H].to(F64), x[:, H:].to(F64)
    gate, lin = (a, g) if gate_first else (g, a)
    act = gate * torch.sigmoid(gate)
    ref = (act.to(BF).to(F64) * lin).to(BF)
    y = ops.swiglu(x, gate_first=gate_first)
    assert_two_roundings(y, ref, act, lin, f"swiglu {rows}x{H} gate_first={gate_first}")
    wide = torch.full((rows, 2 * H + 24), float("nan"), dtype=BF, device="cuda")
    wide[:, 16:16 + 2 * H] = x
    assert torch.equal(ops.swiglu(wide[:, 16:16 + 2 * H], gate_first=gate_first), y)


def test_embed_splice_at_width():
    """``ops.splice_plan`` + ``ops.embed_splice`` at V = 128256, d = 4096 against a Python loop, bit for bit: two clips in one
    sequence, a sequence with none, a clip of ``audio_token_len`` 0, a left-padded sequence (pad ids before the text, the clip's
    start index counted from the padded row) and a clip that runs to the last position; ids 0 and V - 1."""
    from ultravox_b200 import ops
    V, d, B, S, stride = 128256, 4096, 4, 96, 24
    table = rnd(V, d, scale=0.02, seed=1)
    audio = rnd(5, stride, d, seed=2)
    ids = torch.randint(0, V, (B, S), generator=torch.Generator().manual_seed(3)).cuda()
    ids[0, 0], ids[0, 1], ids[1, S - 1], ids[3, :40] = 0, V - 1, V - 1, 0
    start = torch.tensor([2, 50, 10, 45, S - 7], dtype=torch.int64, device="cuda")
    tlen = torch.tensor([24, 13, 0, 19, 7], dtype=torch.int32, device="cuda")
    per_seq = torch.tensor([2, 0, 1, 2], dtype=torch.int64, device="cuda")
    ref = table[ids].clone()
    a = 0
    for b, cnt in enumerate(per_seq.tolist()):
        for _ in range(cnt):
            s, n = int(start[a]), int(tlen[a])
            ref[b, s:s + n] = audio[a, :n]
            a += 1
    src = ops.splice_plan(start, tlen, per_seq, B, S, stride)
    want_src = torch.full((B, S), -1, dtype=torch.int32, device="cuda")
    a = 0
    for b, cnt in enumerate(per_seq.tolist()):
        for _ in range(cnt):
            s, n = int(start[a]), int(tlen[a])
            want_src[b, s:s + n] = a * stride + torch.arange(n, dtype=torch.int32, device="cuda")
            a += 1
    assert torch.equal(src.view(B, S), want_src)
    out = ops.embed_splice(ids, table, audio, src)
    assert torch.equal(out, ref)
    assert torch.equal(out[0, 0], table[0]) and torch.equal(out[0, 1], table[V - 1]) and torch.equal(out[1, S - 1], table[V - 1])
    assert torch.equal(ops.embed_splice(ids, table, None, None), table[ids])
