"""The split weight / activation ring of the prefill GEMM (gemm_tc.cu: calls one m-tile covers, one batch) against the one ring
of A + W stages (``uvx_debug_gemm_split_ring(0)``), bit for bit, the split ring forced (5 activation slots) wherever the shape
allows it, in the forms ``UltravoxModel.llama_hidden`` runs: q|k|v with the
fused RoPE, o_proj / down_proj with split-K, in-place residual and fused RMSNorm, and gate|up over the SwiGLU-interleaved image.
(q|k|v runs 128-row tiles: above 128 rows two m-tiles, so the one ring in both arms; at 100 and 128 rows the split ring.)

The split ring's A box holds round8(M) rows, so the MMAs over rows round8(M) .. MT * 128 - 1 read whatever follows the slot in
shared memory; those rows must never reach an output.  Hence M runs over the box edges 129, 200, 201, 207, 208, 209, 255, 256
(and 100, 128), A is a window of a NaN-filled buffer, the split-K workspace is NaN-filled before every call, and output /
``norm_out`` rows past M keep a sentinel.  Widths: Llama-3.1-8B and Llama-3.3-70B.  The static-weight flag (``ops.GEMM_W_STATIC``) is checked in a
graph of back-to-back flagged calls, and a weight written by the kernel just before an unflagged call must be the one it uses."""
import contextlib

import pytest
import torch

gpu = pytest.mark.gpu
BF = torch.bfloat16
SENT = -1984.0
MS = (100, 128, 129, 200, 201, 207, 208, 209, 255, 256)
WIDTHS = {"8b": dict(d=4096, Hq=32, Hkv=8, ffn=14336), "70b": dict(d=8192, Hq=64, Hkv=8, ffn=28672)}
FORMS = ("qkv", "o", "gate_up", "down")
PAD = 8   # sentinel rows past M


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


@contextlib.contextmanager
def config(split_ring, splits=0, cluster=(0, 0)):
    from ultravox_b200 import _lib
    lib = _lib.lib()
    lib.uvx_debug_gemm_split_ring(split_ring)
    lib.uvx_debug_gemm_override(0, splits)
    lib.uvx_debug_gemm_cluster(*cluster)
    try:
        yield
    finally:
        lib.uvx_debug_gemm_split_ring(-1)
        lib.uvx_debug_gemm_override(0, 0)
        lib.uvx_debug_gemm_cluster(0, 0)


def window(rows, cols, gen):
    """[rows, cols] view at the top of a NaN-filled [256 + PAD, cols] buffer"""
    buf = torch.full((256 + PAD, cols), float("nan"), dtype=BF, device="cuda")
    buf[:rows] = torch.randn(rows, cols, device="cuda", generator=gen).to(BF)
    return buf[:rows]


class Form:
    """one prefill GEMM at one width; ``__call__(M)`` runs it on the first M rows and returns (output, norm_out or None) including
    PAD sentinel rows past M"""

    def __init__(self, ops, name, w, gen):
        self.ops, self.name = ops, name
        d, ffn, hd = w["d"], w["ffn"], 128
        self.N, self.K = {"qkv": ((w["Hq"] + 2 * w["Hkv"]) * hd, d), "o": (d, w["Hq"] * hd), "gate_up": (2 * ffn, d),
                          "down": (d, ffn)}[name]
        self.x = (torch.randn(256, self.K, device="cuda", generator=gen)).to(BF)
        W = (torch.randn(self.N, self.K, device="cuda", generator=gen) * 0.02).to(BF)
        if name == "gate_up":
            self.W = ops.TiledWeight(W, 128, swiglu=True)
            del W
        else:
            self.W = W
        if name == "qkv":
            inv = ops.llama3_inv_freq(hd, 500000.0, dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                                         original_max_position_embeddings=8192))
            self.cos, self.sin = ops.rope_tables(inv, 512, "cuda")
            self.rope_cols = (w["Hq"] + w["Hkv"]) * hd
        if name in ("o", "down"):
            self.h0 = (torch.randn(256, self.N, device="cuda", generator=gen)).to(BF)
            self.nw = (1.0 + 0.1 * torch.randn(self.N, device="cuda", generator=gen)).to(BF)
        torch.cuda.synchronize()

    def __call__(self, M):
        ops = self.ops
        xbuf = torch.full((256 + PAD, self.K), float("nan"), dtype=BF, device="cuda")
        xbuf[:M] = self.x[:M]
        x = xbuf[:M]                                                 # A: a window of a NaN-filled buffer
        ops.gemm_workspace(torch.device("cuda")).fill_(255)        # NaN partial sums
        n_out = self.N // 2 if self.name == "gate_up" else self.N
        out = torch.full((M + PAD, n_out), SENT, dtype=BF, device="cuda")
        xn = None
        if self.name == "qkv":
            ops.linear(x, self.W, out=out[:M], rope=(self.cos, self.sin, None, M, 3, self.rope_cols))
        elif self.name == "gate_up":
            ops.linear_tiled(x, self.W, out=out[:M], act=ops.ACT_SWIGLU, flags=ops.GEMM_W_STATIC)   # as the model calls it
        else:
            out[:M] = self.h0[:M]
            xn = torch.full((M + PAD, n_out), SENT, dtype=BF, device="cuda")
            ops.linear(x, self.W, residual=out[:M], out=out[:M], norm=(self.nw, 1e-5, xn[:M]))
        torch.cuda.synchronize()
        return out, xn


def same_bits(a, b):
    return a is None and b is None or torch.equal(a.view(torch.int16), b.view(torch.int16))


def check_rows_past_m(t, M, what):
    if t is not None:
        assert torch.all(t[M:] == SENT), f"{what}: rows past M = {M} lost their sentinel"


_FORMS: dict = {}


def form(ops, width, name):
    key = (width, name)
    if key not in _FORMS:
        _FORMS.clear()             # one (width, form) at a time: the 70B weights are large
        torch.cuda.empty_cache()
        seed = 10 * list(WIDTHS).index(width) + FORMS.index(name)
        _FORMS[key] = Form(ops, name, WIDTHS[width], torch.Generator(device="cuda").manual_seed(seed))
    return _FORMS[key]


@gpu
@pytest.mark.parametrize("width", tuple(WIDTHS))
@pytest.mark.parametrize("name", FORMS)
def test_split_ring_matches_single_ring(ops, width, name):
    """split ring vs one ring, every M box edge, forced split counts 1 / 3 / 7 (o / down; the fused RoPE and SwiGLU epilogues
    are tile-local and run one split), 2 x 2 clusters (the heuristic, q|k|v) on and off; and two runs give the same bits"""
    f = form(ops, width, name)
    bad = []
    for M in MS:
        for splits in ((1, 3, 7) if name in ("o", "down") else (0,)):
            for cluster in ((0, 0), (1, 1)):
                with config(5, splits, cluster):
                    got, got_n = f(M)
                    again, again_n = f(M)
                with config(0, splits, cluster):
                    ref, ref_n = f(M)
                tag = f"M={M} splits={splits} cluster={cluster}"
                assert torch.isfinite(got[:M].float()).all(), f"{tag}: non-finite output"
                check_rows_past_m(got, M, f"{tag} output")
                check_rows_past_m(got_n, M, f"{tag} norm_out")
                if not (same_bits(got, ref) and same_bits(got_n, ref_n)):
                    bad.append(f"{tag}: split ring differs from the one ring")
                if not (same_bits(got, again) and same_bits(got_n, again_n)):
                    bad.append(f"{tag}: two runs differ")
    assert not bad, "\n".join(bad)


@gpu
def test_static_weight_flag_in_graph_matches_eager(ops):
    """flagged gate|up calls over several images, back to back in a CUDA graph (each call's weight stream starts under the
    previous kernel), give the eager bits"""
    gen = torch.Generator(device="cuda").manual_seed(11)
    d, ffn, M = 4096, 14336, 201
    imgs = [ops.TiledWeight((torch.randn(2 * ffn, d, device="cuda", generator=gen) * 0.02).to(BF), 128, swiglu=True)
            for _ in range(3)]
    torch.cuda.synchronize()
    xs = [window(M, d, gen) for _ in range(3)]
    outs = [torch.empty(M, ffn, dtype=BF, device="cuda") for _ in range(6)]

    def seq():
        for i, o in enumerate(outs):
            ops.linear_tiled(xs[i % 3], imgs[(i + 1) % 3], out=o, act=ops.ACT_SWIGLU, flags=ops.GEMM_W_STATIC)

    seq()
    torch.cuda.synchronize()
    eager = [o.clone() for o in outs]
    for o in outs:
        o.fill_(SENT)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        seq()                                   # the graph's split-K workspace and warm-up
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            seq()
    torch.cuda.current_stream().wait_stream(s)
    for o in outs:
        o.fill_(SENT)
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(outs, eager)):
        assert same_bits(a, b), f"graph replay call {i} differs from eager"


@gpu
@pytest.mark.parametrize("graphed", (False, True))
def test_weight_written_by_previous_kernel_is_read(ops, graphed):
    """the GEMM just before writes the weight (its output is W); the unflagged call after it must use the new W"""
    gen = torch.Generator(device="cuda").manual_seed(12)
    M, K, N = 201, 4096, 4096
    W = (torch.randn(N, K, device="cuda", generator=gen) * 0.02).to(BF)
    src_a = (torch.randn(N, 256, device="cuda", generator=gen) * 0.1).to(BF)
    src_b = (torch.randn(K, 256, device="cuda", generator=gen) * 0.1).to(BF)
    x = window(M, K, gen)
    y = torch.empty(M, N, dtype=BF, device="cuda")

    def seq():
        ops.linear(src_a, src_b, out=W)           # W <- src_a @ src_b.T, [N, K]
        ops.linear(x, W, out=y)

    if graphed:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            seq()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                seq()
        torch.cuda.current_stream().wait_stream(s)
        W.zero_()
        y.fill_(SENT)
        g.replay()
    else:
        seq()
    torch.cuda.synchronize()
    W_new = ops.linear(src_a, src_b)
    assert torch.equal(W, W_new)
    assert same_bits(y, ops.linear(x, W_new)), "the call read a stale weight"
