"""The plain GEMM epilogue loads its bias columns and residual rows ahead of its stores on the narrow tilings (MT * BN <= 128: 128 x
64 and 128 x 128, 256 x 64) and next to each store on the wide ones (256 x 128, 128 x 256).  K is summed in k-block order whatever the
tiling, so every tiling must give the same bits: at the Whisper encoder shapes (with the in-place residual stream), the conv stem
with its guard rows, batches, fp32 output, M / K tails, few tiles and windows of larger buffers."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


def rnd(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def run(fn, cfg=0):
    """fn() on the default path (cfg 0) or under a forced tiling MT*1000 + BN with one split"""
    from ultravox_b200 import _lib
    lib = _lib.lib()
    lib.uvx_debug_gemm_override(cfg, 1 if cfg else 0)
    try:
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        lib.uvx_debug_gemm_override(0, 0)


def same_everywhere(fn):
    """the default path and the hoisting tilings (128 x 128, 128 x 64, 256 x 64) give the bits of the 256 x 128 tiling, whose
    epilogue loads next to its stores; returns the default's"""
    want = run(fn, cfg=2128)
    got = run(fn)
    assert torch.equal(got, want)
    for cfg in (1128, 1064, 2064):
        assert torch.equal(run(fn, cfg), want), cfg
    return got


# the four encoder GEMMs at T = 1500 with the epilogue each runs in the model
@pytest.mark.parametrize("N,K,epi", [(3840, 1280, "bias"), (1280, 1280, "bias_res_inplace"), (5120, 1280, "bias_gelu"),
                                     (1280, 5120, "bias_res")])
def test_hoisted_epilogue_encoder_shapes_bit_identical(ops, N, K, epi):
    M = 1500
    x, w, b, r = rnd(M, K, seed=1), rnd(N, K, scale=0.03, seed=2), rnd(N, seed=3), rnd(M, N, seed=4)

    def fn():
        if epi == "bias":
            return ops.linear(x, w, b)
        if epi == "bias_gelu":
            return ops.linear(x, w, b, act=ops.ACT_GELU)
        if epi == "bias_res":
            return ops.linear(x, w, b, residual=r)
        h = r.clone()                                       # the encoder's residual stream: out aliases the residual
        return ops.linear(x, w, b, residual=h, out=h)

    got = same_everywhere(fn)
    ref = x.float() @ w.float().T + b.float()
    if epi == "bias_gelu":
        ref = torch.nn.functional.gelu(ref)
    if epi.startswith("bias_res"):
        ref = ref + r.float()
    assert ((got.float() - ref).norm() / ref.norm()).item() < 5e-3


@pytest.mark.parametrize("batch", [1, 2])
def test_hoisted_epilogue_conv_stem_guard_rows(ops, batch):
    """both conv-stem GEMMs at T = 3000 (conv1 writes rows t + 1 of a guarded buffer whose guard rows stay zero)"""
    T, Cin, D = 3000, 128, 1280
    x = torch.zeros(batch, T + 2, Cin, dtype=BF, device="cuda")
    x[:, 1:T + 1] = rnd(batch, T, Cin, seed=5)
    w1, b1 = rnd(D, 3 * Cin, scale=0.05, seed=6), rnd(D, seed=7)
    w2, b2 = rnd(D, 3 * D, scale=0.02, seed=8), rnd(D, seed=9)
    pos = rnd(T // 2, D, seed=10)

    def conv1():
        h1 = torch.zeros(batch, T + 2, D, dtype=BF, device="cuda")
        return ops.conv1d_k3(x, w1, b1, 1, h1, out_guard=True)

    h1 = same_everywhere(conv1)
    assert not h1[:, 0].any() and not h1[:, T + 1].any()
    assert h1[:, 1:T + 1].abs().sum() > 0

    def conv2():
        h = torch.empty(batch, T // 2, D, dtype=BF, device="cuda")
        return ops.conv1d_k3(h1, w2, b2, 2, h, out_guard=False, pos=pos)

    same_everywhere(conv2)


def test_hoisted_epilogue_batched_and_fp32_alpha(ops):
    """a_batch = 2 through gemm_raw's batch strides; fp32 output with alpha != 1"""
    B, M, K, N = 2, 700, 1280, 1280
    x, w, b = rnd(B, M, K, seed=11), rnd(N, K, scale=0.03, seed=12), rnd(N, seed=13)

    def batched():
        out = torch.empty(B, M, N, dtype=BF, device="cuda")
        ops.gemm_raw(x.data_ptr(), B, M, K, K, M * K, w, out, N, M, 0, None, b, None, 0, 0, 1.0, ops.ACT_GELU)
        return out

    got = same_everywhere(batched)
    ref = torch.nn.functional.gelu(x.float() @ w.float().T + b.float())
    assert ((got.float() - ref).norm() / ref.norm()).item() < 5e-3
    x2 = x.reshape(B * M, K)
    f32 = same_everywhere(lambda: ops.linear(x2, w, b, out_dtype=torch.float32, alpha=0.37))
    assert f32.dtype == torch.float32


# M tails (257, 1499), a K tail (200), a single k-block and few tiles.  Shapes the heuristic runs with one split (at 257 x 1280
# x 1280 it splits K, which is a different sum order from one split by design).
@pytest.mark.parametrize("M,N,K", [(257, 3840, 1280), (1499, 3840, 1280), (1500, 1280, 200), (1500, 5120, 640),
                                   (384, 128, 256), (1500, 3840, 64), (3000, 1280, 384)])
def test_hoisted_epilogue_tails_and_tile_counts(ops, M, N, K):
    x, w, b, r = rnd(M, K, seed=14), rnd(N, K, scale=0.05, seed=15), rnd(N, seed=16), rnd(M, N, seed=17)
    same_everywhere(lambda: ops.linear(x, w, b, residual=r))
    same_everywhere(lambda: ops.linear(x, w))


def test_hoisted_epilogue_output_window_of_guarded_buffer(ops):
    """the output is a window of a larger buffer: the window is written and nothing outside it"""
    M, N, K = 1500, 1280, 1280
    x, w, b = rnd(M, K, seed=18), rnd(N, K, scale=0.03, seed=19), rnd(N, seed=20)

    def fn():
        guard = torch.full((M + 2, N + 64), 7.0, dtype=BF, device="cuda")
        ops.linear(x, w, b, act=ops.ACT_GELU, out=guard[1:M + 1, :N])
        return guard

    g = same_everywhere(fn)
    assert (g[0] == 7).all() and (g[M + 1] == 7).all() and (g[:, N:] == 7).all()


def test_hoisted_epilogue_reproducible(ops):
    M, N, K = 1500, 5120, 1280
    x, w, b = rnd(M, K, seed=21), rnd(N, K, scale=0.03, seed=22), rnd(N, seed=23)
    first = run(lambda: ops.linear(x, w, b, act=ops.ACT_GELU))
    for _ in range(3):
        assert torch.equal(run(lambda: ops.linear(x, w, b, act=ops.ACT_GELU)), first)
