"""The staged GEMM epilogue (output tile through shared memory and out by TMA store, the residual loaded by TMA ahead of the tile)
gives the register epilogue's bits: every call is run with uvx_debug_gemm_tma_store(0) (register epilogue) and (1) (staged wherever
it applies) and the results must be equal.  Covers the Whisper encoder GEMMs (in-place residual stream), the conv stem (guard rows,
the positional residual shared by every clip), batches, fp32 output, M / K tails, one and several tiles per CTA, output windows,
the row-map fallback and the adapter-training shapes."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF)


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def run(fn, on):
    from ultravox_b200 import _lib
    lib = _lib.lib()
    lib.uvx_debug_gemm_tma_store(on)
    try:
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        lib.uvx_debug_gemm_tma_store(-1)


def same_bits(fn):
    """fn() with the register epilogue and with the staged one: identical bits; returns the staged result"""
    want = run(fn, 0)
    got = run(fn, 1)
    assert got.dtype == want.dtype and torch.equal(got, want)
    return got


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.mark.parametrize("N,K,epi", [(3840, 1280, "bias"), (1280, 1280, "bias_res_inplace"), (5120, 1280, "bias_gelu"),
                                     (1280, 5120, "bias_res")])
def test_staged_encoder_calls(ops, N, K, epi):
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

    got = same_bits(fn)
    ref = x.float() @ w.float().T + b.float()
    if epi == "bias_gelu":
        ref = torch.nn.functional.gelu(ref)
    if epi.startswith("bias_res"):
        ref = ref + r.float()
    assert rel(got, ref) < 5e-3


@pytest.mark.parametrize("batch", [1, 2])
def test_staged_conv_stem(ops, batch):
    """conv1 writes rows t + 1 of a guarded buffer (guard rows stay zero); conv2 adds the positional embedding, one residual
    for every clip (batch stride 0)"""
    T, Cin, D = 3000, 128, 1280
    x = torch.zeros(batch, T + 2, Cin, dtype=BF, device="cuda")
    x[:, 1:T + 1] = rnd(batch, T, Cin, seed=5)
    w1, b1 = rnd(D, 3 * Cin, scale=0.05, seed=6), rnd(D, seed=7)
    w2, b2 = rnd(D, 3 * D, scale=0.02, seed=8), rnd(D, seed=9)
    pos = rnd(T // 2, D, seed=10)

    def conv1():
        h1 = torch.zeros(batch, T + 2, D, dtype=BF, device="cuda")
        return ops.conv1d_k3(x, w1, b1, 1, h1, out_guard=True)

    h1 = same_bits(conv1)
    assert not h1[:, 0].any() and not h1[:, T + 1].any()
    assert h1[:, 1:T + 1].abs().sum() > 0

    def conv2(p):
        h = torch.empty(batch, T // 2, D, dtype=BF, device="cuda")
        return ops.conv1d_k3(h1, w2, b2, 2, h, out_guard=False, pos=p)

    with_pos = same_bits(lambda: conv2(pos))
    without = same_bits(lambda: conv2(None))
    for i in range(batch):
        assert rel(with_pos[i].float() - without[i].float(), pos) < 3e-2


def test_staged_batched_and_fp32_alpha(ops):
    """a_batch = 2 through gemm_raw's batch strides, with a per-batch residual; fp32 output with alpha != 1"""
    B, M, K, N = 2, 700, 1280, 1280
    x, w, b = rnd(B, M, K, seed=11), rnd(N, K, scale=0.03, seed=12), rnd(N, seed=13)
    r = rnd(B, M, N, seed=14)

    def batched():
        out = torch.empty(B, M, N, dtype=BF, device="cuda")
        ops.gemm_raw(x.data_ptr(), B, M, K, K, M * K, w, out, N, M, 0, None, b, r, N, M * N, 1.0, ops.ACT_GELU)
        return out

    got = same_bits(batched)
    ref = torch.nn.functional.gelu(x.float() @ w.float().T + b.float()) + r.float()
    assert rel(got, ref) < 5e-3
    x2 = x.reshape(B * M, K)
    f32 = same_bits(lambda: ops.linear(x2, w, b, out_dtype=torch.float32, alpha=0.37))
    assert f32.dtype == torch.float32
    assert rel(f32, 0.37 * (x2.float() @ w.float().T) + b.float()) < 5e-3


# M tails, a K tail (200), a single k-block (64), N % 128 == 64 (64-wide tiles), one tile per CTA (384 x 128: three tiles) and
# several (1500 x 5120: 480 tiles)
@pytest.mark.parametrize("M,N,K", [(257, 3840, 1280), (1499, 3840, 1280), (1500, 1280, 200), (1500, 3840, 64), (1500, 1344, 640),
                                   (384, 128, 256), (1500, 5120, 640), (3000, 1280, 384)])
def test_staged_tails_and_tile_counts(ops, M, N, K):
    x, w, b, r = rnd(M, K, seed=15), rnd(N, K, scale=0.05, seed=16), rnd(N, seed=17), rnd(M, N, seed=18)
    got = same_bits(lambda: ops.linear(x, w, b, residual=r))
    assert rel(got, x.float() @ w.float().T + b.float() + r.float()) < 5e-3
    same_bits(lambda: ops.linear(x, w))
    same_bits(lambda: ops.linear(x, w, b, act=ops.ACT_GELU, out_dtype=torch.float32))


def test_staged_output_window_of_guarded_buffer(ops):
    """the output and the residual are windows of larger buffers: the window is written and nothing outside it"""
    M, N, K = 1499, 1280, 1280
    x, w, b = rnd(M, K, seed=19), rnd(N, K, scale=0.03, seed=20), rnd(N, seed=21)
    rbuf = rnd(M + 3, N + 128, seed=22)
    r = rbuf[2:M + 2, 64:N + 64]

    def fn():
        guard = torch.full((M + 2, N + 64), 7.0, dtype=BF, device="cuda")
        ops.linear(x, w, b, act=ops.ACT_GELU, residual=r, out=guard[1:M + 1, :N])
        return guard

    g = same_bits(fn)
    assert (g[0] == 7).all() and (g[M + 1] == 7).all() and (g[:, N:] == 7).all()


def test_staged_row_map_falls_back(ops):
    """a c_row_map call keeps the register epilogue under either switch value"""
    M, N, K = 600, 1280, 640
    x, w, b = rnd(M, K, seed=23), rnd(N, K, scale=0.03, seed=24), rnd(N, seed=25)
    rows = torch.randperm(M, generator=torch.Generator().manual_seed(0)).to(torch.int32)
    rows[::7] = -1                                          # dropped rows

    def fn():
        out = torch.full((M, N), 7.0, dtype=BF, device="cuda")
        return ops.linear(x, w, b, out=out, row_map=rows.cuda())

    got = same_bits(fn)
    keep = rows >= 0
    want = ops.linear(x, w, b)
    assert torch.equal(got[rows[keep].long().cuda()], want[keep.cuda()])
    assert (got[torch.tensor(sorted(set(range(M)) - set(rows[keep].tolist())), dtype=torch.long, device="cuda")] == 7).all()


# adapter training (cfg3, 4 clips of 30 s): the encoder at 6000 rows, the Llama GEMMs at ~1000 rows (256-wide tiles where they
# fill a wave: the register epilogue), the fp32 logits of the loss rows against the 128256-row head
@pytest.mark.parametrize("M,N,K,epi", [(6000, 3840, 1280, "bias"), (6000, 1280, 5120, "bias_res"), (6000, 5120, 1280, "bias_gelu"),
                                       (1000, 6144, 4096, "plain"), (1000, 4096, 4096, "res"), (1000, 4096, 14336, "res"),
                                       (300, 128256, 4096, "f32")])
def test_staged_training_shapes(ops, M, N, K, epi):
    x, w = rnd(M, K, seed=26), rnd(N, K, scale=0.02, seed=27)
    b = rnd(N, seed=28) if epi.startswith("bias") else None
    r = rnd(M, N, seed=29) if epi.endswith("res") else None
    act = ops.ACT_GELU if epi == "bias_gelu" else ops.ACT_NONE
    dt = torch.float32 if epi == "f32" else BF
    same_bits(lambda: ops.linear(x, w, b, act=act, residual=r, out_dtype=dt))


def test_staged_reproducible(ops):
    M, N, K = 1500, 1280, 1280
    x, w, b, r = rnd(M, K, seed=30), rnd(N, K, scale=0.03, seed=31), rnd(N, seed=32), rnd(M, N, seed=33)
    first = run(lambda: ops.linear(x, w, b, residual=r), 1)
    for _ in range(3):
        assert torch.equal(run(lambda: ops.linear(x, w, b, residual=r), 1), first)
