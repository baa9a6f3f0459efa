"""Thread-block clusters of the Hopper GEMM (gemm_tc.cu): TMA multicast of the A box along N and of the W box along M moves
bytes, not arithmetic.  At the same tile configuration and split count, every cluster shape must give the bits of the run
without a cluster - in the model's own argument forms at the bench's prefill shapes, at M tails, batched, and in the implicit
GEMM of the encoder convolution - including shapes whose tile grid the cluster does not divide and grid caps that are not a
whole number of clusters."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
SHAPES = [(1, 2), (2, 1), (2, 2), (1, 4)]


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(BF).cuda()


@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


def run(fn, cfg, splits, cm, cn, grid=0):
    """fn() under a forced tile configuration, split count, cluster shape and persistent-grid cap; hooks reset afterwards"""
    from ultravox_b200 import _lib
    lib = _lib.lib()
    lib.uvx_debug_gemm_override(cfg, splits)
    lib.uvx_debug_gemm_cluster(cm, cn)
    lib.uvx_debug_gemm_ws(-1, 0, grid)
    try:
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        lib.uvx_debug_gemm_override(0, 0)
        lib.uvx_debug_gemm_cluster(0, 0)
        lib.uvx_debug_gemm_ws(-1, 0, 0)


def same_bits(fn, cfg, splits, shapes=SHAPES, grid=0):
    want = run(fn, cfg, splits, 1, 1)
    for cm, cn in shapes:
        got = run(fn, cfg, splits, cm, cn, grid)
        for w, g in zip(want, got):
            assert torch.equal(w, g), (cfg, splits, cm, cn, grid)
    return want


def _bench_forms(ops, M):
    """the four Llama-3.1-8B prefill GEMMs of one layer (S = M tokens) in the model's argument forms"""
    D, F, Hq, Hkv, hd = 4096, 14336, 32, 8, 128
    x, att, act = rnd(M, D, seed=1), rnd(M, D, seed=2), rnd(M, F, seed=3)
    inv = ops.llama3_inv_freq(hd, 500000.0, dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                                 original_max_position_embeddings=8192))
    cos, sin = ops.rope_tables(inv, 512, "cuda")
    rope = (cos, sin, None, M, 0, (Hq + Hkv) * hd)
    wqkv = rnd((Hq + 2 * Hkv) * hd, D, scale=0.02, seed=4)
    wo, wd = rnd(D, D, scale=0.02, seed=5), rnd(D, F, scale=0.02, seed=6)
    gu = ops.TiledWeight(rnd(2 * F, D, scale=0.02, seed=7), 128, swiglu=True)
    h0, nw = rnd(M, D, seed=8), rnd(D, seed=9)

    def residual_norm(a, w):
        def f():
            h, xn = h0.clone(), torch.empty(M, D, dtype=BF, device="cuda")
            ops.linear(a, w, residual=h, out=h, norm=(nw, 1e-5, xn))
            return h, xn
        return f
    return {"qkv": (lambda: (ops.linear(x, wqkv, rope=rope),), 1128, 1),
            "o": (residual_norm(att, wo), 2128, 4),
            "gate_up": (lambda: (ops.linear_tiled(x, gu, act=ops.ACT_SWIGLU),), 1128, 1),
            "down": (residual_norm(act, wd), 2128, 4)}


@pytest.mark.parametrize("form", ["qkv", "o", "gate_up", "down"])
def test_cluster_bench_prefill_forms_bit_identical(ops, form):
    fn, cfg, splits = _bench_forms(ops, 201)[form]
    same_bits(fn, cfg, splits)
    if cfg == 1128 and form == "gate_up":
        same_bits(fn, 2128, 1, shapes=[(1, 2), (1, 4)])


@pytest.mark.parametrize("M", [77, 129])
def test_cluster_m_tails_bit_identical(ops, M):
    forms = _bench_forms(ops, M)
    for form in ("qkv", "gate_up", "o"):
        fn, cfg, splits = forms[form]
        same_bits(fn, cfg, splits)


def test_cluster_batched_a_bit_identical(ops):
    """a_batch = 2 (batch-strided A, c_batch_rows): cm pairs m-tiles of different batches"""
    B, M, K, N = 2, 150, 1024, 768
    x, w, b = rnd(B, M, K, seed=1), rnd(N, K, scale=0.05, seed=2), rnd(N, seed=3)

    def f():
        out = torch.empty(B, M, N, dtype=BF, device="cuda")
        ops.gemm_raw(x.data_ptr(), B, M, K, K, M * K, w, out, N, M, bias=b)
        return (out,)
    for cfg, splits in ((1128, 1), (2128, 3), (1064, 2)):
        out = same_bits(f, cfg, splits)[0]
    ref = x.float() @ w.float().T + b.float()
    assert ((out.float() - ref).norm() / ref.norm()).item() < 3e-3


def test_cluster_conv_implicit_gemm_bit_identical(ops):
    """encoder conv2 (k = 3, stride 2) as an implicit GEMM over overlapping rows of the time-major input, T = 3000"""
    T, C = 3000, 1280
    x = torch.zeros(1, T + 2, C, dtype=BF, device="cuda")
    x[:, 1:T + 1] = rnd(1, T, C, seed=1)
    w, b = rnd(C, 3 * C, scale=0.02, seed=2), rnd(C, seed=3)

    def f():
        out = torch.zeros(1, T // 2 + 2, C, dtype=BF, device="cuda")
        ops.conv1d_k3(x, w, b, 2, out, out_guard=True)
        return (out,)
    same_bits(f, 1128, 1)
    same_bits(f, 1256, 1, shapes=[(2, 1)])


def test_cluster_not_dividing_tile_grid(ops):
    """3 n-tiles and 1 m-tile: cn = 2 / 4 and cm = 2 fall back to 1 on that axis; 5 ragged n-tiles of 208"""
    M, N, K = 201, 384, 512
    x, w = rnd(M, K, seed=1), rnd(N, K, scale=0.05, seed=2)
    same_bits(lambda: (ops.linear(x, w),), 2128, 1, shapes=[(2, 2), (1, 4), (2, 1), (4, 4)])
    w2 = rnd(1024, K, scale=0.05, seed=3)
    same_bits(lambda: (ops.linear(x, w2),), 1208, 1, shapes=[(2, 2), (4, 1)])


@pytest.mark.parametrize("grid", [5, 7, 3])
def test_cluster_grid_cap_not_whole_clusters(ops, grid):
    """a persistent-grid cap below or between whole clusters runs at least one cluster, every unit exactly once"""
    M, N, K = 201, 1536, 2048
    x, w, r = rnd(M, K, seed=1), rnd(N, K, scale=0.03, seed=2), rnd(M, N, seed=3)
    want = run(lambda: (ops.linear(x, w, residual=r),), 1128, 2, 1, 1)
    for cm, cn in SHAPES:
        got = run(lambda: (ops.linear(x, w, residual=r),), 1128, 2, cm, cn, grid=grid)
        assert torch.equal(want[0], got[0]), (cm, cn, grid)


def test_cluster_llama_hidden_bit_identical():
    """the prefill stack at cfg2 widths (2 layers, S = 201): the default dispatch (clusters) and no clusters give the same
    hidden states bit for bit - the cluster table keeps every tiling and split count"""
    from ultravox_b200 import _lib
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=2, vocab_size=2048))
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=1)
    g = torch.Generator().manual_seed(0)
    emb = (torch.randn(1, 201, 4096, generator=g) * 0.5).to(torch.bfloat16).cuda()
    default = model.llama_hidden(emb.clone()).clone()
    _lib.lib().uvx_debug_gemm_cluster(1, 1)
    try:
        off = model.llama_hidden(emb.clone()).clone()
    finally:
        _lib.lib().uvx_debug_gemm_cluster(0, 0)
    assert torch.equal(default, off)
