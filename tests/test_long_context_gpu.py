"""Per-op parity of the KV-cache attention kernels at long contexts (8 k - 131 072 keys): the decode form over a contiguous cache
(``attn_fwd_kernel``), the row-mapped and paged (bf16 / e4m3) decode forms, the chunk forms of ``attn_wg_kernel`` (contiguous,
paged bf16 / e4m3) and the prefill-on-a-cache form, at the Llama-3.1-8B heads (32 q / 8 kv, D 128) and, on the decode form,
the 70B heads (64 / 8).

Every form gets three score patterns:

* flat (seeded randn q, k, v): against fp32 softmax and against the rounding-matched 64-key tile walk, per batch row;
* needle: one key whose scaled log2 score gap to every other visible key is > 160, so every other ``exp2`` (and the rescale of
  everything before it) underflows to exactly 0 in fp32 and the output is that key's V row bit for bit.  A wrong page, a wrong
  or skipped tile, or a dropped rescale anywhere in a 2048-tile walk moves it;
* sink + recency: a large score at the first visible key and a higher band over the last 256, flat noise between - the running
  max is set in the first tile and corrected in the last ones.

The decode form also gets ties (the same maximal score in many tiles).  Each test also checks that two runs give the same bits,
that keys outside the visible range are never read (NaN / +-Inf there change no bit), and that another row's cache or pages
change no bit of this row.  The e4m3 forms are also checked bit for bit against the bf16 kernel on the dequantized pool.

Bounds: ``rel`` is the Frobenius-norm relative error of one batch row.  Against fp32 the error is the bf16 rounding of P (at
most 2^-9 relative per probability, independent between keys) and of the output: relative to the output that stays near
2^-9 / sqrt(3) ~ 1.1e-3 however many keys there are, so the short-context bound rel < 3e-3 holds.  Against the rounding-matched
walk the scores, the running max and P are the kernel's, but the scores come out of a different fp32 summation order (bf16
tensor-core products against an fp32 GEMM), so a few P round to the neighbouring bf16 value, and the kernel's O accumulates
T = ceil(n / 64) tile products in the tensor cores' fp32 accumulators: that part grows like sqrt(T).  Measured on an H100 80GB
HBM3 (700 W): 3.7e-4 at T = 125, 4.2e-4 at T = 509, 8.9e-4 at T = 1024 - 2048 and 1.03e-3 at T = 2047 (row-mapped decode,
kv_len 131009), so the bound is 1e-3 (the short-context suites' bound) up to T = 1024 and 1e-3 sqrt(T / 1024) above it:
1.41e-3 at 131 072 keys.  The needle patterns, not these bounds, are what catch a wrong or skipped tile.

The references run one KV head (one GQA group) at a time: a C = 248 chunk over 131 072 keys is a 0.5 GB fp32 score tensor per
group.  Pools and caches are freed after every test; the peak device memory of each test is printed (7.4 GiB at most measured,
the whole module about a minute on an H100 80GB HBM3)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
E4M3 = torch.float8_e4m3fn
NAN = float("nan")
NAN_BYTE = 0x7F                 # e4m3fn NaN
LOG2E = 1.4426950408889634

HQ8, HQ70, HKV, HD = 32, 64, 8, 128
PAGE = 64
W = 2048                        # table width: 131 072 keys
SMAX = W * PAGE
NEEDLE_Q = 4.0                  # every q element of a needle query; the needle key is the same vector
NEEDLE_GAP = 160.0              # required scaled log2 score gap (exp2(-150) is already 0 in fp32)
SCALES = [(1.0, 1.0), (2.0 ** -3, 0.37), (0.37, 2.0 ** -3)]      # (K, V) scales of the fp8 pool tests
BOUND_FP32 = 3e-3              # 2.63e-3 measured at most (H100 80GB HBM3, 700 W, every case here)


def bound_matched(n_keys):
    """rel bound against the rounding-matched walk over n_keys keys (module docstring): 1.03e-3 measured at most, at 2047 tiles."""
    return 1e-3 * max(1.0, math.sqrt(-(-n_keys // PAGE) / 1024))


# ================================================================================================ references
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


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def attention_refs(q, k, v, begin, end, shift=None, scale=None):
    """One batch row: q [Sq, Hq, D], k / v [S >= end, Hkv, D] (index = key position) -> (fp32 softmax(q k^T scale) v [Sq, Hq * D]
    fp32, rounding-matched reference [Sq, Hq * D] bf16) over the keys [begin, end), causal j <= i + shift when shift is given.

    The matched reference is the kernels' 64-key tile walk from tile begin // 64: scores unscaled in fp32, a running max m_t
    (the max over tiles <= t), P = exp2((s - m_t) scale log2 e) rounded to bf16 before P.V, l summed in fp32 on the unrounded P,
    every earlier tile rescaled by exp2((m_t - m_T) scale log2 e) (the product of the walk's per-tile factors), the output
    rounded once.  It runs one KV head at a time on the device of q."""
    Sq, Hq, D = q.shape
    Hkv = k.shape[1]
    G = Hq // Hkv
    dev = q.device
    sc = torch.tensor(D ** -0.5 if scale is None else scale, dtype=torch.float32)
    sl2 = float(sc * torch.tensor(LOG2E, dtype=torch.float32))
    t0 = begin // PAGE * PAGE
    n = max(end - t0, 0)
    nt = max(-(-n // PAGE), 1)
    j = torch.arange(t0, t0 + nt * PAGE, device=dev)
    ok = ((j >= begin) & (j < end))[None].expand(Sq, -1)
    if shift is not None:
        ok = ok & (j[None] <= torch.arange(Sq, device=dev)[:, None] + shift)
    ref = torch.empty(Sq, Hkv, G, D, device=dev)
    matched = torch.empty(Sq, Hkv, G, D, dtype=BF, device=dev)
    for h in range(Hkv):
        kh = torch.zeros(nt * PAGE, D, device=dev)
        vh = torch.zeros(nt * PAGE, D, device=dev)
        kh[:n], vh[:n] = k[t0:t0 + n, h].float(), v[t0:t0 + n, h].float()
        vh[:n].masked_fill_(~ok[-1, :n, None], 0.0)                          # keys no query sees may hold NaN / Inf
        qh = q[:, h * G:(h + 1) * G].float().transpose(0, 1)                  # [G, Sq, D]
        s = (qh @ kh.T).masked_fill(~ok, float("-inf"))                        # [G, Sq, nt * 64], unscaled
        ref[:, h] = (torch.softmax(s * sc, -1).nan_to_num(0.0) @ vh).transpose(0, 1)
        st = s.view(G, Sq, nt, PAGE)
        m = st.amax(-1).cummax(-1).values                                     # running max after each tile
        mref = torch.where(m == float("-inf"), torch.zeros_like(m), m)
        p = torch.exp2((st - mref[..., None]) * sl2)
        w = torch.where(m == float("-inf"), torch.zeros_like(m), torch.exp2((mref - mref[..., -1:]) * sl2))
        l = (p.sum(-1) * w).sum(-1)
        o = (p.to(BF).float() * w[..., None]).view(G, Sq, nt * PAGE) @ vh
        inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
        matched[:, h] = (o * inv[..., None]).to(BF).transpose(0, 1)
        del s, st, p, o
    return ref.view(Sq, Hq * D), matched.view(Sq, Hq * D)


# ================================================================================================ score patterns
def flat(*shape, seed, device, scale=1.0):
    """Seeded bf16 normal values generated on ``device``."""
    g = torch.Generator(device=device).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=device) * scale).to(BF)


def needle_q(rows, Hq, D, device, val=NEEDLE_Q):
    """Needle queries [rows, Hq * D]: every element ``val``."""
    return torch.full((rows, Hq * D), val, dtype=BF, device=device)


def plant_needle(k, p, val=NEEDLE_Q):
    """Key p of k [..., S, Hkv, D] (every head) becomes the needle query's own vector: score NEEDLE_Q^2 D = 2048 at D = 128,
    against 4 sum(k_j) ~ N(0, 2048) for randn keys, a scaled log2 gap of ~ (2048 - 5.2 * 45) / sqrt(128) * log2 e ~ 230."""
    k[..., p, :, :] = val


def needle_gap(k, p, begin, end, D=HD, val=NEEDLE_Q):
    """min over KV heads and visible keys j != p of (s_p - s_j) * D^-0.5 * log2 e for the needle query (fp64): the kernels'
    exp2 of minus this underflows to 0 in fp32 when it is > 150."""
    s = val * k[begin:end].float().sum(-1).double()               # [n, Hkv]
    sp = s[p - begin].clone()
    s[p - begin] = float("-inf")
    return float(((sp - s.amax(0)) * D ** -0.5 * LOG2E).min())


def sink_recency(q, k, begin, end, Hq, D):
    """q channel 0 = 8 in every head; key ``begin`` gets channel 0 = 14 (sink: ~9.9 nats above flat noise of std ~1.2) and the
    last 256 visible keys channel 0 = 15 (band: ~10.6 nats, many of them above the sink), in every KV head."""
    q.view(q.shape[0], Hq, D)[..., 0] = 8.0
    k[begin, :, 0] = 14.0
    k[max(begin + 1, end - 256):end, :, 0] = 15.0


def tie_positions(begin, end, every=37):
    """Key positions in every ``every``-th tile of [begin, end), at offsets that walk through the tile."""
    t0 = -(-begin // PAGE)
    return [PAGE * t + (7 * i) % PAGE for i, t in enumerate(range(t0, (end - 1) // PAGE, every)) if PAGE * t + (7 * i) % PAGE < end]


def poison_outside(k, v, start, end):
    """Copies of caches k / v [B, S, Hkv, D] with every position outside [start_b, end_b) set to NaN / +Inf / -Inf."""
    kp, vp = k.clone(), v.clone()
    vals = torch.tensor([NAN, float("inf"), float("-inf")], device=k.device).to(k.dtype)
    pos = torch.arange(k.shape[1], device=k.device)
    for b in range(k.shape[0]):
        out = (pos < int(start[b])) | (pos >= int(end[b]))
        kp[b, out] = vals[pos[out] % 3][:, None, None].expand(-1, k.shape[2], k.shape[3])
        vp[b, out] = vals[(pos[out] + 1) % 3][:, None, None].expand(-1, k.shape[2], k.shape[3])
    return kp, vp


# ================================================================================================ GPU plumbing
@pytest.fixture(autouse=True)
def _gpu_state():
    """fp32 references in full fp32 (no TF32); peak memory printed per test; buffers freed between tests."""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    torch.cuda.empty_cache()


def kernels_run(fn) -> str:
    """The names of the CUDA kernels ``fn`` (idempotent) launches (torch.profiler), one per line."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return "\n".join(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def assert_kernel(fn, want):
    """``fn`` runs the attention kernel ``want`` (e.g. "attn_fwd_kernel<128, false, false>") and no other attention kernel.  The
    profiler reports a kernel by its demangled or its mangled name.  A window without activity records is profiled again; when
    the profiler delivers no CUDA record at all (it does so now and then after earlier sessions in the same process) there is
    nothing to check and the miss is printed."""
    name, args = want[:-1].split("<")
    args = [a.strip() for a in args.split(",")]
    mangled = f"{name}ILi{args[0]}E" + "".join("Lb1E" if a == "true" else "Lb0E" for a in args[1:]) + "E"
    for _ in range(5):
        names = kernels_run(fn)
        if names:
            break
    if not names:
        print(f"profiler delivered no CUDA activity records: dispatch to {want} not checked")
        return
    attn = {ln.split("(")[0] for ln in names.splitlines() if "attn_" in ln}
    assert len(attn) == 1 and any(want in a or mangled in a for a in attn), (want, names)


class Stats:
    """Largest errors seen in one test, printed at its end."""

    def __init__(self, what, D=HD):
        self.what, self.D, self.r32, self.rm = what, D, 0.0, 0.0

    def check(self, got, q, k, v, begin, end, shift=None, what=""):
        """got [Sq, Hq * D] against both references of one batch row; returns the rounding-matched reference."""
        Sq = got.shape[0]
        ref, matched = attention_refs(q.view(Sq, -1, self.D), k, v, begin, end, shift)
        r32, rm = rel(got, ref.to(BF)), rel(got, matched)
        self.r32, self.rm = max(self.r32, r32), max(self.rm, rm)
        assert torch.isfinite(got.float()).all(), (self.what, what, "non-finite output")
        assert r32 < BOUND_FP32, (self.what, what, "vs fp32", r32)
        assert rm < bound_matched(end - begin // PAGE * PAGE), (self.what, what, "vs rounding-matched", rm)
        return matched

    def report(self):
        print(f"{self.what}: vs fp32 max rel {self.r32:.3e}, vs rounding-matched max rel {self.rm:.3e}")


def twice(fn):
    """fn() twice: the same bits both times."""
    a = fn().clone()
    assert torch.equal(a, fn()), "two runs differ"
    return a


def i32(x):
    return torch.tensor(x, dtype=torch.int32, device="cuda")


# ================================================================================================ 1. decode, contiguous cache
def decode(q, kc, vc, Hq, lens, start=None):
    """``ops.attention`` with one query per row (Sq = 1, non-causal) over caches [B, S_max, Hkv, D]."""
    from ultravox_b200 import ops
    B, smax, Hkv, D = kc.shape
    out = torch.empty(B, Hq * D, dtype=BF, device="cuda")
    cs = smax * Hkv * D
    return ops.attention(q.data_ptr(), kc.data_ptr(), vc.data_ptr(), out, B, Hq, Hkv, 1, smax, D,
                         (Hq * D, Hq * D, Hkv * D, cs, Hkv * D, cs, Hq * D, Hq * D), D ** -0.5, False, lens, 0, start)


def decode_rows(smax, B):
    """(kv_len, kv_start) per row: S_max, 64 k + 1 (65537 at S_max = 131072) and S_max - 1 behind a left pad (70 001 at S_max =
    131072: tile0 = 1093) for B = 3; 64 k - 1 for B = 1."""
    if B == 1:
        return [PAGE * (smax // PAGE - 3) - 1], [0]
    return [smax, PAGE * (smax // 128) + 1, smax - 1], [0, 0, 70001 if smax == SMAX else smax // 2 + 3]


DECODE_CASES = [("8b", 8193, 1), ("8b", 8193, 3), ("8b", 32768, 3), ("8b", SMAX, 1), ("8b", SMAX, 3), ("70b", 32768, 1),
                ("70b", SMAX, 3)]


@pytest.mark.parametrize("width,smax,B", DECODE_CASES)
def test_decode_long_cache(width, smax, B):
    decode_long_case(HQ8 if width == "8b" else HQ70, smax, B, width)


def decode_long_case(Hq, smax, B, width, D=HD, needle=NEEDLE_Q, check_dispatch=True):
    """``ops.attention`` with one query per row over a contiguous cache of S_max keys at head_dim D; ``needle`` is the needle's
    q / k element value (large enough for NEEDLE_GAP at that D); ``check_dispatch=False`` for callers that assert the kernel of
    the same call in a process of their own."""
    lens, starts = decode_rows(smax, B)
    lens_t, start_t = i32(lens), i32(starts)
    what = f"decode {width} S_max={smax} B={B} lens={lens} starts={starts}"
    st = Stats(what, D)
    seed = smax + B + Hq
    kc, vc = flat(B, smax, HKV, D, seed=seed, device="cuda"), flat(B, smax, HKV, D, seed=seed + 1, device="cuda")
    q = flat(B, Hq * D, seed=seed + 2, device="cuda")
    run = lambda: decode(q, kc, vc, Hq, lens_t, start_t)          # noqa: E731
    if check_dispatch:
        assert_kernel(run, f"attn_fwd_kernel<{D}, false, false>")
    # flat: both references per row, the same bits twice, masked positions never read, row isolation
    out = twice(run)
    for b in range(B):
        st.check(out[b:b + 1], q[b], kc[b], vc[b], starts[b], lens[b], what=f"flat row {b}")
    kp, vp = poison_outside(kc, vc, starts, lens)
    assert torch.equal(decode(q, kp, vp, Hq, lens_t, start_t), out), (what, "reads a masked cache position")
    del kp, vp
    if B > 1:
        k2, v2 = kc.clone(), vc.clone()
        k2[0], v2[0] = flat(smax, HKV, D, seed=seed + 3, device="cuda"), flat(smax, HKV, D, seed=seed + 4, device="cuda")
        o2 = decode(q, k2, v2, Hq, lens_t, start_t)
        assert torch.equal(o2[1:], out[1:]) and not torch.equal(o2[0], out[0]), (what, "row isolation")
        del k2, v2
    # needle: bit for bit the needle's V row in every q head of its group
    qn = needle_q(B, Hq, D, "cuda", needle)
    G = Hq // HKV
    for b in range(B):
        e = lens[b]
        spots = sorted({0, 63, 64, starts[b], PAGE * ((starts[b] + e) // 128) + 17, PAGE * ((e - 1) // PAGE), e - 1})
        for p in (p for p in spots if starts[b] <= p < e):
            k0 = kc[b, p].clone()
            plant_needle(kc[b], p, needle)
            assert needle_gap(kc[b], p, starts[b], e, D, needle) > NEEDLE_GAP
            got = decode(qn, kc, vc, Hq, lens_t, start_t)[b]
            want = vc[b, p].repeat_interleave(G, 0).reshape(-1)
            assert torch.equal(got, want), (what, f"needle row {b} at {p}", int((got != want).sum()))
            kc[b, p] = k0
    # sink + recency
    qs = q.clone()
    k3 = kc.clone()
    for b in range(B):
        sink_recency(qs[b:b + 1], k3[b], starts[b], lens[b], Hq, D)
    out = twice(lambda: decode(qs, k3, vc, Hq, lens_t, start_t))
    for b in range(B):
        st.check(out[b:b + 1], qs[b], k3[b], vc[b], starts[b], lens[b], what=f"sink row {b}")
    # ties: the needle score at keys in every 37th tile; every other key underflows
    k3.copy_(kc)
    for b in range(B):
        for p in tie_positions(starts[b], lens[b]):
            plant_needle(k3[b], p, needle)
    out = twice(lambda: decode(qn, k3, vc, Hq, lens_t, start_t))
    for b in range(B):
        st.check(out[b:b + 1], qn[b], k3[b], vc[b], starts[b], lens[b], what=f"ties row {b}")
        # P = 1 at every tie and exactly 0 elsewhere: the mean of the tied V rows, within one bf16 ulp
        mean = vc[b, tie_positions(starts[b], lens[b])].double().mean(0).repeat_interleave(G, 0).reshape(-1)
        assert_within(out[b], mean, bf16_ulp(mean), f"{what} ties row {b}")
    st.report()


# ================================================================================================ 2. row-mapped decode
def test_rows_decode_long_cache():
    """``attention_rows``: six query rows over two 131072-key cache rows (three per row, different kv_len), as slot lookup
    maps them: each query row against both references, the needle through its cache row, the same bits as the row alone."""
    from ultravox_b200 import ops
    Hq = HQ8
    kc, vc = flat(2, SMAX, HKV, HD, seed=1, device="cuda"), flat(2, SMAX, HKV, HD, seed=2, device="cuda")
    rows = [1, 0, 1, 1, 0, 0]
    lens = [SMAX, SMAX - 1, 65537, 64 * 1500 - 1, 8193, 131009]
    row_t, lens_t = i32(rows), i32(lens)
    q = flat(len(rows), Hq * HD, seed=3, device="cuda")
    what = "rows decode"
    st = Stats(what)

    def run(qq=q, k=kc, v=vc):
        out = torch.empty(len(rows), Hq * HD, dtype=BF, device="cuda")
        return ops.attention_rows(qq, k, v, out, Hq, HD ** -0.5, lens_t, row_t)
    assert_kernel(run, "attn_fwd_kernel<128, false, false>")
    out = twice(run)
    for r, (c, e) in enumerate(zip(rows, lens)):
        st.check(out[r:r + 1], q[r], kc[c], vc[c], 0, e, what=f"flat query row {r}")
        one = torch.empty(1, Hq * HD, dtype=BF, device="cuda")
        ops.attention_rows(q[r:r + 1], kc, vc, one, Hq, HD ** -0.5, lens_t[r:r + 1], row_t[r:r + 1])
        assert torch.equal(one[0], out[r]), (what, "alone != together", r)
    # positions past each cache row's longest kv_len never read; cache row 0 changes no bit of the rows on cache row 1
    kp, vp = poison_outside(kc, vc, [0, 0], [max(e for c, e in zip(rows, lens) if c == x) for x in (0, 1)])
    assert torch.equal(run(k=kp, v=vp), out), (what, "reads a masked cache position")
    kp[0], vp[0] = flat(SMAX, HKV, HD, seed=4, device="cuda"), flat(SMAX, HKV, HD, seed=5, device="cuda")
    o2 = run(k=kp, v=vp)
    on1 = [r for r, c in enumerate(rows) if c == 1]
    assert torch.equal(o2[on1], out[on1]), (what, "cache row isolation")
    del kp, vp
    qn = needle_q(len(rows), Hq, HD, "cuda")
    for c in (0, 1):
        e = max(x for cc, x in zip(rows, lens) if cc == c)
        for p in (0, 64, 70001, 64 * 1500 + 3, e - 1):
            k0 = kc[c, p].clone()
            plant_needle(kc[c], p)
            got = run(qq=qn)
            for r in (r for r, (cc, x) in enumerate(zip(rows, lens)) if cc == c and p < x):
                assert torch.equal(got[r], vc[c, p].repeat_interleave(Hq // HKV, 0).reshape(-1)), (what, "needle", r, p)
            kc[c, p] = k0
    qs = q.clone()
    for c in (0, 1):
        sink_recency(qs, kc[c], 0, max(x for cc, x in zip(rows, lens) if cc == c), Hq, HD)
    out = twice(lambda: run(qq=qs))
    for r, (c, e) in enumerate(zip(rows, lens)):
        st.check(out[r:r + 1], qs[r], kc[c], vc[c], 0, e, what=f"sink query row {r}")
    st.report()


# ================================================================================================ 3. paged decode (bf16, e4m3)
def paged_table(lens, n_pages, hot, seed):
    """table [B, W] int32 of distinct pool pages, shuffled; the tiles in ``hot`` get the largest page indices of the pool; entries
    past each row's last tile are -1."""
    B = len(lens)
    top = n_pages - B * len(hot)
    g = torch.Generator().manual_seed(seed)
    table = torch.randperm(top, generator=g)[:B * W].view(B, W).to(torch.int32)
    for b in range(B):
        for i, t in enumerate(hot):
            table[b, t] = top + b * len(hot) + i
        table[b, -(-lens[b] // PAGE):] = -1
    return table


def rows_with_nan_tail(B, lens, seed, scale=1.0, D=HD):
    """k, v [B, 131072, Hkv, D] randn rows, NaN at positions >= lens[b]."""
    k, v = flat(B, SMAX, HKV, D, seed=seed, device="cuda", scale=scale), flat(B, SMAX, HKV, D, seed=seed + 1, device="cuda")
    for b, e in enumerate(lens):
        k[b, e:], v[b, e:] = NAN, NAN
    return k, v


def fill_pool(pool, rows, table):
    """Write rows [B, 131072, Hkv, D] into pool [n_pages, 64, Hkv, D] through table [B, W] (entries -1 skipped)."""
    for b in range(rows.shape[0]):
        t = table[b]
        live = t >= 0
        pool[t[live].long()] = rows[b].view(W, PAGE, *rows.shape[2:])[live]


def quant(x, s):
    """The host quantizer of include/uvx.h, on the device: clamp to +-448 (NaN passes), round to e4m3."""
    return (x.float() / s).clamp(-448, 448).to(E4M3)


def dequant(x8, s):
    return (x8.float() * s).to(BF)


def page_of(table, b, p):
    return int(table[b, p // PAGE]), p % PAGE


def put_keys(pool, table_row, pos, rows, s=None):
    """pool[page of position pos[i], pos[i] % 64] = rows[i] (bf16 values; quantized with scale s into an e4m3 pool)."""
    pos = torch.as_tensor(pos, device=pool.device)
    pool[table_row[pos // PAGE].long(), pos % PAGE] = rows if s is None else quant(rows, s)


PAGED_LENS = [SMAX, 100001]


def paged_needles(e):
    return sorted({0, 63, 64, PAGE * 1500 + 17, PAGE * ((e - 1) // PAGE), e - 1})


@pytest.mark.parametrize("kind", ["bf16", "fp8-0", "fp8-1", "fp8-2"])
def test_paged_decode_long_table(kind):
    paged_long_case(kind)


def paged_long_case(kind, D=HD, needle=NEEDLE_Q, check_dispatch=True):
    """``attention_paged`` (and its ``kv_row`` form) through 2048-entry tables into a pool of > 16384 bf16 pages (page byte
    offsets >= 2^31) or > 32768 e4m3 pages (element and byte offsets >= 2^31), every page outside the tables NaN; the needle's
    tiles sit in the pages with the largest pool indices.  e4m3: also bit for bit the bf16 kernel on the dequantized pool."""
    from ultravox_b200 import ops
    fp8 = kind != "bf16"
    sk, sv = SCALES[int(kind[-1])] if fp8 else (1.0, 1.0)
    Hq, B, lens = HQ8, 2, PAGED_LENS
    n_pages = (32768 if fp8 else 16384) + 1024 + 3
    hot = sorted({p // PAGE for e in lens for p in paged_needles(e)})
    table = paged_table(lens, n_pages, hot, seed=5 + fp8).cuda()
    assert int(table.max()) >= (32768 if fp8 else 16384)
    lens_t = i32(lens)
    what = f"paged decode {kind} n_pages={n_pages}"
    st = Stats(what, D)
    k, v = rows_with_nan_tail(B, lens, seed=11, D=D)
    if fp8:
        kq, vq = quant(k, sk), quant(v, sv)
        k, v = dequant(kq, sk), dequant(vq, sv)                      # what the kernel sees; also the bf16 twin's pool
        pk = torch.full((n_pages, PAGE, HKV, D), NAN_BYTE, dtype=torch.uint8, device="cuda").view(E4M3)
        pv = pk.clone()
        fill_pool(pk, kq, table), fill_pool(pv, vq, table)
        del kq, vq
        scale = torch.tensor([sk, sv], dtype=torch.float32, device="cuda")
        twin_table = torch.arange(B * W, dtype=torch.int32, device="cuda").view(B, W).masked_fill(table < 0, -1)
    else:
        pk = torch.full((n_pages, PAGE, HKV, D), NAN, dtype=BF, device="cuda")
        pv = pk.clone()
        fill_pool(pk, k, table), fill_pool(pv, v, table)
        scale = None
    q = flat(B, Hq * D, seed=12, device="cuda")

    def run(qq=q, rows=None, lt=lens_t):
        out = torch.zeros(B, Hq * D, dtype=BF, device="cuda")
        return ops.attention_paged(qq, pk, pv, out, Hq, D ** -0.5, table, lt, kv_scale=scale, kv_row=rows)

    def twin(qq):
        out = torch.zeros(B, Hq * D, dtype=BF, device="cuda")
        return ops.attention_paged(qq, k.view(B * W, PAGE, HKV, D), v.view(B * W, PAGE, HKV, D), out, Hq, D ** -0.5, twin_table,
                                   lens_t)

    if check_dispatch:
        assert_kernel(run, f"attn_fwd_kernel<{D}, true, {'true' if fp8 else 'false'}>")
    out = twice(run)
    for b in range(B):
        st.check(out[b:b + 1], q[b], k[b], v[b], 0, lens[b], what=f"flat row {b}")
    if fp8:
        assert torch.equal(twin(q), out), (what, "fp8 != bf16 on the dequantized pool")
    # the kv_row form: query rows swapped, reading the table rows swapped, give the output rows swapped
    assert torch.equal(run(qq=q[[1, 0]], rows=i32([1, 0]), lt=i32(lens[::-1])), out[[1, 0]]), (what, "kv_row form")
    # row isolation: new values in row 1's pages change no bit of row 0
    pages1 = table[1][table[1] >= 0].long()
    keep = pk[pages1].clone(), pv[pages1].clone()
    pk[pages1] = (flat(len(pages1), PAGE, HKV, D, seed=13, device="cuda").float() / sk).to(pk.dtype)
    o2 = run()
    assert torch.equal(o2[0], out[0]) and not torch.equal(o2[1], out[1]), (what, "row isolation")
    pk[pages1], pv[pages1] = keep
    del keep
    # needle in the pages with the largest pool indices
    qn = needle_q(B, Hq, D, "cuda", needle)
    G = Hq // HKV
    needle_byte = quant(torch.tensor(needle, device="cuda"), sk) if fp8 else None
    for b in range(B):
        for p in paged_needles(lens[b]):
            pg, off = page_of(table, b, p)
            saved = pk[pg, off].clone(), k[b, p].clone()
            if fp8:
                pk[pg, off] = needle_byte
                k[b, p] = dequant(needle_byte, sk)
            else:
                pk[pg, off] = needle
                k[b, p] = needle
            assert needle_gap(k[b], p, 0, lens[b], D, needle) > NEEDLE_GAP
            got = run(qq=qn)
            assert torch.equal(got[b], v[b, p].repeat_interleave(G, 0).reshape(-1)), (what, f"needle row {b} at {p} page {pg}")
            if fp8:
                assert torch.equal(twin(qn), got), (what, "needle: fp8 != bf16 twin", b, p)
            pk[pg, off], k[b, p] = saved
    # sink + recency
    qs = q.clone()
    for b in range(B):
        sink_recency(qs[b:b + 1], k[b], 0, lens[b], Hq, D)
        pos = [0] + list(range(lens[b] - 256, lens[b]))
        if fp8:
            k[b, pos] = dequant(quant(k[b, pos], sk), sk)            # the sink / band values as the pool holds them
        put_keys(pk, table[b], pos, k[b, pos], sk if fp8 else None)
    out = twice(lambda: run(qq=qs))
    for b in range(B):
        st.check(out[b:b + 1], qs[b], k[b], v[b], 0, lens[b], what=f"sink row {b}")
    if fp8:
        assert torch.equal(twin(qs), out), (what, "sink: fp8 != bf16 twin")
    st.report()


# ================================================================================================ 4. chunk forms
def chunk_pasts(C):
    return 8191, 65536, SMAX - C


@pytest.mark.parametrize("kind", ["contiguous", "paged-bf16", "paged-fp8"])
@pytest.mark.parametrize("C", [64, 70, 248])
def test_chunk_long_past(kind, C):
    """One prompt chunk of C queries on ``attn_wg_kernel`` after past in {8191, 65536, 131072 - C} cached keys: the slot cache
    (``attention_indexed``, cache row 1 of 2) or a 2048-entry table into a > 16384-page bf16 / > 32768-page e4m3 pool
    (``attention_indexed_paged``).  Everything the chunk may not read - the other cache row or the other table row's pages,
    positions >= past + C - is NaN / +-Inf."""
    from ultravox_b200 import ops
    Hq, j = HQ8, 1
    paged, fp8 = kind != "contiguous", kind == "paged-fp8"
    sk, sv = SCALES[[64, 70, 248].index(C)] if fp8 else (1.0, 1.0)
    n_pages = (32768 if fp8 else 16384) + 1024 + 3
    what = f"chunk {kind} C={C}"
    st = Stats(what)
    G = Hq // HKV
    scale = torch.tensor([sk, sv], dtype=torch.float32, device="cuda") if fp8 else None
    if paged:
        pk = torch.full((n_pages, PAGE, HKV, HD), NAN_BYTE if fp8 else 0, dtype=torch.uint8 if fp8 else BF, device="cuda")
        pk = pk.view(E4M3) if fp8 else pk.fill_(NAN)
        pv = pk.clone()
    kern = "attn_wg_kernel<128, true, " + ("false, false>" if not paged else "true, true>" if fp8 else "true, false>")
    for past in chunk_pasts(C):
        end = past + C
        seed = 100 * C + past
        k, v = rows_with_nan_tail(1, [end], seed=seed)
        if fp8:
            k, v = dequant(quant(k, sk), sk), dequant(quant(v, sv), sv)
        q = flat(1, C, Hq * HD, seed=seed + 2, device="cuda")
        args = (i32([j]), i32([past]), i32([end]))
        needles = sorted(p for p in {0, 63, 64, PAGE * 1023 + 5, past // 2 + 1, past - 1, PAGE * ((end - 1) // PAGE), end - 1}
                         if p < end)
        if paged:
            hot = sorted({p // PAGE for p in needles})
            table = paged_table([SMAX, end], n_pages, hot, seed=seed).cuda()       # row 0: another slot's pages, all NaN
            assert int(table.max()) >= (32768 if fp8 else 16384)
            if fp8:
                pk.view(torch.uint8).fill_(NAN_BYTE), pv.view(torch.uint8).fill_(NAN_BYTE)
                fill_pool(pk, quant(k, sk), table[1:]), fill_pool(pv, quant(v, sv), table[1:])
            else:
                pk.fill_(NAN), pv.fill_(NAN)
                fill_pool(pk, k, table[1:]), fill_pool(pv, v, table[1:])

            def put(p, val):                    # key rows p (bf16 values) into the pool and the reference rows
                k[0, p] = dequant(quant(val, sk), sk) if fp8 else val
                put_keys(pk, table[1], p, k[0, p], sk if fp8 else None)
        else:
            kc = torch.cat([flat(1, SMAX, HKV, HD, seed=seed + 3, device="cuda"), k.nan_to_num(0.0)])
            vc = torch.cat([flat(1, SMAX, HKV, HD, seed=seed + 4, device="cuda"), v.nan_to_num(0.0)])
            kc[1, end:] = flat(SMAX - end, HKV, HD, seed=seed + 5, device="cuda")
            vc[1, end:] = flat(SMAX - end, HKV, HD, seed=seed + 6, device="cuda")
            k, v = kc[1:], vc[1:]

            def put(p, val):
                k[0, p] = val

        def run(qq=q):
            out = torch.zeros(1, C, Hq * HD, dtype=BF, device="cuda")
            if paged:
                return ops.attention_indexed_paged(qq, pk, pv, out, Hq, HD ** -0.5, table, *args, kv_scale=scale)[0]
            return ops.attention_indexed(qq, kc, vc, out, Hq, HD ** -0.5, *args)[0]

        def twin(qq):
            out = torch.zeros(1, C, Hq * HD, dtype=BF, device="cuda")
            t2 = torch.arange(W, dtype=torch.int32, device="cuda").view(1, W).masked_fill(table[1:] < 0, -1)
            return ops.attention_indexed_paged(qq, k[0].view(W, PAGE, HKV, HD), v[0].view(W, PAGE, HKV, HD), out, Hq, HD ** -0.5,
                                               t2, i32([0]), *args[1:])[0]

        if past == chunk_pasts(C)[0]:
            assert_kernel(run, kern)
        out = twice(run)
        st.check(out, q[0], k[0], v[0], 0, end, shift=past, what=f"flat past={past}")
        if fp8:
            assert torch.equal(twin(q), out), (what, past, "fp8 != bf16 on the dequantized pool")
        if not paged:                             # the other cache row and positions >= end: NaN / +-Inf change no bit
            kp, vp = poison_outside(kc, vc, [SMAX, 0], [SMAX, end])
            o2 = torch.zeros(1, C, Hq * HD, dtype=BF, device="cuda")
            assert torch.equal(ops.attention_indexed(q, kp, vp, o2, Hq, HD ** -0.5, *args)[0], out), (what, past, "masked read")
            del kp, vp
        # needle: every query that sees it returns its V row bit for bit
        qn = needle_q(C, Hq, HD, "cuda").view(1, C, -1)
        for p in needles:
            k0 = k[0, p].clone()
            put(p, torch.full_like(k0, NEEDLE_Q))
            assert needle_gap(k[0], p, 0, end) > NEEDLE_GAP
            got = run(qq=qn)
            first = max(0, p - past)                # query i sees keys <= past + i
            want = v[0, p].repeat_interleave(G, 0).reshape(-1)
            bad = [i for i in range(first, C) if not torch.equal(got[i], want)]
            assert not bad, (what, f"past={past} needle at {p}", bad[:8])
            if fp8:
                assert torch.equal(twin(qn), got), (what, "needle: fp8 != bf16 twin", past, p)
            put(p, k0)
        # sink + recency
        qs = q.clone()
        ks = k[0].clone()
        sink_recency(qs[0], ks, 0, end, Hq, HD)
        pos = [0] + list(range(end - 256, end))
        put(pos, ks[pos])
        out = twice(lambda: run(qq=qs))
        st.check(out, qs[0], k[0], v[0], 0, end, shift=past, what=f"sink past={past}")
        if fp8:
            assert torch.equal(twin(qs), out), (what, past, "sink: fp8 != bf16 twin")
        del k, v
        if not paged:
            del kc, vc
    st.report()


# ================================================================================================ 5. prefill on a cache
@pytest.mark.parametrize("left_pad", [False, True])
@pytest.mark.parametrize("Sq", [70, 201])
def test_prefill_on_long_cache(Sq, left_pad):
    """``ops.attention`` with Sq queries causal on top of a 32768-key cache (shift = Skv - Sq) on the wgmma kernel, B = 2, kv_start
    {0, 20001} with left padding."""
    Hq, B, Skv = HQ8, 2, 32768
    past = Skv - Sq
    starts = [0, 20001] if left_pad else [0, 0]
    start_t = i32(starts) if left_pad else None
    seed = Sq + 7 * left_pad
    kc, vc = flat(B, Skv, HKV, HD, seed=seed, device="cuda"), flat(B, Skv, HKV, HD, seed=seed + 1, device="cuda")
    q = flat(B * Sq, Hq * HD, seed=seed + 2, device="cuda")
    what = f"prefill on cache Sq={Sq} Skv={Skv} starts={starts}"
    st = Stats(what)
    G = Hq // HKV

    def run(qq=q, k=kc, v=vc):
        from ultravox_b200 import ops
        out = torch.empty(B * Sq, Hq * HD, dtype=BF, device="cuda")
        rs, cs = Hq * HD, Skv * HKV * HD
        return ops.attention(qq.data_ptr(), k.data_ptr(), v.data_ptr(), out, B, Hq, HKV, Sq, Skv, HD,
                             (rs, Sq * rs, HKV * HD, cs, HKV * HD, cs, rs, Sq * rs), HD ** -0.5, True, None, 0, start_t)
    assert_kernel(run, "attn_wg_kernel<128, false, false, false>")
    out = twice(run)
    for b in range(B):
        st.check(out[b * Sq:(b + 1) * Sq], q[b * Sq:(b + 1) * Sq], kc[b], vc[b], starts[b], Skv, shift=past, what=f"flat row {b}")
    kp, vp = poison_outside(kc, vc, starts, [Skv] * B)
    assert torch.equal(run(k=kp, v=vp), out), (what, "reads a masked cache position")
    kp[0], vp[0] = flat(Skv, HKV, HD, seed=seed + 3, device="cuda"), flat(Skv, HKV, HD, seed=seed + 4, device="cuda")
    o2 = run(k=kp, v=vp)
    assert torch.equal(o2[Sq:], out[Sq:]) and not torch.equal(o2[:Sq], out[:Sq]), (what, "row isolation")
    del kp, vp
    qn = needle_q(B * Sq, Hq, HD, "cuda")
    for b in range(B):
        for p in sorted({0, 63, 64, starts[b], 16000 + 17, past - 1, Skv - 1}):
            if p < starts[b]:
                continue
            k0 = kc[b, p].clone()
            plant_needle(kc[b], p)
            assert needle_gap(kc[b], p, starts[b], Skv) > NEEDLE_GAP
            got = run(qq=qn)[b * Sq:(b + 1) * Sq]
            want = vc[b, p].repeat_interleave(G, 0).reshape(-1)
            bad = [i for i in range(max(0, p - past), Sq) if not torch.equal(got[i], want)]
            assert not bad, (what, f"needle row {b} at {p}", bad[:8])
            kc[b, p] = k0
    qs, ks = q.clone(), kc.clone()
    for b in range(B):
        sink_recency(qs[b * Sq:(b + 1) * Sq], ks[b], starts[b], Skv, Hq, HD)
    out = twice(lambda: run(qq=qs, k=ks))
    for b in range(B):
        st.check(out[b * Sq:(b + 1) * Sq], qs[b * Sq:(b + 1) * Sq], ks[b], vc[b], starts[b], Skv, shift=past, what=f"sink row {b}")
    st.report()
