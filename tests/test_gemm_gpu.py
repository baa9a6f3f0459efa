"""Per-element parity of the tensor-core GEMM (``uvx_gemm_bf16``, gemm_tc.cu) in every dispatch form and epilogue, at the shapes
inference and training run (DESIGN section 5).

Every call goes through ``ops.linear`` / ``ops.linear_tiled`` / ``ops.conv1d_k3`` / ``ops.gemm_raw``; the ``uvx_debug_gemm_*``
hooks force tile configurations, split counts, cluster shapes, the single-pass form and the register epilogue where a case needs
them.  Every call asserts the kernels it ran (``torch.profiler`` CUDA activity): a change in ``pick_cfg`` that moves a case onto
another path fails here instead of silently testing something else.  Widths: Whisper-large-v3 (d 1280, ffn 5120, 128 mel,
T = 3000 -> 1500), Llama-3.1-8B (d 4096, 32 / 8 heads of 128, ffn 14336, V 128256) and Llama-3.3-70B (d 8192, 64 / 8 heads,
ffn 28672).

Two input regimes; each case runs in both unless its docstring says otherwise.

* ``exact``: integer-valued bf16 entries in [-4, 4], every A row and every W row scaled by its own power of two in 2^-6 .. 2^6.
  Every product of output (m, n) is then an integer multiple of 2^(e_m + e_n), and ``exact_acc`` asserts that the sum of their
  magnitudes stays below 2^24 such units: every fp32 addition is exact in any order (the tensor core's, the split-K reduce's),
  so the accumulator equals the fp64 matmul.  The epilogue is modelled at its documented rounding points (alpha, bias, residual
  in fp32, one bf16 round-to-nearest-even at the store; SwiGLU and RoPE round the projection to bf16 first; the RoPE rotation
  without FMA) and the output must match **bit for bit**.  Alpha is a power of two here (``acc * alpha + x`` may be contracted
  to an FMA, which only a power-of-two alpha makes order-free).  GELU and SiLU are approximations (``gelu_fast``, ``gelu_erf``
  in the split-K reduce, ``silu_fast``): GELU outputs are checked against the exact function within ``gelu_bound``, SwiGLU
  outputs may differ only where bf16(silu(gate)) lands on a neighbouring bf16 value because silu(gate) lies within 2^-19 of
  the rounding boundary.
* ``round``: seeded normal bf16 data at model scales, including non-power-of-two alpha.  Per element
  |got - ref64| <= ulp(ref) + gamma'(4 ceil(K / 16) + S + 3) (|alpha| sum_k |a w| + |bias| + |res|), gamma'(n) = n 2^-23 /
  (1 - n 2^-23), with S = 16 (no dispatch here picks more splits).  The rounding steps are counted per k16 MMA chunk, not per
  scalar, and 2^-23 covers tensor cores that truncate instead of rounding.  At K = 14336 the bound is about 4 sigma_a sigma_w;
  one dropped k-block moves an output by about 8 sigma_a sigma_w.  It catches precision losses integers cannot see (partials
  rounded through bf16, a reduced-precision accumulation).  GELU adds ``gelu_bound`` and its slope (at most 1.13) on the
  gamma' term; RoPE and SwiGLU add the bf16 rounding of the projection they rotate or multiply.

Bit-level contracts, exact regime: everything outside the output window keeps a sentinel (guard rows, columns past N, rows the
row map drops, ``norm_out`` rows past M); the split-K workspace is filled with NaN before every call; an in-place residual gives
the out-of-place bits; a change to one clip's input changes no bit of another clip's output; two runs give identical bits.

``UVX_GEMM_RATIO_LOG=<file>`` writes the largest error / bound ratio of every rounding-regime case there as JSON."""
import contextlib
import json
import math
import os

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U23 = 2.0 ** -23
S_MAX = 16            # largest split count a dispatch picks (pick_cfg caps at 16; the forced cases here use at most 7)
GELU_AS = 7.5e-8      # A&S 7.1.26: |erf error| <= 1.5e-7, i.e. |Phi error| <= 7.5e-8
SENT = -1984.0        # sentinel, exact in bf16
REGIMES = ("exact", "round")
RATIOS: dict = {}

W8B = dict(d=4096, Hq=32, Hkv=8, ffn=14336)
W70B = dict(d=8192, Hq=64, Hkv=8, ffn=28672)
V_LLM = 128256


# ================================================================================================ reference helpers (pure torch)
def gamma_p(n):
    return n * U23 / (1 - n * U23)


def bf16_ulp(ref: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 (8 significant bits) at |ref|; the smallest normal spacing at 0."""
    _, e = torch.frexp(ref.double())
    return torch.ldexp(torch.ones_like(ref, dtype=F64), (e - 8).clamp_min(-133).to(torch.int32))


def exact_acc(A: torch.Tensor, W: torch.Tensor, a_unit: torch.Tensor, w_unit: torch.Tensor) -> torch.Tensor:
    """fp64 A @ W.T for A [M, K], W [N, K] whose rows are integer multiples of a_unit [M] / w_unit [N] (powers of two).  Asserts
    the exact-sum precondition: sum_k |a w| < 2^24 units of a_unit[m] * w_unit[n] for every output, so every partial sum in any
    order is an fp32 number and the fp32 accumulator equals this result."""
    ai = A.double() / a_unit.double()[:, None]
    wi = W.double() / w_unit.double()[:, None]
    assert torch.equal(ai, ai.round()) and torch.equal(wi, wi.round()), "operands are not integer multiples of their units"
    # sum_k |a_k w_k| <= min(|a|_1 |w|_inf, |a|_inf |w|_1), per output
    mag = torch.minimum(ai.abs().sum(1)[:, None] * wi.abs().amax(1)[None, :], ai.abs().amax(1)[:, None] * wi.abs().sum(1)[None, :])
    assert float(mag.max()) < 2.0 ** 24, f"exact-sum precondition broken: a partial sum may reach {float(mag.max()):.3g} units"
    acc = A.double() @ W.double().T
    assert torch.equal(acc.float().double(), acc)
    return acc


def rope_emul(x1, x2, c, s):
    """uvx rope_pair in fp32 with every product and sum rounded (no FMA): o1 = x1 c - x2 s, o2 = x2 c + x1 s."""
    x1, x2, c, s = x1.float(), x2.float(), c.float(), s.float()
    return x1 * c - x2 * s, x2 * c + x1 * s


def gelu64(v):
    v = v.double()
    return 0.5 * v * (1.0 + torch.erf(v * (0.5 ** 0.5)))


def gelu_bound(v):
    """|gelu_fast(v) - gelu(v)| in fp32 (and gelu_erf's, far smaller): the A&S 7.1.26 term 7.5e-8 |v|; the fp32 roundings of
    1 - erfc / 2 and of the final product, 2^-23 |v|; the ex2 / rcp approximations and the roundings of the polynomial,
    relative 2^-20 on the x * erfc / 2 term, whose exponent argument -z^2 / ln 2 is itself rounded (relative z^2 2^-23)."""
    v = v.double().abs()
    half_erfc = 0.5 * torch.special.erfc(v * (0.5 ** 0.5))
    return v * (GELU_AS + U23 + half_erfc * (2.0 ** -20) * (1.0 + v * v))


def gelu_fast_emul(x: np.ndarray) -> np.ndarray:
    """gelu_fast of uvx_common.cuh in numpy float32 (exact reciprocal and exp2 in place of rcp.approx / ex2.approx)."""
    x = x.astype(np.float32)
    z = np.abs(x) * np.float32(0.70710678118654752440)
    t = np.float32(1.0) / (np.float32(0.3275911) * z + np.float32(1.0))
    pl = np.float32(1.061405429) * t + np.float32(-1.453152027)
    pl = pl * t + np.float32(1.421413741)
    pl = pl * t + np.float32(-0.284496736)
    pl = pl * t + np.float32(0.254829592)
    ex = np.exp2(np.float32(-1.4426950408889634) * z * z).astype(np.float32)
    he = np.float32(0.5) * pl * t * ex
    return (x * np.where(x >= 0, np.float32(1.0) - he, he)).astype(np.float32)


def bf16_neighbours(x: torch.Tensor):
    """(next lower, next higher) bf16 values of the bf16 tensor x."""
    b = x.contiguous().view(torch.int16).to(torch.int32)
    up = torch.where(x >= 0, b + 1, b - 1)
    dn = torch.where(x > 0, b - 1, torch.where(x == 0, torch.full_like(b, -32767), b + 1))   # below +0 is the smallest -denormal
    to = lambda t: t.to(torch.int16).view(BF)
    return torch.minimum(to(up), to(dn)), torch.maximum(to(up), to(dn))


def swiglu_exact_ok(got, gate_b, up_b):
    """True where got is bf16(bf16(silu(gate)) * up) with silu rounded to its bf16 value, or to a neighbour when silu(gate) lies
    within 2^-19 relative of the boundary between them (silu_fast's ex2 / rcp error is near 2^-21); gates below -80 may give 0
    (the ex2 argument overflows, rcp.approx.ftz flushes)."""
    g = gate_b.double()
    s64 = g * torch.sigmoid(g)
    s0 = s64.to(BF)
    lo, hi = bf16_neighbours(s0)
    tol = (2.0 ** -19) * s64.abs() + 1e-40
    ok = got == (s0.float() * up_b.float()).to(BF)
    for nb in (lo, hi):
        mid = (s0.double() + nb.double()) / 2
        ok |= ((s64 - mid).abs() <= tol) & (got == (nb.float() * up_b.float()).to(BF))
    ok |= (g < -80) & (got == 0)
    return ok


def locate(bad: torch.Tensor, shape, tile, K):
    i = int(torch.nonzero(bad.reshape(-1))[0])
    idx = np.unravel_index(i, shape)
    b, m, n = (0,) * (3 - len(idx)) + tuple(int(t) for t in idx)
    bm, bn = tile
    return i, f"(batch {b}, row {m}, col {n}), tile ({m // bm}, {n // bn}) of {bm} x {bn}, k-range [0, {K})"


def assert_exact(got, want, what, K, tile=(128, 128)):
    bad = got != want
    if bool(bad.any()):
        i, where = locate(bad, tuple(got.shape), tile, K)
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} outputs differ; first at {where}: got "
                             f"{float(got.reshape(-1)[i])!r} want {float(want.reshape(-1)[i])!r}")


def assert_within(got, ref, bound, what, K, tile=(128, 128)):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i, where = locate(bad, tuple(got.shape), tile, K)
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} outputs out of bound; first at {where}: got "
                             f"{float(got.reshape(-1)[i])!r} ref {float(ref.reshape(-1)[i])!r} bound {float(bound.reshape(-1)[i])!r}")
    return float((err / bound.clamp_min(1e-300)).max())


# ================================================================================================ CPU self-tests of the helpers
def test_exact_precondition_and_refusal():
    g = torch.Generator().manual_seed(0)
    A = torch.randint(-4, 5, (3, 40), generator=g).double() * torch.tensor([2.0 ** -6, 1.0, 2.0 ** 6])[:, None]
    W = torch.randint(-4, 5, (5, 40), generator=g).double() * torch.tensor([2.0 ** 6, 2.0 ** -6, 1.0, 0.5, 4.0])[:, None]
    acc = exact_acc(A.to(BF), W.to(BF), torch.tensor([2.0 ** -6, 1.0, 2.0 ** 6]), torch.tensor([2.0 ** 6, 2.0 ** -6, 1.0, 0.5, 4.0]))
    assert torch.equal(acc, A @ W.T)
    # 2^20 terms of 4 * 4 reach 2^24: refused
    big = torch.full((1, 1 << 20), 4.0, dtype=BF)
    with pytest.raises(AssertionError, match="precondition"):
        exact_acc(big, big, torch.ones(1), torch.ones(1))
    # just below the limit is accepted, and the sum is an fp32 number
    ok = torch.full((1, (1 << 20) - 8), 4.0, dtype=BF)
    assert float(exact_acc(ok, ok, torch.ones(1), torch.ones(1))) == 16.0 * ((1 << 20) - 8)
    # entries that are not multiples of the stated unit are refused
    with pytest.raises(AssertionError, match="integer multiples"):
        exact_acc(torch.full((1, 8), 0.5, dtype=BF), torch.ones(1, 8, dtype=BF), torch.ones(1), torch.ones(1))


def test_bf16_round_to_nearest_even_ties():
    """The reference rounds to bf16 with torch's cast; it must be round-to-nearest-even at ties, as __float2bfloat16_rn is."""
    x = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, 257.0, 259.0, -257.0, -259.0, 2 ** -126 * (1 + 2 ** -8), 1 + 2 ** -8 + 2 ** -20],
                     dtype=F32)
    want = torch.tensor([1.0, 1 + 2 ** -6, 256.0, 260.0, -256.0, -260.0, 2 ** -126, 1 + 2 ** -7], dtype=F64)
    assert torch.equal(x.to(BF).double(), want)
    # integer data gives ties: an odd integer of 9 significant bits
    odd = torch.arange(257, 513, 2, dtype=F32)
    r = odd.to(BF).double()
    assert bool(((r - odd.double()).abs() == 1).all()) and bool((torch.remainder(r, 4) == 0).all())
    lo, hi = bf16_neighbours(torch.tensor([1.0, -1.0, 0.0], dtype=BF))
    assert lo.double().tolist() == [1 - 2 ** -8, -1 - 2 ** -7, -(2.0 ** -133)]
    assert hi.double().tolist() == [1 + 2 ** -7, -1 + 2 ** -8, 2.0 ** -133]


def test_rope_emulation_against_fp64():
    c = torch.tensor([1.0, 0.0, 0.5, math.cos(1.0), math.cos(1e5)], dtype=F32)
    s = torch.tensor([0.0, 1.0, math.sqrt(0.75), math.sin(1.0), math.sin(1e5)], dtype=F32)
    x1 = torch.tensor([3.0, 3.0, 1.5, -2.25, 100.0], dtype=BF)
    x2 = torch.tensor([-5.0, -5.0, 0.75, 7.0, -0.125], dtype=BF)
    o1, o2 = rope_emul(x1, x2, c, s)
    assert o1[:2].tolist() == [3.0, 5.0] and o2[:2].tolist() == [-5.0, 3.0]            # identity and a quarter turn are exact
    c64, s64, a, b = c.double(), s.double(), x1.double(), x2.double()
    r1, r2 = a * c64 - b * s64, b * c64 + a * s64
    tol = U23 * (a.abs() * c64.abs() + b.abs() * s64.abs())                               # three fp32 roundings
    assert bool(((o1.double() - r1).abs() <= tol).all()) and bool(((o2.double() - r2).abs() <= tol).all())
    # no FMA: x1 c - x2 s with the products rounded first differs from the fused form here
    x1b, x2b = torch.tensor([1 + 2 ** -7], dtype=BF), torch.tensor([1.0], dtype=BF)
    cb, sb = torch.tensor([1 + 2 ** -23]), torch.tensor([1 + 2 ** -7 + 2 ** -23])
    o1b, _ = rope_emul(x1b, x2b, cb, sb)
    fused = (1 + 2 ** -7) * (1 + 2 ** -23) - (1 + 2 ** -7 + 2 ** -23)
    assert float(o1b) == 0.0 and fused != 0.0


def test_gelu_bound_against_scipy_erf():
    """gelu_fast's formula (in fp32, exact exp2 / reciprocal) stays within gelu_bound of x Phi(x) with scipy's erf over the bf16
    grid in [-20, 20]; the reference's torch erf agrees with scipy's."""
    from scipy.special import erf
    bits = np.arange(0, 1 << 16, dtype=np.uint32).astype(np.uint32) << 16
    x = bits.view(np.float32)
    x = np.unique(x[np.isfinite(x) & (np.abs(x) <= 20)])
    exact = 0.5 * x.astype(np.float64) * (1.0 + erf(x.astype(np.float64) / math.sqrt(2.0)))
    got = gelu_fast_emul(x).astype(np.float64)
    bound = gelu_bound(torch.from_numpy(x.astype(np.float64))).numpy()
    ratio = np.abs(got - exact) / np.maximum(bound, 1e-300)
    assert ratio.max() <= 1.0, float(x[ratio.argmax()])
    assert ratio.max() > 0.25                     # and not vacuous: 0.58 of it is reached (at x = 3.02)
    assert np.abs(gelu64(torch.from_numpy(x.astype(np.float64))).numpy() - exact).max() <= 1e-15 * max(1.0, np.abs(exact).max())


def test_swiglu_acceptance_is_tight():
    gate = torch.tensor([0.5, 3.0, -2.0, -90.0, 1.0], dtype=BF)
    up = torch.tensor([2.0, -1.5, 4.0, 3.0, 1.0], dtype=BF)
    s = (gate.double() * torch.sigmoid(gate.double())).to(BF)
    want = (s.float() * up.float()).to(BF)
    assert bool(swiglu_exact_ok(want, gate, up)[:3].all())
    lo, hi = bf16_neighbours(s)
    off = (hi.float() * up.float()).to(BF)
    assert not bool(swiglu_exact_ok(off, gate, up)[:3].any())     # a neighbour far from the boundary is refused
    assert bool(swiglu_exact_ok(torch.zeros(5, dtype=BF), gate, up)[3])


# ================================================================================================ GPU fixtures and drivers
@pytest.fixture(scope="module")
def ops():
    from ultravox_b200 import ops as o
    return o


@pytest.fixture(autouse=True, scope="module")
def _fp64_refs():
    """References are fp64 matmuls; the magnitudes sum_k |a w| run in TF32, which holds bf16 magnitudes exactly."""
    prev = torch.backends.cuda.matmul.allow_tf32
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev
    path = os.environ.get("UVX_GEMM_RATIO_LOG")
    if path and RATIOS:
        with open(path, "w") as f:
            json.dump(RATIOS, f, indent=1, sort_keys=True)


def record(request, r):
    key = request.node.name
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)


@contextlib.contextmanager
def hooks(cfg=0, splits=0, cm=0, cn=0, store=-1, ws=-1):
    from ultravox_b200 import _lib
    lib = _lib.lib()
    lib.uvx_debug_gemm_override(cfg, splits)
    lib.uvx_debug_gemm_cluster(cm, cn)
    lib.uvx_debug_gemm_tma_store(store)
    lib.uvx_debug_gemm_ws(ws, 0, 0)
    try:
        yield
    finally:
        lib.uvx_debug_gemm_override(0, 0)
        lib.uvx_debug_gemm_cluster(0, 0)
        lib.uvx_debug_gemm_tma_store(-1)
        lib.uvx_debug_gemm_ws(-1, 0, 0)


def short(name: str) -> str:
    """'void uvx::gemm_wg_kernel<1, 128, true>(CUtensorMap_st, ...)' -> 'gemm_wg_kernel<1, 128, true>'."""
    head = name.split("(")[0]
    head = head[5:] if head.startswith("void ") else head
    base, _, tmpl = head.partition("<")
    return base.split("::")[-1] + ("<" + tmpl if tmpl else "")


def run(ops, fn, expect, twice=True):
    """fn() -> tuple of fresh output tensors.  The split-K workspace is filled with NaN before each call; the first call runs under
    the profiler and exactly the kernels in ``expect`` must have run; the second must give the same bits.  ``expect=None``: the
    first call is not profiled (for callers that assert the dispatch of the same call in a process of its own)."""
    from torch.profiler import ProfilerActivity, profile
    if expect is None:
        ops.gemm_workspace(torch.device("cuda")).fill_(255)
        out = fn()
    for _ in range(8 if expect is not None else 0):
        ops.gemm_workspace(torch.device("cuda")).fill_(255)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        ran = sorted({short(e.name) for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and "uvx::" in e.name})
        if set(expect) <= set(ran):    # now and then the profiler drops some or all records of a window: profile the call again
            break
    if expect is not None:
        assert ran == sorted(set(expect)), f"dispatch: ran {ran}, expected {sorted(set(expect))}"
    if twice:
        ops.gemm_workspace(torch.device("cuda")).fill_(255)
        again = fn()
        for i, (a, b) in enumerate(zip(out, again)):
            assert torch.equal(a, b), f"output {i} differs between two identical calls"
    return out


def wg(mt, bn, staged=False):
    return f"gemm_wg_kernel<{mt}, {bn}, {'true' if staged else 'false'}>"


def swap(rows):
    return f"gemm_swap_kernel<{8 if rows <= 8 else 16 if rows <= 16 else 32}>"


RED, RED_NORM, RED_ROPE, NORM = "splitk_reduce_kernel", "splitk_reduce_rmsnorm_kernel", "splitk_reduce_rope_kernel", "rmsnorm_kernel"


class Gen:
    """Seeded device inputs for one regime.  ``exact``: integers in [-4, 4] times a power of two per row (``unit``);
    ``round``: normal values at the given scale."""

    def __init__(self, regime, seed):
        self.exact = regime == "exact"
        self.g = torch.Generator(device="cuda").manual_seed(seed)

    def _ints(self, shape, lim):
        return torch.randint(-lim, lim + 1, shape, generator=self.g, device="cuda").double()

    def mat(self, rows, cols, scale=1.0, elo=-6, ehi=6):
        """-> (bf16 [rows, cols], fp64 unit [rows] or None)."""
        if self.exact:
            unit = torch.exp2(torch.randint(elo, ehi + 1, (rows,), generator=self.g, device="cuda").double())
            return (self._ints((rows, cols), 4) * unit[:, None]).to(BF), unit
        return (torch.randn(rows, cols, generator=self.g, device="cuda") * scale).to(BF), None

    def bias(self, n, w_unit, scale=0.5):
        if self.exact:
            return (self._ints((n,), 64) * w_unit).to(BF)
        return (torch.randn(n, generator=self.g, device="cuda") * scale).to(BF)

    def res(self, m, n, a_unit, w_unit, scale=1.0):
        if self.exact:
            return (self._ints((m, n), 64) * a_unit[:, None] * w_unit[None, :]).to(BF)
        return (torch.randn(m, n, generator=self.g, device="cuda") * scale).to(BF)

    def vec(self, n, scale=1.0):
        return (torch.randn(n, generator=self.g, device="cuda") * scale).to(BF)


def mm_ref(A, W, au, wu):
    """(fp64 A @ W.T, sum_k |a w| or None in the exact regime)."""
    if au is not None:
        return exact_acc(A, W, au, wu), None
    acc = A.double() @ W.double().T
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        mag = (A.abs().float() @ W.abs().float().T).double()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    return acc, mag * (1 + A.shape[1] * 2.0 ** -23)


def epi_model(acc, alpha=1.0, bias=None, res=None, out=BF):
    """The plain epilogue's rounding points in fp32 (exact accumulator): v = acc * alpha (+ bias) (+ res), one rounding to out."""
    v = acc.float() * alpha
    if bias is not None:
        v = v + bias.float()
    if res is not None:
        v = v + res.float()
    return v.to(out)


def check_plain(request, got, acc, mag, K, what, alpha=1.0, bias=None, res=None, gelu=False, tile=(128, 128)):
    """Plain epilogue act(alpha acc + bias) + res against the exact model (bit-exact without GELU) or the per-element bound."""
    if mag is None and not gelu:
        return assert_exact(got, epi_model(acc, alpha, bias, res, got.dtype), what, K, tile)
    if mag is None:                                                       # exact accumulator, GELU: the pre-activation is exact
        v = acc.float() * alpha
        if bias is not None:
            v = v + bias.float()
        v = v.double()
        slack = 0.0
    else:
        alpha = float(torch.tensor(alpha, dtype=F32))                    # the kernel's fp32 alpha
        v = alpha * acc + (bias.double() if bias is not None else 0.0)
        slack = gamma_p(4 * math.ceil(K / 16) + S_MAX + 3) * (abs(alpha) * mag + (bias.double().abs() if bias is not None else 0.0)
                                                            + (res.double().abs() if res is not None else 0.0))
    ref = gelu64(v) if gelu else v
    if res is not None:
        ref = ref + res.double()
    ulp = bf16_ulp(ref) if got.dtype == BF else U23 * ref.abs()
    bound = ulp + (1.13 * slack + gelu_bound(v) if gelu else slack)
    if gelu:
        bound = bound + U23 * ref.abs()                                   # the fp32 sum with the residual
    r = assert_within(got, ref, bound, what, K, tile)
    if mag is not None:
        record(request, r)
    return r


def sentinel(*shape):
    return torch.full(shape, SENT, dtype=BF, device="cuda")


def untouched(t):
    return bool((t == SENT).all())


# ================================================================================================ Whisper encoder (tensor-bound)
@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("M", [1500, 3000])
@pytest.mark.parametrize("layer,N,K", [("qkv", 3840, 1280), ("out", 1280, 1280), ("fc1", 5120, 1280), ("fc2", 1280, 5120)])
def test_whisper_encoder(request, ops, regime, M, layer, N, K):
    """cfg2 encoder linears on the staged epilogue (128 x 128 tiles, shared-memory tile + TMA store, residual by TMA): q|k|v +
    bias, out / fc2 + bias + residual (in place == out of place), fc1 + bias + GELU.  M = 3000 runs the exact regime only."""
    if M == 3000 and regime == "round":
        pytest.skip("two clips: exact regime only")
    gen = Gen(regime, seed=N + K + M)
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    b = gen.bias(N, wu)
    acc, mag = mm_ref(x, w, au, wu)
    exp = [wg(1, 128, True)]
    if layer in ("qkv", "fc1"):
        act = ops.ACT_GELU if layer == "fc1" else ops.ACT_NONE
        (y,) = run(ops, lambda: (ops.linear(x, w, bias=b, act=act),), exp)
        check_plain(request, y, acc, mag, K, layer, bias=b, gelu=layer == "fc1")
    else:
        r = gen.res(M, N, au, wu)
        (y,) = run(ops, lambda: (ops.linear(x, w, bias=b, residual=r),), exp)

        def inplace():
            h = r.clone()
            ops.linear(x, w, bias=b, residual=h, out=h)
            return (h,)
        (h,) = run(ops, inplace, exp)
        assert torch.equal(h, y), "in-place residual differs from out-of-place"
        check_plain(request, y, acc, mag, K, layer, bias=b, res=r)


# ================================================================================================ conv stem (implicit GEMM)
def conv_input(gen, B, T, C):
    """Guard-padded time-major [B, T + 2, C] (rows 0 and T + 1 zero) and, exact regime, each frame's power-of-two unit."""
    if gen.exact:
        e = torch.randint(-2, 3, (B, T + 2), generator=gen.g, device="cuda").double()
        e[:, 0] = e[:, -1] = 2.0
        x = gen._ints((B, T + 2, C), 4) * torch.exp2(e)[..., None]
    else:
        e = None
        x = torch.randn(B, T + 2, C, generator=gen.g, device="cuda").double()
    x[:, 0] = x[:, -1] = 0
    return x.to(BF), e


def im2col(x_tm, e, stride, Tout):
    """Rows of the implicit GEMM: row m of clip b = frames stride*m .. stride*m + 2 of the padded input, flattened."""
    B, Tp, C = x_tm.shape
    A = torch.stack([x_tm[:, stride * torch.arange(Tout, device="cuda") + j] for j in range(3)], 2).reshape(B * Tout, 3 * C)
    if e is None:
        return A, None
    ef = torch.stack([e[:, stride * torch.arange(Tout, device="cuda") + j] for j in range(3)], 2).amin(2)
    return A, torch.exp2(ef).reshape(-1)


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("B,T,store", [(1, 3000, -1), (2, 2999, -1), (2, 3000, 0)])
def test_conv_stem(request, ops, regime, B, T, store):
    """conv1 (K = 3 * 128, GELU, output rows at c_row_offset 1 of [B, T + 2, 1280]: guard rows keep their sentinel) and conv2
    (K = 3 * 1280, stride 2, GELU + the positional embedding broadcast over the clips, r_batch_stride 0) as implicit GEMMs on the
    staged epilogue, and with store = 0 on the register epilogue.  Changing clip 1's input changes no bit of clip 0."""
    if store == 0 and regime == "round":
        pytest.skip("register-epilogue twin: exact regime only")
    gen = Gen(regime, seed=B * 10 + T % 7)
    d, mel = 1280, 128
    staged = store != 0
    # conv1
    x1, e1 = conv_input(gen, B, T, mel)
    w1, wu1 = gen.mat(d, 3 * mel, scale=0.05)
    b1 = gen.bias(d, wu1)
    with hooks(store=store):
        (h1,) = run(ops, lambda: (ops.conv1d_k3(x1, w1, b1, 1, sentinel(B, T + 2, d), out_guard=True),), [wg(1, 128, staged)])
    A, au = im2col(x1, e1, 1, T)
    acc, mag = mm_ref(A, w1, au, wu1)
    assert untouched(h1[:, 0]) and untouched(h1[:, T + 1])
    check_plain(request, h1[:, 1:T + 1].reshape(B * T, d), acc, mag, 3 * mel, "conv1", bias=b1, gelu=True)
    # conv2
    T2 = (T + 1) // 2
    x2, e2 = conv_input(gen, B, T, d)
    w2, wu2 = gen.mat(d, 3 * d, scale=0.02)
    b2 = gen.bias(d, wu2)
    pos = gen.vec(T2 * d).view(T2, d) if not gen.exact else (gen._ints((T2, d), 64) * wu2[None, :] * 0.25).to(BF)
    with hooks(store=store):
        (h2,) = run(ops, lambda: (ops.conv1d_k3(x2, w2, b2, 2, sentinel(B, T2, d), out_guard=False, pos=pos),), [wg(1, 128, staged)])
    A, au = im2col(x2, e2, 2, T2)
    acc, mag = mm_ref(A, w2, au, wu2)
    check_plain(request, h2.reshape(B * T2, d), acc, mag, 3 * d, "conv2", bias=b2, res=pos.repeat(B, 1), gelu=True)
    if B > 1:
        x2b = x2.clone()
        x2b[1] = x2b[1].flip(0)
        with hooks(store=store):
            other = ops.conv1d_k3(x2b, w2, b2, 2, sentinel(B, T2, d), out_guard=False, pos=pos)
        assert torch.equal(other[0], h2[0]) and not torch.equal(other[1], h2[1]), "clip 1's input changed clip 0's output"


# ================================================================================================ batched calls, per-clip residual
@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_batched_per_clip_residual(request, ops, regime):
    """a_batch = 2 through gemm_raw with a residual per clip (r_batch_stride != 0) on the staged epilogue and on the register
    epilogue; each clip's input only moves that clip's bits."""
    gen = Gen(regime, seed=77)
    B, M, N, K = 2, 1500, 1280, 1280
    x, au = gen.mat(B * M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    b = gen.bias(N, wu)
    r = gen.res(B * M, N, au, wu)
    acc, mag = mm_ref(x, w, au, wu)

    def call(xx):
        out = torch.empty(B * M, N, dtype=BF, device="cuda")
        ops.gemm_raw(xx.data_ptr(), B, M, K, K, M * K, w, out, N, M, bias=b, R=r, r_row_stride=N, r_batch_stride=M * N)
        return (out,)
    outs = {}
    for store in (-1, 0):
        with hooks(store=store):
            (outs[store],) = run(ops, lambda: call(x), [wg(1, 128, store != 0)])
    assert torch.equal(outs[-1], outs[0])
    check_plain(request, outs[-1], acc, mag, K, "batched", bias=b, res=r)
    x2 = x.clone()
    x2[M:] = x2[M:].flip(0)
    (y2,) = call(x2)
    assert torch.equal(y2[:M], outs[-1][:M]) and not torch.equal(y2[M:], outs[-1][M:])


# ================================================================================================ Llama prefill, M = 201
def rope_tables(ops, max_pos):
    inv = ops.llama3_inv_freq(128, 500000.0, dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                                  original_max_position_embeddings=8192))
    return ops.rope_tables(inv, max_pos, "cuda")


def check_rope(request, got, acc, mag, K, cos, sin, pos, rope_cols, what):
    """Head columns d and d + 64 of every head below rope_cols rotated by (cos, sin)[pos]; the rest is the bf16 projection."""
    M, N = got.shape
    H = N // 128
    c, s = cos[pos.long()], sin[pos.long()]                                   # [M, 64]
    a = acc.view(M, H, 2, 64)
    g = got.view(M, H, 2, 64)
    rot = torch.arange(H, device="cuda") * 128 < rope_cols
    if mag is None:
        x = a.float().to(BF)                                                  # the projection rounded to bf16 (alpha = 1)
        o1, o2 = rope_emul(x[:, :, 0], x[:, :, 1], c[:, None], s[:, None])
        want = torch.stack([o1, o2], 2).to(BF)
        want = torch.where(rot[None, :, None, None], want, x)
        return assert_exact(got, want.view(M, N), what, K)
    mg = mag.view(M, H, 2, 64)
    c64, s64 = c[:, None].double(), s[:, None].double()
    x1, x2 = a[:, :, 0], a[:, :, 1]
    gm = gamma_p(4 * math.ceil(K / 16) + 3)
    e1, e2 = bf16_ulp(x1) + gm * mg[:, :, 0], bf16_ulp(x2) + gm * mg[:, :, 1]
    r1, r2 = x1 * c64 - x2 * s64, x2 * c64 + x1 * s64
    b1 = bf16_ulp(r1) + c64.abs() * e1 + s64.abs() * e2 + 2 * U23 * (x1.abs() * c64.abs() + x2.abs() * s64.abs())
    b2 = bf16_ulp(r2) + c64.abs() * e2 + s64.abs() * e1 + 2 * U23 * (x2.abs() * c64.abs() + x1.abs() * s64.abs())
    rr = rot[None, :, None]
    ref = torch.stack([torch.where(rr, r1, x1), torch.where(rr, r2, x2)], 2).view(M, N)
    bound = torch.stack([torch.where(rr, b1, bf16_ulp(x1) + gm * mg[:, :, 0]),
                         torch.where(rr, b2, bf16_ulp(x2) + gm * mg[:, :, 1])], 2).view(M, N)
    record(request, assert_within(got, ref, bound, what, K))


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("width", ["8B", "70B"])
@pytest.mark.parametrize("form", ["positions", "pos_offset"])
def test_llama_qkv_rope(request, ops, regime, width, form):
    """q|k|v with the fused RoPE at M = 201: 1 x 128 tiles in 2 x 2 clusters; ``positions`` on the row-major weight,
    ``pos_offset`` (a turn on a kept cache) on the 128-row tiled image.  v heads are the plain bf16 projection."""
    cfg = W8B if width == "8B" else W70B
    M, K = 201, cfg["d"]
    N = (cfg["Hq"] + 2 * cfg["Hkv"]) * 128
    rope_cols = (cfg["Hq"] + cfg["Hkv"]) * 128
    gen = Gen(regime, seed=K + (form == "positions"))
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    cos, sin = rope_tables(ops, 8192)
    acc, mag = mm_ref(x, w, au, wu)
    if form == "positions":
        pos = torch.randint(0, 8000, (M,), generator=gen.g, device="cuda", dtype=torch.int32)
        rope = (cos, sin, pos, M, 0, rope_cols)
        (y,) = run(ops, lambda: (ops.linear(x, w, rope=rope),), [wg(1, 128)])
    else:
        past = 4321
        pos = past + torch.arange(M, device="cuda", dtype=torch.int32)
        rope = (cos, sin, None, M, past, rope_cols)
        tw = ops.TiledWeight(w, 128)
        (y,) = run(ops, lambda: (ops.linear_tiled(x, tw, rope=rope),), [wg(1, 128)])
    check_rope(request, y, acc, mag, K, cos, sin, pos, rope_cols, f"qkv {width} {form}")


def check_norm(h, xn, nw, eps, ops, what):
    """norm_out = w * bf16(h * rsqrt(mean(h^2) + eps)): the same bits as uvx_rmsnorm on the finished rows, and within
    ulp + |w| ulp(h rstd) + 2^-20 |ref| of the fp64 norm of those rows (rstd in fp32 with rsqrtf)."""
    assert torch.equal(xn, ops.rmsnorm(h, nw, eps)), f"{what}: fused norm differs from uvx_rmsnorm on the same rows"
    h64 = h.double()
    rstd = torch.rsqrt((h64 * h64).mean(1, keepdim=True) + eps)
    xh = h64 * rstd
    ref = nw.double() * xh
    bound = bf16_ulp(ref) + nw.double().abs() * bf16_ulp(xh) + 2.0 ** -20 * ref.abs()
    assert_within(xn, ref, bound, what + " norm_out", h.shape[1])


def residual_norm_case(request, ops, gen, M, N, K, call, expect, what, eps=1e-5, prep=None):
    """h <- x @ w.T + h (in place) and norm_out = RMSNorm(h), through ``call(x, prep(w), r, out, norm_w, xn)``; out of place
    gives the same bits; norm_out rows past M keep their sentinel."""
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    r = gen.res(M, N, au, wu)
    nw = gen.vec(N, 0.5) + 1
    acc, mag = mm_ref(x, w, au, wu)
    wo = prep(w) if prep else w

    def inplace():
        h, xn = r.clone(), sentinel(M + 3, N)
        call(x, wo, h, h, nw, xn[:M])
        return h, xn
    h, xn = run(ops, inplace, expect)
    assert untouched(xn[M:]), "norm_out rows past M were written"

    def oop():
        y, xn2 = torch.empty(M, N, dtype=BF, device="cuda"), sentinel(M, N)
        call(x, wo, r, y, nw, xn2)
        return y, xn2
    y, xn2 = run(ops, oop, expect)
    assert torch.equal(y, h) and torch.equal(xn2, xn[:M]), "in-place residual differs from out-of-place"
    check_plain(request, h, acc, mag, K, what, res=r)
    check_norm(h, xn[:M], nw, eps, ops, what)


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("width,N,K,cfg", [("8B o", 4096, 4096, 0), ("70B o", 8192, 8192, 0), ("8B down", 4096, 14336, 0),
                                           ("70B down", 8192, 28672, 0), ("N 8256", 8256, 2048, 3)])
def test_llama_residual_norm(request, ops, regime, width, N, K, cfg):
    """o_proj / down_proj at M = 201: split-K over 256-row tiles, residual in place and the fused RMSNorm in the reduce
    (splitk_reduce_rmsnorm_kernel) up to its N = 8192 limit; N = 8256 (gemm_raw, 3 forced splits) takes the plain reduce and
    then uvx_rmsnorm."""
    if width == "70B down" and regime == "exact":
        pytest.skip("70B down_proj: rounding regime only (the 8B shape covers the same kernels exactly)")
    gen = Gen(regime, seed=N + K)
    M = 201
    if cfg:
        def call(x, w, r, out, nw, xn):
            ops.gemm_raw(x.data_ptr(), 1, M, K, K, 0, w, out, N, M, R=r, r_row_stride=N, norm=(nw, 1e-5, xn))
        with hooks(splits=cfg):
            residual_norm_case(request, ops, gen, M, N, K, call, [wg(2, 64), RED, NORM], width)
        return

    def call(x, tw, r, out, nw, xn):
        ops.linear_tiled(x, tw, residual=r, out=out, norm=(nw, 1e-5, xn))
    residual_norm_case(request, ops, gen, M, N, K, call, [wg(2, 128), RED_NORM], width, prep=lambda w: ops.TiledWeight(w, 128))


def check_swiglu(request, got, acc, mag, K, what, tile=(128, 128)):
    """got [M, F] = bf16(bf16(silu(bf16(gate))) * bf16(up)) from acc [M, 2F] (gate | up row-major halves)."""
    F = got.shape[1]
    g, u = acc[:, :F], acc[:, F:]
    if mag is None:
        ok = swiglu_exact_ok(got, g.float().to(BF), u.float().to(BF))
        if not bool(ok.all()):
            i, where = locate(~ok, tuple(got.shape), tile, K)
            raise AssertionError(f"{what}: {int((~ok).sum())} outputs off; first at {where}: got {float(got.reshape(-1)[i])!r}"
                                 f" gate {float(g.reshape(-1)[i])!r} up {float(u.reshape(-1)[i])!r}")
        return
    sg = g * torch.sigmoid(g)
    ref = sg * u
    gm = gamma_p(4 * math.ceil(K / 16) + 3)
    eg, eu = bf16_ulp(g) + gm * mag[:, :F], bf16_ulp(u) + gm * mag[:, F:]
    bound = bf16_ulp(ref) + u.abs() * (bf16_ulp(sg) + 1.1 * eg + 2.0 ** -20 * sg.abs()) + (sg.abs() + 1.1 * eg) * eu
    record(request, assert_within(got, ref, bound, what, K, tile))


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("R,K,expect", [(128, 4096, wg(2, 128)), (64, 1024, wg(2, 64)), (208, 1024, wg(1, 208)),
                                        (256, 1024, wg(1, 256))])
def test_llama_gate_up_swiglu(request, ops, regime, R, K, expect):
    """8B gate|up (2 x 14336 rows) at M = 201 with silu(gate) * up in the epilogue: the 128-row interleave-16 image on 256 x 128
    tiles, and the interleave-8 images at R = 64 / 208 (ragged last tile) / 256 (clusters on the 1 x R tiles) at K = 1024."""
    gen = Gen(regime, seed=R)
    M, F = 201, W8B["ffn"]
    x, au = gen.mat(M, K)
    w, wu = gen.mat(2 * F, K, scale=0.02)
    acc, mag = mm_ref(x, w, au, wu)
    tw = ops.TiledWeight(w, R, swiglu=True)
    (y,) = run(ops, lambda: (ops.linear_tiled(x, tw, act=ops.ACT_SWIGLU),), [expect])
    check_swiglu(request, y, acc, mag, K, f"gate|up R={R}")


@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_batched_prefill_rope_and_norm(request, ops, regime):
    """4 x 201 rows (more than 256: tensor-bound tiling, no clusters): q|k|v with the fused RoPE over 201-row sequences at
    pos_offset 17, and o_proj + residual with the norm as its own pass (uvx_rmsnorm)."""
    gen = Gen(regime, seed=804)
    M, K, cfg = 4 * 201, W8B["d"], W8B
    N = (cfg["Hq"] + 2 * cfg["Hkv"]) * 128
    rope_cols = (cfg["Hq"] + cfg["Hkv"]) * 128
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    cos, sin = rope_tables(ops, 512)
    acc, mag = mm_ref(x, w, au, wu)
    (y,) = run(ops, lambda: (ops.linear(x, w, rope=(cos, sin, None, 201, 17, rope_cols)),), [wg(1, 128)])
    pos = 17 + torch.arange(M, device="cuda") % 201
    check_rope(request, y, acc, mag, K, cos, sin, pos, rope_cols, "batched qkv")

    def call(x, w, r, out, nw, xn):
        ops.linear(x, w, residual=r, out=out, norm=(nw, 1e-5, xn))
    residual_norm_case(request, ops, gen, M, 4096, K, call, [wg(1, 128), NORM], "batched o_proj")


# ================================================================================================ decode form
@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("K", [4096, 512])
@pytest.mark.parametrize("M", [1, 8, 9, 16, 17, 32])
def test_decode_form(request, ops, regime, K, M):
    """Rows <= 32 on the decode form (128 weight rows on wgmma M, tokens on N: BT 8 / 16 / 32 and their tails): K = 4096 splits
    the weight stream (split-K reduce), K = 512 is one split (the kernel's own epilogue).  Plain, + residual, + bias + GELU,
    q|k|v with RoPE through splitk_reduce_rope_kernel (a turn suffix at pos_offset 3000, or explicit positions for odd M), and
    the fused norm."""
    gen = Gen(regime, seed=M * 7 + K)
    N = 4096
    split = K == 4096
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    b = gen.bias(N, wu)
    r = gen.res(M, N, au, wu)
    acc, mag = mm_ref(x, w, au, wu)
    base = [swap(M)] + ([RED] if split else [])
    (y,) = run(ops, lambda: (ops.linear(x, w),), base)
    check_plain(request, y, acc, mag, K, "decode plain")
    (y,) = run(ops, lambda: (ops.linear(x, w, residual=r),), base)
    check_plain(request, y, acc, mag, K, "decode residual", res=r)
    (y,) = run(ops, lambda: (ops.linear(x, w, bias=b, act=ops.ACT_GELU),), base)
    check_plain(request, y, acc, mag, K, "decode bias+gelu", bias=b, gelu=True)
    # q|k|v with RoPE (8B: 48 heads, 40 rotated)
    Nq, rope_cols = 6144, 40 * 128
    wq, wqu = gen.mat(Nq, K, scale=0.02)
    accq, magq = mm_ref(x, wq, au, wqu)
    cos, sin = rope_tables(ops, 4096)
    if M % 2:
        pos = torch.randint(0, 4000, (M,), generator=gen.g, device="cuda", dtype=torch.int32)
        rope = (cos, sin, pos, 1, 0, rope_cols)
    else:
        pos = 3000 + torch.arange(M, device="cuda", dtype=torch.int32)
        rope = (cos, sin, None, M, 3000, rope_cols)
    (y,) = run(ops, lambda: (ops.linear(x, wq, rope=rope),), [swap(M), RED_ROPE])
    check_rope(request, y, accq, magq, K, cos, sin, pos, rope_cols, "decode rope")

    def call(x, w, r, out, nw, xn):
        ops.linear(x, w, residual=r, out=out, norm=(nw, 1e-5, xn))
    residual_norm_case(request, ops, gen, M, N, K, call, [swap(M), RED_NORM if split else NORM], "decode norm")


# ================================================================================================ row-count switch points
def switch_expect(M, N):
    """Dispatch of a K = 1024 call (16 k-blocks) with M rows on 132 SMs (pick_cfg / pick_cluster / the staged condition)."""
    if M <= 32:
        return [swap(M), RED]
    if M <= 128:
        return [wg(1, 128), RED]
    if M <= 256:
        return [wg(2, 128), RED] if N == 2048 else [wg(1, 128)]          # N = 5120: 1 x 128 tiles in 2 x 2 clusters fill the SMs
    return [wg(1, 64 if N == 2048 else 128, True)]


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("N", [2048, 5120])
@pytest.mark.parametrize("M", [1, 32, 33, 127, 128, 129, 200, 255, 256, 257, 383])
def test_row_switch_points(request, ops, regime, N, M):
    """bias + residual (alpha 0.5 / 0.3) across the switches decode form -> wg form -> MT 2 -> clusters -> staged, with
    the residual in place as well."""
    K = 1024
    gen = Gen(regime, seed=M * 3 + N)
    alpha = 0.5 if gen.exact else 0.3
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    b = gen.bias(N, wu)
    r = gen.res(M, N, au, wu)
    acc, mag = mm_ref(x, w, au, wu)
    exp = switch_expect(M, N)
    (y,) = run(ops, lambda: (ops.linear(x, w, bias=b, residual=r, alpha=alpha),), exp)

    def inplace():
        h = r.clone()
        ops.linear(x, w, bias=b, residual=h, out=h, alpha=alpha)
        return (h,)
    (h,) = run(ops, inplace, exp)
    assert torch.equal(h, y)
    check_plain(request, y, acc, mag, K, f"M={M}", alpha=alpha, bias=b, res=r)


@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_cluster_cta_past_last_row(request, ops, regime):
    """M = 130 on forced 1 x 128 tiles in 2 x 2 clusters: the second m-tile's CTAs load A slices of rows 192 .. 255, wholly past
    the last row (TMA zero fill), and multicast them to their peer."""
    gen = Gen(regime, seed=130)
    M, N, K = 130, 2048, 1024
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    b = gen.bias(N, wu)
    acc, mag = mm_ref(x, w, au, wu)
    with hooks(cfg=1128, splits=1, cm=2, cn=2):
        (y,) = run(ops, lambda: (ops.linear(x, w, bias=b),), [wg(1, 128)])
    check_plain(request, y, acc, mag, K, "M=130 clusters", bias=b)


# ================================================================================================ K and N tails
@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("M", [4, 201])
@pytest.mark.parametrize("K", [8, 24, 64, 72, 200, 1288])
def test_k_tails_nan_windows(request, ops, regime, M, K):
    """K with a partial (or a single) k-block, A and W as column windows of NaN-filled buffers 64 columns wider: TMA's zero fill
    past K must keep every NaN out of the sum.  Decode form at M = 4, 256 x 128 tiles at M = 201; K = 1288 splits."""
    gen = Gen(regime, seed=K + M)
    N = 256
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.05)
    b = gen.bias(N, wu)
    xa = torch.full((M, K + 64), float("nan"), dtype=BF, device="cuda")
    wa = torch.full((N, K + 64), float("nan"), dtype=BF, device="cuda")
    xa[:, :K], wa[:, :K] = x, w
    acc, mag = mm_ref(x, w, au, wu)
    exp = ([swap(M)] if M <= 32 else [wg(2, 128)]) + ([RED] if K == 1288 else [])
    (y,) = run(ops, lambda: (ops.linear(xa[:, :K], wa[:, :K], bias=b),), exp)
    check_plain(request, y, acc, mag, K, f"K={K}", bias=b)


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("case", ["192 on 128 (tiled)", "1984 on 208", "1984 on 208 (tiled)", "64 at 201", "64 at 1500"])
def test_n_tails(request, ops, regime, case):
    """N not a multiple of the tile width (ragged last column tile) and N = 64, written into a buffer 64 columns wider whose extra
    columns keep their sentinel."""
    N, M, K = {"192 on 128 (tiled)": (192, 201, 512), "1984 on 208": (1984, 201, 1024), "1984 on 208 (tiled)": (1984, 201, 1024),
               "64 at 201": (64, 201, 1024), "64 at 1500": (64, 1500, 1024)}[case]
    gen = Gen(regime, seed=N + M)
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.05)
    acc, mag = mm_ref(x, w, au, wu)
    if "tiled" in case:
        tw = ops.TiledWeight(w, 128 if N == 192 else 208)

        def call():
            buf = sentinel(M, N + 64)
            ops.linear_tiled(x, tw, out=buf[:, :N])
            return (buf,)
        exp, tile = ([wg(2, 128)], (256, 128)) if N == 192 else ([wg(1, 208)], (128, 208))
        (buf,) = run(ops, call, exp)
    else:
        def call():
            buf = sentinel(M, N + 64)
            ops.linear(x, w, out=buf[:, :N])
            return (buf,)
        if N == 1984:
            with hooks(cfg=1208):
                (buf,) = run(ops, call, [wg(1, 208)])
            tile = (128, 208)
        else:
            (buf,) = run(ops, call, [wg(2, 64) if M == 201 else wg(1, 64), RED])
            tile = (256, 64) if M == 201 else (128, 64)
    assert untouched(buf[:, N:]), "columns past N were written"
    check_plain(request, buf[:, :N], acc, mag, K, case, tile=tile)


# ================================================================================================ every forced tiling x split count
@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("splits", [1, 3, 7])
@pytest.mark.parametrize("cfg", [1064, 1128, 1208, 1256, 2064, 2128])
def test_forced_tiles_and_splits(request, ops, regime, cfg, splits):
    """M = 201, N = 1024, K = 1000 (16 k-blocks, the last one partial): 3 splits of 6 / 6 / 4 k-blocks, 7 requested -> 6 splits
    of 3 / .. / 1; 208-wide tiles are ragged on N = 1024 and run one split.  bias + residual, MT = 1 tiles in 2 x 2 clusters."""
    gen = Gen(regime, seed=cfg + splits)
    M, N, K = 201, 1024, 1000
    mt, bn = divmod(cfg, 1000)
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.05)
    b = gen.bias(N, wu)
    r = gen.res(M, N, au, wu)
    acc, mag = mm_ref(x, w, au, wu)
    exp = [wg(mt, bn)] + ([RED] if splits > 1 and bn != 208 else [])
    with hooks(cfg=cfg, splits=splits):
        (y,) = run(ops, lambda: (ops.linear(x, w, bias=b, residual=r),), exp)
    check_plain(request, y, acc, mag, K, f"cfg {cfg} splits {splits}", bias=b, res=r, tile=(mt * 128, bn))


# ================================================================================================ training
@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_training_forward_256_wide(request, ops, regime):
    """cfg3 forward rows (2 clips x 201) against a wide weight with K >= 32 k-blocks: 128 x 256 tiles."""
    gen = Gen(regime, seed=402)
    M, N, K = 402, W8B["ffn"], 2048
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    acc, mag = mm_ref(x, w, au, wu)
    (y,) = run(ops, lambda: (ops.linear(x, w),), [wg(1, 256)])
    check_plain(request, y, acc, mag, K, "cfg3 fwd", tile=(128, 256))


@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_lm_head_logits_fp32(request, ops, regime):
    """40 gathered hidden rows against the V = 128256 LM head, fp32 logits (the exact regime: the accumulator itself)."""
    gen = Gen(regime, seed=128)
    M, N, K = 40, V_LLM, W8B["d"]
    x, au = gen.mat(M, K)
    w, wu = gen.mat(N, K, scale=0.02)
    acc, mag = mm_ref(x, w, au, wu)
    (y,) = run(ops, lambda: (ops.linear(x, w, out_dtype=F32),), [wg(1, 128)])
    check_plain(request, y, acc, mag, K, "logits")


@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_wgrad_and_dgrad(request, ops, regime):
    """fc1 weight gradient dW = dy^T x in fp32 over K = 402 tokens (ops.transpose pads to 408: a K tail) on the staged epilogue
    with fp32 panels, and the data gradient dx = dy W against the ops.transpose weight."""
    gen = Gen(regime, seed=5120)
    T, Dout, Din = 402, 5120, 1280
    dyT, dyu = gen.mat(Dout, T)                         # rows of dy^T (the wgrad A) carry the units
    xT, xu = gen.mat(Din, T)
    dy, x = dyT.T.contiguous(), xT.T.contiguous()
    acc, mag = mm_ref(dyT, xT, dyu, xu)
    At, Wt = ops.transpose(dy), ops.transpose(x)
    assert At.shape == (Dout, 408) and bool((At[:, T:] == 0).all())
    (g,) = run(ops, lambda: (ops.linear(At, Wt, out=torch.empty(Dout, Din, dtype=F32, device="cuda")),), [wg(1, 128, True)])
    check_plain(request, g, acc, mag, T, "wgrad")
    # dgrad: dy [T, Dout] @ W1 [Dout, Din] -> W1^T is the GEMM's [Din, Dout] weight
    w1T, w1u = gen.mat(Din, Dout, scale=0.02)
    dy2, dy2u = gen.mat(T, Dout)
    w1 = w1T.T.contiguous()
    acc, mag = mm_ref(dy2, w1T, dy2u, w1u)
    wt = ops.transpose(w1)
    assert torch.equal(wt, w1T)
    (dx,) = run(ops, lambda: (ops.linear(dy2, wt),), [wg(1, 64, True)])
    check_plain(request, dx, acc, mag, Dout, "dgrad", tile=(128, 64))


@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_lm_head_backward_row_map(request, ops, regime):
    """d_hn = dlogits @ lm_head (K = 128256) scattered through a row map with dropped (-1) rows, through split-K: rows the map
    does not name keep their sentinel."""
    gen = Gen(regime, seed=198)
    M, N, K, rows = 40, W8B["d"], V_LLM, 64
    x, au = gen.mat(M, K)
    wT, wu = gen.mat(N, K, scale=0.02)                  # lm_head^T [4096, 128256]
    acc, mag = mm_ref(x, wT, au, wu)
    perm = torch.randperm(rows, generator=torch.Generator().manual_seed(5))[:M].to(torch.int32)
    perm[[3, 17, 39]] = -1
    rmap = perm.cuda()

    def call():
        out = sentinel(rows, N)
        ops.linear(x, wT, out=out, row_map=rmap)
        return (out,)
    (out,) = run(ops, call, [wg(1, 128), RED])
    keep = perm >= 0
    assert untouched(out[sorted(set(range(rows)) - set(perm[keep].tolist()))]), "rows outside the row map were written"
    sel = torch.nonzero(keep).flatten().cuda()
    check_plain(request, out[perm[keep].long().cuda()], acc[sel], None if mag is None else mag[sel], K, "row map")


@gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_lora_merge(request, ops, regime):
    """LoRA merge of the encoder q / k rows: qkv_w[:d] <- base + alpha B A^T with K = 64 (rank 64), alpha = lora_alpha / r
    (2 in the exact regime, 0.3 otherwise), written into a window of the fused [3d, d] weight whose v rows keep their bits."""
    gen = Gen(regime, seed=64)
    d, r = 1280, 64
    alpha = 2.0 if gen.exact else 0.3
    Bq, bu = gen.mat(d, r)
    A, aunit = gen.mat(r, d, scale=0.02)
    At = ops.transpose(A)                                 # [d, 64]
    # the GEMM's W rows are columns of A, which mix the A rows' units: their common unit is the smallest
    wu = None if aunit is None else torch.full((d,), float(aunit.min()), device="cuda", dtype=F64)
    base = gen.res(d, d, bu, wu) if gen.exact else gen.mat(d, d)[0]
    acc, mag = mm_ref(Bq, At, bu, wu)
    vrows = gen.mat(d, d)[0]

    def call():
        qkv = torch.cat([sentinel(2 * d, d), vrows])
        ops.linear(Bq, At, residual=base, out=qkv[:d], alpha=alpha)
        return (qkv,)
    (qkv,) = run(ops, call, [wg(1, 128, True)])
    assert untouched(qkv[d:2 * d]) and torch.equal(qkv[2 * d:], vrows)
    check_plain(request, qkv[:d], acc, mag, r, "lora merge", alpha=alpha, res=base)


# ================================================================================================ opt-in single-pass form
@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("shape", ["qkv", "o", "gate_up", "down"])
def test_single_pass_form(request, ops, regime, shape):
    """uvx_debug_gemm_ws(1): the four 8B prefill shapes at M = 201 as one K pass per 1 x 128 tile (2 x 2 clusters, no split-K):
    q|k|v with RoPE on the pair-permuted image, o / down + residual + norm (norm as its own pass), gate|up SwiGLU."""
    gen = Gen(regime, seed=("qkv", "o", "gate_up", "down").index(shape))
    M, d, F = 201, W8B["d"], W8B["ffn"]
    with hooks(ws=1):
        if shape == "qkv":
            N, rope_cols = 6144, 40 * 128
            x, au = gen.mat(M, d)
            w, wu = gen.mat(N, d, scale=0.02)
            acc, mag = mm_ref(x, w, au, wu)
            cos, sin = rope_tables(ops, 512)
            tw = ops.TiledWeight(w, 128, rope_pairs=True)
            (y,) = run(ops, lambda: (ops.linear_tiled(x, tw, rope=(cos, sin, None, M, 5, rope_cols)),), [wg(1, 128)])
            check_rope(request, y, acc, mag, d, cos, sin, 5 + torch.arange(M, device="cuda"), rope_cols, "ws qkv")
        elif shape == "gate_up":
            x, au = gen.mat(M, d)
            w, wu = gen.mat(2 * F, d, scale=0.02)
            acc, mag = mm_ref(x, w, au, wu)
            tw = ops.TiledWeight(w, 128, swiglu=True)
            (y,) = run(ops, lambda: (ops.linear_tiled(x, tw, act=ops.ACT_SWIGLU),), [wg(1, 128)])
            check_swiglu(request, y, acc, mag, d, "ws gate|up")
        else:
            N, K = (d, d) if shape == "o" else (d, F)

            def call(x, tw, r, out, nw, xn):
                ops.linear_tiled(x, tw, residual=r, out=out, norm=(nw, 1e-5, xn))
            residual_norm_case(request, ops, gen, M, N, K, call, [wg(1, 128), NORM], f"ws {shape}",
                               prep=lambda w: ops.TiledWeight(w, 128))
