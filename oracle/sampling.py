"""Oracle (test infrastructure): float64 restatement of the token sampler (``uvx_sample``, ``uvx_sample_top_p``,
``uvx_sample_slots``, ``uvx_sample_rows``) and of the set ``uvx_record_scores`` leaves finite.

Functional torch on whatever device the logits live on; every value that decides a pick is float64 and uses only
elementwise ops, sort, cumsum and searchsorted.

* ``kept``        HF's order (hf:generation/logits_process.py TemperatureLogitsWarper -> TopKLogitsWarper ->
                  TopPLogitsWarper) with the library's tie rule (include/uvx.h): a tie group - equal logits, ``-0.0`` and
                  ``+0.0`` being one value - is kept or dropped whole, and the maximum always stays.
* ``check_draws`` the inverse-CDF pick for each uniform (masses ``exp((x - max) / T)`` over the kept set, cumulative sum in
                  vocabulary order, target ``fl32(min(u, 1 - 2^-24) * Z)``, the first kept index whose CDF exceeds it) and
                  the window every fp32 pick of the kernel must fall in (``error_bound``).
"""
from __future__ import annotations

import math

import torch

U_MAX = 1.0 - 2.0 ** -24        # fminf(u, 0.99999994f): the largest uniform the sampler uses
EXPF_ULP_SLOPE = 1.173          # __expf(x): at most 2 + floor(|1.173 x|) ulp (CUDA C++ Programming Guide, intrinsic functions)
EPS32 = 2.0 ** -24              # unit roundoff of fp32


def gamma(n: int) -> float:
    """Higham's gamma_n = n u / (1 - n u) for fp32: the relative error of a sum of n nonnegative terms however it is ordered."""
    return n * EPS32 / (1.0 - n * EPS32)


def f32(v: float) -> float:
    return float(torch.tensor(v, dtype=torch.float32))


def kernel_arg(x: torch.Tensor, temperature: float) -> torch.Tensor:
    """The fp32 argument the kernel hands __expf: (x - max) * (1 / T), each step rounded to fp32 (1 / T as the host's
    ``1.0f / temperature`` and the slot kernel's ``__frcp_rn``).  Rows are the last dimension; float64 out."""
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(temperature, dtype=torch.float32)
    x = x.float()
    mx = x.max(-1, keepdim=True).values
    return ((x - mx) * inv.to(x.device)).double()


def masses(x: torch.Tensor, temperature: float, keep: torch.Tensor):
    """(p, err): the exact masses exp((x - max) / T) of the kept entries (0 elsewhere) and a bound on |m - p| for the
    kernel's fp32 mass m = __expf(kernel_arg): the Guide's ulp bound (one ulp <= 2^-23 of the value), the argument's own
    fp32 roundings (evaluated exactly), and 2^-126 for a result flushed to zero."""
    xd = x.double()
    a = (xd - xd.max(-1, keepdim=True).values) / f32(temperature)
    p = torch.where(keep, torch.exp(a), torch.zeros_like(a))
    a32 = kernel_arg(x, temperature)
    e32 = torch.exp(a32)
    ulps = 2.0 + torch.floor((EXPF_ULP_SLOPE * a32).abs())
    err = ulps * 2.0 ** -23 * e32 + (e32 - torch.exp(a)).abs() + 2.0 ** -50 * e32 + 2.0 ** -126
    err = torch.where(keep, err, torch.zeros_like(err))
    return p, err


def kept(x: torch.Tensor, temperature: float, top_k: int = 0, top_p: float = 1.0, margin: float = 0.0) -> torch.Tensor:
    """x [R, V] fp32 -> bool [R, V]: the finite entries a draw may pick.  top_k <= 0 or >= V keeps every entry; otherwise
    the entries >= the k-th largest value.  top_p < 1 then keeps token i iff the mass of the kept entries with x_j <= x_i,
    over their total, exceeds 1 - top_p (top_p as the fp32 the kernel reads); ``margin`` moves that cut by +margin (fewer
    tokens) or, negative, by -|margin| (more), which brackets a cut the kernel's fixed-point sums may place either way."""
    xd = x.double()
    R, V = xd.shape
    mx = xd.max(-1, keepdim=True).values
    keep = torch.ones_like(xd, dtype=torch.bool)
    if 0 < top_k < V:
        kth = xd.sort(-1, descending=True).values[:, top_k - 1:top_k]
        keep = xd >= kth                                   # the whole tie group at the k-th value; -0.0 == +0.0
    p32 = f32(top_p)
    if p32 < 1.0:
        m = torch.where(keep, torch.exp((xd - mx) / f32(temperature)), torch.zeros_like(xd))
        z = m.sum(-1, keepdim=True)
        xs = torch.where(keep, xd, torch.full_like(xd, -math.inf))
        vals, order = xs.sort(-1)
        cum = m.gather(-1, order).cumsum(-1)
        last_le = torch.searchsorted(vals.contiguous(), xs.contiguous(), right=True) - 1   # the last sorted entry <= x_i
        frac = cum.gather(-1, last_le.clamp_min(0)) / z
        keep = keep & (frac > (1.0 - p32) + margin)
    keep = keep | (xd == mx)
    return keep & torch.isfinite(xd)


def top_p_margin(x: torch.Tensor, temperature: float, top_k: int = 0) -> float:
    """A bound on how far the kernel's top-p cut can sit from the float64 one, as a fraction of the mass: the masses are
    __expf rounded to 2^-40 fixed point (error per entry <= its __expf bound + 2^-41), compared against the floor of
    (1 - top_p) * total; both sides of that comparison move by at most that total error."""
    keep = kept(x, temperature, top_k, 1.0)
    p, err = masses(x, temperature, keep)
    e = float(err.sum()) + int(keep.sum()) * 2.0 ** -41 + 2.0 ** -40
    z = float(p.sum())
    return 2.0 * e / (z - e) + 2.0 ** -50


def error_bound(x: torch.Tensor, temperature: float, keep: torch.Tensor) -> float:
    """delta for one row: the kernel's fp32 cumulative sums (chunk sums of c = ceil(V / 1024) terms, two 32-wide scans,
    the exclusive prefix, then up to c more terms added onto it in the walk: depth <= 2c + 13) each lie within
    sum(err) + gamma_(2c+13) Z of the float64 CDF, and its target, formed from its own total, within
    sum(err) + gamma_(c+11) Z + 2 * 2^-24 Z of the oracle's target.  The float64 cumsum adds V 2^-53 Z."""
    V = x.shape[-1]
    c = (V + 1023) // 1024
    p, err = masses(x, temperature, keep)
    z, e = float(p.sum()), float(err.sum())
    return 2.0 * e + (gamma(2 * c + 13) + gamma(c + 11) + 2.0 * EPS32 + V * 2.0 ** -53) * z


def targets(u: torch.Tensor, z: float) -> torch.Tensor:
    """fl32(min(u, 1 - 2^-24) * Z) as float64 (exact when Z is an integer below 2^24: the product then has <= 49 bits)."""
    uu = torch.clamp(u.double(), max=U_MAX)
    return (uu * z).float().double()


def check_draws(x: torch.Tensor, temperature: float, keep: torch.Tensor, u: torch.Tensor, pick: torch.Tensor,
                delta: float | None = None) -> dict:
    """One row x [V] fp32, its kept mask [V], uniforms u [n] fp32 and the kernel's picks [n] int64, on one device.
    Returns the oracle's picks and, per draw: ``inside`` - the pick has positive float64 mass and its CDF interval
    [C_{j-1}, C_j] widened by delta contains the target; ``width`` - how many tokens' widened intervals contain it.
    delta = None uses ``error_bound``; delta = 0 is the exact tier (``expected`` is then the only admissible pick).
    A target at or past the last CDF value expects the last kept token (the kernel's walk runs out there)."""
    x1, keep1 = x.view(1, -1), keep.view(1, -1)
    p, _ = masses(x1, temperature, keep1)
    p = p.view(-1)
    if delta is None:
        delta = error_bound(x1, temperature, keep1)
    pos_idx = (p > 0).nonzero().view(-1)
    cp = p.cumsum(0)[pos_idx].contiguous()
    prev = torch.cat([cp.new_zeros(1), cp[:-1]])
    t = targets(u, float(p.sum()))
    n = pos_idx.numel()
    expected = pos_idx[torch.searchsorted(cp, t, right=True).clamp_max(n - 1)]
    lo = torch.searchsorted(cp, t - delta)                      # first token with C_j >= t - delta
    hi = torch.searchsorted(prev.contiguous(), t + delta, right=True)   # tokens with C_{j-1} <= t + delta
    at = torch.searchsorted(pos_idx, pick.to(pos_idx.device)).clamp_max(n - 1)
    inside = (pos_idx[at] == pick) & (at >= lo) & (at < hi)
    return dict(expected=expected, inside=inside, width=hi - lo, delta=delta)
