"""FP8 (e4m3) paged KV pool, host side: the host quantizer the GPU tests compare against (clamp, then torch's cast) is
saturating round-to-nearest-even on the whole e4m3 grid, and SlotScheduler rejects bad pool settings before it builds an engine."""
import math
import types

import numpy as np
import pytest
import torch

E4M3 = torch.float8_e4m3fn


def host_quant(x: torch.Tensor) -> torch.Tensor:
    """What tests/test_kv_fp8_gpu.py uses with s = 1: torch's cast alone turns +-Inf and |x| > 464 into NaN."""
    return x.float().clamp(-448, 448).to(E4M3)


def e4m3_grid() -> np.ndarray:
    """Values of the positive codes 0x00..0x7E (0x7F is NaN), in code order."""
    vals = []
    for c in range(0x7F):
        e, m = c >> 3, c & 7
        vals.append(m / 8 * 2.0 ** -6 if e == 0 else (1 + m / 8) * 2.0 ** (e - 7))
    return np.array(vals)


def satfinite_rne(x: float) -> int:
    """Reference cvt.rn.satfinite.e4m3: the code of the nearest grid value (ties to the even code), +-448 beyond the grid,
    None for NaN."""
    if math.isnan(x):
        return None
    grid = e4m3_grid()
    sign = 0x80 if math.copysign(1.0, x) < 0 else 0
    a = abs(x)
    if a >= 448.0:
        return sign | 0x7E
    hi = int(np.searchsorted(grid, a))          # grid[hi - 1] < a <= grid[hi]
    if grid[hi] == a:
        return sign | hi
    lo = hi - 1
    d_lo, d_hi = a - grid[lo], grid[hi] - a
    code = lo if d_lo < d_hi else hi if d_hi < d_lo else (lo if lo % 2 == 0 else hi)
    return sign | code


def test_host_quantizer_is_saturating_rne_on_the_whole_grid():
    grid = e4m3_grid()
    mids = (grid[:-1] + grid[1:]) / 2
    xs = list(grid) + list(mids)
    f32 = np.float32
    for m in mids:                               # just off each midpoint, in fp32
        xs += [float(np.nextafter(f32(m), f32(0))), float(np.nextafter(f32(m), f32(1e9)))]
    xs += [449.0, 463.9, 464.0, 470.0, 480.0, 1e6, 3.4e38, math.inf, 2.0 ** -10, 2.0 ** -11, 2.0 ** -10 * 1.0001, 1e-30]
    xs += [-x for x in xs] + [math.nan, 0.0, -0.0]
    got = host_quant(torch.tensor(xs, dtype=torch.float32)).view(torch.uint8).tolist()
    for x, c in zip(xs, got):
        want = satfinite_rne(float(np.float32(x)))
        if want is None:
            assert c & 0x7F == 0x7F, (x, c)
        else:
            assert c == want, (x, hex(c), hex(want))
    assert torch.isnan(torch.tensor([math.inf, 500.0]).to(E4M3).float()).all()   # why the clamp is needed


def _fake_model(layers=3):
    return types.SimpleNamespace(config=types.SimpleNamespace(text_config=types.SimpleNamespace(num_hidden_layers=layers)))


@pytest.mark.parametrize("kw,msg", [
    (dict(kv_pages=8, kv_cache_dtype="fp16"), "kv_cache_dtype"),
    (dict(kv_pages=8, kv_cache_dtype="fp8"), "kv_cache_dtype"),
    (dict(kv_cache_dtype="fp8_e4m3"), "kv_pages"),
    (dict(kv_pages=8, kv_cache_dtype="fp8_e4m3", kv_scales=torch.ones(2, 2)), "shape"),
    (dict(kv_pages=8, kv_cache_dtype="fp8_e4m3", kv_scales=torch.ones(3)), "shape"),
    (dict(kv_pages=8, kv_cache_dtype="fp8_e4m3", kv_scales=torch.ones(3, 2, 1)), "shape"),
    (dict(kv_pages=8, kv_cache_dtype="fp8_e4m3", kv_scales=[[1.0, 1.0], [0.0, 1.0], [1.0, 1.0]]), "positive"),
    (dict(kv_pages=8, kv_cache_dtype="fp8_e4m3", kv_scales=[[1.0, 1.0], [1.0, -2.0], [1.0, 1.0]]), "positive"),
    (dict(kv_pages=8, kv_cache_dtype="fp8_e4m3", kv_scales=[[1.0, math.inf], [1.0, 1.0], [1.0, 1.0]]), "finite"),
    (dict(kv_pages=8, kv_cache_dtype="fp8_e4m3", kv_scales=[[1.0, 1.0], [math.nan, 1.0], [1.0, 1.0]]), "finite"),
    (dict(kv_pages=8, kv_scales=torch.ones(3, 2)), "fp8_e4m3"),
])
def test_scheduler_rejects_bad_pool_settings(kw, msg):
    from ultravox_b200.serving import SlotScheduler
    with pytest.raises(ValueError, match=msg):
        SlotScheduler(_fake_model(), slots=2, max_len=128, **kw)


def test_kv_scales_default_and_accepted_forms():
    from ultravox_b200.engine import check_kv_scales
    assert torch.equal(check_kv_scales(None, 4), torch.ones(4, 2))
    t = check_kv_scales([[0.5, 2.0]] * 4, 4)
    assert t.dtype == torch.float32 and t.shape == (4, 2) and float(t[0, 1]) == 2.0
    assert check_kv_scales(torch.full((4, 2), 0.37, dtype=torch.float64), 4).dtype == torch.float32
    mine = torch.full((4, 2), 0.5)
    t = check_kv_scales(mine, 4)
    mine.fill_(2.0)                  # the caller's tensor changing later does not change the validated scales
    assert torch.equal(t, torch.full((4, 2), 0.5))
