"""Times the Whisper-large-v3 encoder GEMMs (T = 1500 rows; q|k|v, out, fc1, fc2) at K in {320, 640, 1280, 2560, 5120} with each
epilogue (plain, +bias, +bias+GELU, +bias+residual) at 128 x 128 and 128 x 64 tiles (forced with uvx_debug_gemm_override) and on
the default path, each with the staged (shared memory + TMA store) epilogue and, in the `_reg` arms, with the register epilogue
(uvx_debug_gemm_tma_store(0)); the arms alternate call shape by call shape.  Run it from two trees (this library and another one)
to compare them call by call.

Each (shape, K, epilogue, arm) is captured in a CUDA graph of `--calls` back-to-back calls (two weight copies alternating) and
timed with CUDA events over `--reps` replays.  Per (shape, epilogue, arm) the time per call is fitted as t = waves * (F + c * kb)
over the k-block counts kb = K / 64, waves = the most tiles one CTA runs: F is the fixed cost of a tile (prologue, epilogue,
pipeline fill), c the cost of one k-block of a tile.  Prints the device name and power limit first, then one JSON line per
timing and per fit, and the per-call table at the encoder's own K (1280; fc2 5120)."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from ultravox_b200 import ops, _lib
from scripts.gemm_cluster_sweep import device_info, rnd

BF = torch.bfloat16
T, E = 1500, 1280
SHAPES = {"qkv": (3 * E, E), "out": (E, E), "fc1": (4 * E, E), "fc2": (E, 4 * E)}   # name -> (N, the encoder's K)
MODEL_EPI = {"qkv": "bias", "out": "bias_res", "fc1": "bias_gelu", "fc2": "bias_res"}
EPILOGUES = ("plain", "bias", "bias_gelu", "bias_res")
KS = (320, 640, 1280, 2560, 5120)
# arm -> (forced MT*1000 + BN (0: heuristic), uvx_debug_gemm_tma_store value (-1: default, staged where it applies; 0: registers))
ARMS = {"wg128": (1128, -1), "wg64": (1064, -1), "default": (0, -1), "wg128_reg": (1128, 0), "wg64_reg": (1064, 0), "default_reg": (0, 0)}


def waves(N, arm, sms):
    bn = 64 if arm.startswith("wg64") else 128
    tiles = -(-T // 128) * (N // bn)
    return -(-tiles // min(tiles, sms))


def time_call(call, arm, calls, reps):
    lib = _lib.lib()
    cfg, tma = ARMS[arm]
    lib.uvx_debug_gemm_override(cfg, 1 if cfg else 0)
    lib.uvx_debug_gemm_tma_store(tma)
    try:
        call(0), call(1)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for j in range(calls):
                call(j % 2)
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    finally:
        lib.uvx_debug_gemm_override(0, 0)
        lib.uvx_debug_gemm_tma_store(-1)
    return e0.elapsed_time(e1) * 1e3 / (reps * calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="qkv,out,fc1,fc2")
    ap.add_argument("--arms", default="wg128,wg128_reg,wg64,wg64_reg,default,default_reg")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write every row to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "encoder_gemm_ab.py times the GPU kernels: it needs a GPU"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps({"device": device_info(), "sms": sms, "calls_per_graph": args.calls, "replays": args.reps}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(0)
    arms = args.arms.split(",")
    rows, fits = [], []
    for name in args.shapes.split(","):
        N, _ = SHAPES[name]
        bias, res, out = rnd(N, gen=gen), rnd(T, N, gen=gen), torch.empty(T, N, dtype=BF, device="cuda")
        for K in KS:
            x = rnd(T, K, gen=gen)
            ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(2)]
            for epi in EPILOGUES:
                b = bias if epi != "plain" else None
                act = ops.ACT_GELU if epi == "bias_gelu" else ops.ACT_NONE
                r = res if epi == "bias_res" else None
                call = (lambda i, b=b, act=act, r=r: ops.linear(x, ws[i], b, act=act, residual=r, out=out))
                for arm in arms:
                    us = time_call(call, arm, args.calls, args.reps)
                    row = {"shape": name, "M": T, "N": N, "K": K, "epilogue": epi, "arm": arm, "us": round(us, 2),
                           "tflops": round(2.0 * T * N * K / us / 1e6, 1)}
                    rows.append(row)
                    print(json.dumps(row), flush=True)
            del x, ws
        for epi in EPILOGUES:
            for arm in arms:
                pts = [(r["K"] // 64, r["us"]) for r in rows if r["shape"] == name and r["epilogue"] == epi and r["arm"] == arm]
                kb, us = np.array(pts, dtype=np.float64).T
                slope, icpt = np.polyfit(kb, us, 1)
                w = waves(N, arm, sms) if not arm.startswith("default") else None
                fit = {"fit": name, "epilogue": epi, "arm": arm, "intercept_us": round(icpt, 2), "slope_us_per_kb": round(slope, 4)}
                if w:
                    F, c = icpt / w, slope / w
                    fit.update({"waves": w, "F_us_per_tile": round(F, 2), "c_us_per_kb": round(c, 4),
                                "F_share_k1280": round(F / (F + 20 * c), 3)})
                fits.append(fit)
                print(json.dumps(fit), flush=True)
    table = {}
    for name in args.shapes.split(","):
        N, K = SHAPES[name]
        for r in rows:
            if r["shape"] == name and r["K"] == K and r["epilogue"] == MODEL_EPI[name]:
                table.setdefault(f"{name} {T}x{N}x{K} {MODEL_EPI[name]}", {})[r["arm"]] = r["us"]
    print(json.dumps({"encoder_calls_us": table}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"rows": rows, "fits": fits, "encoder_calls_us": table}, f, indent=1)


if __name__ == "__main__":
    main()
