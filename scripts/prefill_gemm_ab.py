"""Times the four Llama-3.1-8B prefill GEMMs of the bench step (M = 201 rows) in the forms `UltravoxModel.llama_hidden` runs them -
row-major q|k|v with fused RoPE, o_proj and down_proj with split-K + residual + fused RMSNorm, the pre-tiled gate|up image
(`ops.TiledWeight`, flagged as static weights like `_tiled_weights()` images) with fused SwiGLU - one call shape at a time and as a
layer sequence (q|k|v -> o -> gate|up -> down, so the kernel boundaries and their overlap are in the measurement).

Each form is captured in a CUDA graph of `--calls` back-to-back calls cycling through weight copies (>= 400 MB, at least two) so
L2 cannot serve the weights, replayed `--reps` times and timed with CUDA events.  Arms:
  depthN      the ring capped at N k-block stages (uvx_debug_gemm_stages(N); 0 = as deep as fits)
  single      the shared A + W ring of every k-block (uvx_debug_gemm_split_ring(0)), when the library has that hook
The arms alternate inside each form.  Run it from two trees (this library and another one) to compare them call by call.  Prints
the device name and power limit first, then one JSON line per timing and a per-call table."""
import argparse, inspect, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ultravox_b200 import ops, _lib
from scripts.gemm_cluster_sweep import device_info, rnd

BF = torch.bfloat16
S, D, FFN, NQ, NKV, HD = 201, 4096, 14336, 32, 8, 128
FORMS = ("qkv", "o", "gate_up", "down")
SHAPES = {"qkv": ((NQ + 2 * NKV) * HD, D), "o": (D, D), "gate_up": (2 * FFN, D), "down": (D, FFN)}   # name -> (N, K)


def tiled_kw():
    """the static-weight flag of `_tiled_weights()` images, where this tree's `linear_tiled` takes one"""
    return {"flags": ops.GEMM_W_STATIC} if "flags" in inspect.signature(ops.linear_tiled).parameters else {}


def build(name, gen, M):
    """-> (call(i) for weight copy i, number of copies)"""
    N, K = SHAPES[name]
    copies = max(2, -(-400_000_000 // (N * K * 2)))
    x = rnd(M, K, gen=gen)
    if name == "qkv":
        inv = ops.llama3_inv_freq(HD, 500000.0, dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                                     original_max_position_embeddings=8192))
        cos, sin = ops.rope_tables(inv, 512, "cuda")
        rope = (cos, sin, None, M, 0, (NQ + NKV) * HD)
        ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(copies)]
        out = torch.empty(M, N, dtype=BF, device="cuda")
        return (lambda i: ops.linear(x, ws[i], out=out, rope=rope)), copies
    if name == "gate_up":
        ws = [ops.TiledWeight(rnd(N, K, scale=0.02, gen=gen), 128, swiglu=True) for _ in range(copies)]
        torch.cuda.synchronize()
        out, kw = torch.empty(M, N // 2, dtype=BF, device="cuda"), tiled_kw()
        return (lambda i: ops.linear_tiled(x, ws[i], out=out, act=ops.ACT_SWIGLU, **kw)), copies
    ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(copies)]
    h, nw, xn = rnd(M, N, gen=gen), rnd(N, gen=gen), torch.empty(M, N, dtype=BF, device="cuda")
    return (lambda i: ops.linear(x, ws[i], residual=h, out=h, norm=(nw, 1e-5, xn))), copies


def set_arm(arm):
    lib = _lib.lib()
    if arm.startswith("depth"):
        lib.uvx_debug_gemm_stages(int(arm[5:]))
    elif arm == "single":
        lib.uvx_debug_gemm_split_ring(0)
    elif arm.startswith("a"):                   # aN[cXY]: split ring with N activation slots [, cluster X x Y]
        n, _, cl = arm[1:].partition("c")
        lib.uvx_debug_gemm_split_ring(int(n))
        if cl:
            lib.uvx_debug_gemm_cluster(int(cl[0]), int(cl[1]))
    else:
        raise ValueError(arm)


def reset_arms():
    lib = _lib.lib()
    lib.uvx_debug_gemm_stages(0)
    lib.uvx_debug_gemm_cluster(0, 0)
    if hasattr(lib, "uvx_debug_gemm_split_ring"):
        lib.uvx_debug_gemm_split_ring(-1)


def time_graph(step, n, reps):
    """`step(j)` for j < n captured in one graph; microseconds per step over `reps` replays"""
    for j in range(n):
        step(j)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for j in range(n):
            step(j)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--forms", default=",".join(FORMS))
    ap.add_argument("--arms", default="depth0", help="comma list of depthN (N = 0: as deep as fits), single, and aN / aNcXY "
                    "(split ring with N activation slots, forced cluster X x Y)")
    ap.add_argument("--rows", type=int, default=S)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2, help="times every arm is timed, alternating")
    ap.add_argument("--no-layer", action="store_true", help="skip the layer-sequence timing")
    ap.add_argument("--out", default=None, help="also write every row to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "prefill_gemm_ab.py times the GPU kernels: it needs a GPU"
    arms = args.arms.split(",")
    if not hasattr(_lib.lib(), "uvx_debug_gemm_split_ring"):
        arms = [a for a in arms if a.startswith("depth")]
    print(json.dumps({"device": device_info(), "rows": args.rows, "calls_per_graph": args.calls, "replays": args.reps,
                      "arms": arms, "static_weight_flag": bool(tiled_kw())}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(0)
    forms = args.forms.split(",")
    calls = {name: build(name, gen, args.rows) for name in forms}
    rows = []
    for name in forms + ([] if args.no_layer else ["layer"]):
        for rnd_i in range(args.rounds):
            for arm in arms:
                set_arm(arm)
                try:
                    if name == "layer":
                        step = lambda j: [calls[f][0](j % calls[f][1]) for f in forms]
                    else:
                        call, copies = calls[name]
                        step = lambda j, call=call, copies=copies: call(j % copies)
                    us = time_graph(step, args.calls, args.reps)
                finally:
                    reset_arms()
                row = {"form": name, "M": args.rows, "arm": arm, "round": rnd_i, "us": round(us, 2)}
                if name != "layer":
                    N, K = SHAPES[name]
                    row.update({"N": N, "K": K, "w_tbs": round(N * K * 2 / us / 1e6, 3)})
                else:
                    row["w_tbs"] = round(sum(SHAPES[f][0] * SHAPES[f][1] * 2 for f in forms) / us / 1e6, 3)
                rows.append(row)
                print(json.dumps(row), flush=True)
    table = {}
    for r in rows:
        t = table.setdefault(r["form"], {})
        t[r["arm"]] = min(t.get(r["arm"], float("inf")), r["us"])
    print(json.dumps({"best_us_per_call": table}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"rows": rows, "best_us_per_call": table}, f, indent=1)


if __name__ == "__main__":
    main()
