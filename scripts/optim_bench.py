"""Times the adapter trainer's optimizer step on the H100: the constant-lr path (``uvx_adamw``, one launch per tensor) against
the recipe path (``uvx_grad_norm_clip`` + ``uvx_adamw_multi``, two launches for every tensor), for the projector of
Whisper-large + Llama-3.1-8B (50,343,936 elements) alone and with the encoder LoRA (3 x 2,621,440 elements).

    python scripts/optim_bench.py [--iters 200] [--out optim_bench.json]

CUDA events around ``--iters`` back-to-back steps after a warm-up; bytes per element are what the kernels must move
(adamw: g 4 + m, v 8 + 8 + p 2 + 2 = 24 B; the norm reads g again: 28 B per element for the recipe step)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PROJ, LORA = 50_343_936, 32 * 64 * 1280


def _time(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "optim_bench measures on the GPU"
    from ultravox_b200 import lr_schedule, ops
    dev = "cuda"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "iters": args.iters, "arms": {}}
    for label, sizes in (("projector", [PROJ]), ("projector+lora", [PROJ, LORA, LORA, LORA])):
        g = [torch.randn(n, device=dev) * 1e-3 for n in sizes]
        p = [torch.randn(n, device=dev).to(torch.bfloat16) for n in sizes]
        m = [torch.zeros(n, device=dev) for n in sizes]
        v = [torch.zeros(n, device=dev) for n in sizes]
        n_el = sum(sizes)
        step, lr = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, device=dev)
        table = lr_schedule.lr_table("constant", 1e-5, device=dev)
        scale, nc, ws = torch.ones(1, device=dev), torch.zeros(2, device=dev), ops.norm_workspace(dev)
        k = [0]

        def old():
            k[0] += 1
            for pi, gi, mi, vi in zip(p, g, m, v):
                ops.adamw_(pi, gi, mi, vi, k[0], 1e-5, (0.9, 0.999), 1e-8, 0.0, 1.0)

        def norm():
            ops.grad_norm_clip(g, scale, 1.0, ws, out=nc, step=step, lr_table=table, lr=lr)

        def adam():
            ops.adamw_multi_(p, g, m, v, lr, step, scale, coef=nc[1:])

        def new():
            norm()
            adam()

        t = {"adamw_per_tensor": _time(old, args.iters), "norm_clip": _time(norm, args.iters),
             "adamw_multi": _time(adam, args.iters), "norm_clip+adamw_multi": _time(new, args.iters)}
        byts = {"adamw_per_tensor": 24, "norm_clip": 4, "adamw_multi": 24, "norm_clip+adamw_multi": 28}
        res["arms"][label] = {a: {"ms": round(ms, 4), "GB/s": round(byts[a] * n_el / ms / 1e6, 1)} for a, ms in t.items()}
        res["arms"][label]["elements"] = n_el
        del g, p, m, v
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
