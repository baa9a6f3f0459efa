"""Cost of prompt lookup decoding on the GPU (Llama-3.1-8B backbone, random init).

  1. ms per graph replay of the plain one-stream decode step (DecodeEngine, GEMV linears) and of the prompt-lookup step
     (LookupDecodeEngine, k + 1 rows on the decode-form GEMM) at k in {1, 3, 7, 10, 15}, alternated over --rounds rounds
     (median, min and max per engine), and the break-even accepted drafts per step t_k / t_1 - 1
  2. uvx_lookup_draft alone at sequence lengths 1 k, 8 k and 32 k (CUDA events over many launches)
  3. generate() with and without prompt_lookup_num_tokens on the random-init model: tokens per step and ms per token.  These
     come from a random-init model's own output and say nothing about real conversations, where the gain depends on how
     often a reply repeats earlier text.

Prints one JSON object (with the GPU name and power limit read in the same run) and writes it to --out if given.
Usage: python scripts/lookup_bench.py [--layers 32] [--steps 200] [--rounds 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KS = (1, 3, 7, 10, 15)


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[0].split(",")] if q else ("?", "?", "?")
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def time_ms(fn, iters: int) -> float:
    """Mean ms per call over `iters` calls between two events (device time; the calls are enqueued back to back)."""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def build_8b(layers: int):
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=layers))
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def bench_steps(model, steps: int, rounds: int) -> dict:
    from ultravox_b200 import ops
    from ultravox_b200.engine import DecodeEngine, LookupDecodeEngine
    S = 16
    n = steps * (rounds + 2) + 16          # the budget never runs out inside the timed window (each step makes >= 1 token)
    ids = torch.randint(0, 128000, (1, S), generator=torch.Generator().manual_seed(2)).cuda()
    emb = ops.embed_splice(ids, model.language_model.model.embed_tokens.weight, None, None)
    plain = DecodeEngine(model, 1, S + n)
    plain.prefill(emb)
    engines = {"plain": plain}
    for k in KS:
        cache = model.new_cache(1, S + n + k)
        out = model.forward(ids, past_key_values=cache, logits_to_keep=1)
        e = LookupDecodeEngine(model, S, n, k, cache=cache)
        e.begin(ids, out.logits.view(1, -1))
        engines[f"k{k}"] = e
    for e in engines.values():
        for _ in range(5):
            e.step()
    per = max(steps // 4, 10)
    times = {name: [] for name in engines}
    for _ in range(rounds):
        for name, e in engines.items():
            times[name].append(time_ms(e.step, per))
    res = {}
    t1 = sorted(times["plain"])[len(times["plain"]) // 2]
    for name, ts in times.items():
        ts.sort()
        med = ts[len(ts) // 2]
        res[f"step_ms_{name}"] = round(med, 4)
        res[f"step_ms_{name}_spread"] = [round(ts[0], 4), round(ts[-1], 4)]
        if name != "plain":
            res[f"break_even_drafts_{name}"] = round(med / t1 - 1.0, 3)
    res["launches_per_step"] = {name: e.launches_per_step for name, e in engines.items()}
    return res


def bench_draft(iters: int) -> dict:
    from ultravox_b200 import ops
    out = {}
    dev = "cuda"
    i32 = dict(dtype=torch.int32, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    k = 10
    for L in (1024, 8192, 32768):
        seq = torch.randint(0, 128000, (L + 64,), device=dev, generator=g)
        seq[L - 3:L] = seq[L // 2:L // 2 + 3]           # the last 3-gram occurs once, half way
        cur, nn, done = torch.tensor([L], **i32), torch.tensor([0], **i32), torch.zeros(1, **i32)
        tok = torch.zeros(k + 1, dtype=torch.int64, device=dev)
        nd = torch.zeros(1, **i32)
        rows = [torch.zeros(k + 1, **i32) for _ in range(5)]
        fn = lambda: ops.lookup_draft(seq, cur, nn, 64, k, 3, None, done, tok, nd, *rows)     # noqa: E731
        for _ in range(20):
            fn()
        out[f"lookup_draft_us_L{L}"] = round(1000 * time_ms(fn, iters), 2)
    return out


def bench_generate(model, max_new: int) -> dict:
    from ultravox_b200 import engine
    ids = torch.randint(0, 128000, (1, 64), generator=torch.Generator().manual_seed(3)).cuda()
    res = {}
    for k in (None, 3, 7):
        kw = {} if k is None else dict(prompt_lookup_num_tokens=k)
        model.generate(ids, max_new_tokens=16, **kw)                     # warm-up (allocator, module load)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = model.generate(ids, max_new_tokens=max_new, **kw)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        new = out.shape[1] - ids.shape[1]
        name = "plain" if k is None else f"k{k}"
        res[f"generate_ms_per_token_{name}"] = round(1000 * dt / new, 4)
        if k is not None:
            res[f"generate_tokens_per_step_{name}"] = round(new / (model.lookup_stats["steps"] + 1), 3)
    res["generate_new_tokens"] = max_new
    res["generate_gemv_max_b"] = engine.GEMV_MAX_B
    res["generate_note"] = "a random-init model's own output: says nothing about real conversations"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32, help="Llama layers of the 8B backbone (32 = the full model)")
    ap.add_argument("--steps", type=int, default=200, help="timed steps per engine")
    ap.add_argument("--rounds", type=int, default=5, help="alternations between the engines")
    ap.add_argument("--kernel-iters", type=int, default=500)
    ap.add_argument("--gen-tokens", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lookup_bench.py needs a GPU")
    from ultravox_b200 import _lib
    _lib.lib()
    res = dict(gpu_info())
    res.update(bench_draft(args.kernel_iters))
    cfg, model = build_8b(args.layers)
    res["llm_layers"] = args.layers
    res.update(bench_steps(model, args.steps, args.rounds))
    res.update(bench_generate(model, args.gen_tokens))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
