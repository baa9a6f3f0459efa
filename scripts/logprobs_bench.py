"""Cost of per-token log-probabilities and recorded scores on the GPU.

  1. uvx_token_logprobs alone at V = 128256, 1 and 8 rows, n_top in {0, 5, 20}  (CUDA events over many launches)
  2. the 8-slot decode step of SlotDecodeEngine on the Llama-3.1-8B backbone: max_logprobs = 0 against max_logprobs = 20 with
     every slot asking for 20 alternatives, graph replays alternated between the two engines
  3. the 1-stream generate() step (DecodeEngine) with and without output_scores + output_logits, alternated the same way

Prints one JSON object (with the GPU name and power limit read in the same run) and writes it to --out if given.
Usage: python scripts/logprobs_bench.py [--layers 32] [--steps 200] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

V = 128256


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


def alternate(fa, fb, rounds: int, per: int):
    """Median over `rounds` of (ms per call of fa, ms per call of fb), the two timed in turn."""
    a, b = [], []
    for _ in range(rounds):
        a.append(time_ms(fa, per))
        b.append(time_ms(fb, per))
    a.sort(), b.sort()
    return a[len(a) // 2], b[len(b) // 2]


def bench_kernel(iters: int) -> dict:
    from ultravox_b200 import ops
    out = {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for rows in (1, 8):
        lg = torch.randn(rows, V, device="cuda", generator=g) * 3
        tok = torch.randint(0, V, (rows,), device="cuda", generator=g)
        dst = torch.zeros(rows, dtype=torch.int32, device="cuda")
        bufs = (torch.empty(rows, 1, device="cuda"), torch.empty(rows, 1, 20, dtype=torch.int64, device="cuda"),
                torch.empty(rows, 1, 20, device="cuda"))
        for n in (0, 5, 20):
            n_top = torch.full((rows,), n, dtype=torch.int32, device="cuda")
            fn = lambda: ops.token_logprobs(lg, tok, n_top, dst, *bufs)     # noqa: E731
            for _ in range(20):
                fn()
            out[f"token_logprobs_rows{rows}_ntop{n}_us"] = round(1000 * time_ms(fn, iters), 2)
        scores = torch.empty(1, rows, V, device="cuda")
        step = torch.zeros(1, dtype=torch.int32, device="cuda")
        for name, kw in (("greedy", dict(temperature=0.0, top_k=0, top_p=1.0)), ("t0.7_k50", dict(temperature=0.7, top_k=50, top_p=1.0)),
                         ("t0.7_p0.9", dict(temperature=0.7, top_k=0, top_p=0.9))):
            fn = lambda: ops.record_scores(lg, kw["temperature"], kw["top_k"], kw["top_p"], step, scores=scores, raw=scores)  # noqa: E731
            for _ in range(20):
                fn()
            out[f"record_scores_rows{rows}_{name}_us"] = round(1000 * time_ms(fn, iters), 2)
    return out


def build_8b(layers: int):
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=layers))
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def bench_slots(model, steps: int, rounds: int) -> dict:
    from ultravox_b200.engine import SlotDecodeEngine
    g = torch.Generator().manual_seed(1)
    max_len = steps * (rounds + 2) + 64

    def engine(max_logprobs):
        e = SlotDecodeEngine(model, 8, max_len, max_logprobs=max_logprobs)
        for j in range(8):
            ids = torch.randint(0, 128000, (1, 16 + j), generator=g).cuda()
            e.admit(j, ids, max_len - 40, logprobs=20 if max_logprobs else None)
        return e

    off, on = engine(0), engine(20)
    for e in (off, on):
        for _ in range(5):
            e.step()
    a, b = alternate(off.step, on.step, rounds, steps // 4)
    return dict(slot_step_8_ms_max_logprobs0=round(a, 4), slot_step_8_ms_max_logprobs20=round(b, 4),
                slot_step_8_overhead_ms=round(b - a, 4), slot_launches_per_step=[off.launches_per_step, on.launches_per_step])


def bench_generate(model, steps: int, rounds: int) -> dict:
    from ultravox_b200 import ops
    from ultravox_b200.engine import DecodeEngine
    n = steps * (rounds + 2) + 8
    ids = torch.randint(0, 128000, (1, 16), generator=torch.Generator().manual_seed(2)).cuda()
    emb = ops.embed_splice(ids, model.language_model.model.embed_tokens.weight, None, None)

    def engine(record):
        e = DecodeEngine(model, 1, 16 + n + 8, output_scores=record, output_logits=record, max_new_tokens=n if record else None)
        e.prefill(emb)
        return e

    off, on = engine(False), engine(True)
    for e in (off, on):
        for _ in range(5):
            e.step()
    a, b = alternate(off.step, on.step, rounds, steps // 4)
    return dict(generate_step_1_ms=round(a, 4), generate_step_1_ms_scores_logits=round(b, 4), generate_step_1_overhead_ms=round(b - a, 4),
                generate_launches_per_step=[off.launches_per_step, on.launches_per_step])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32, help="Llama layers of the 8B backbone (32 = the full model)")
    ap.add_argument("--steps", type=int, default=200, help="timed steps per engine")
    ap.add_argument("--rounds", type=int, default=8, help="alternations between the two engines")
    ap.add_argument("--kernel-iters", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logprobs_bench.py needs a GPU")
    from ultravox_b200 import _lib
    _lib.lib()
    res = dict(gpu_info())
    res.update(bench_kernel(args.kernel_iters))
    cfg, model = build_8b(args.layers)
    res["llm_layers"] = args.layers
    res.update(bench_slots(model, args.steps, args.rounds))
    res.update(bench_generate(model, args.steps, args.rounds))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
