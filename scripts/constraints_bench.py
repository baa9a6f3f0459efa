"""Cost of the token constraints on the GPU (Llama-3.1-8B widths, random init).

  1. uvx_logits_constraints alone on one V = 128256 row at sequence lengths 1 k / 8 k / 32 k / 128 k, no_repeat_ngram_size 2 and 4,
     and packed tables of 0 / 100 / 1000 entries (CUDA events over many launches).  The n-gram scan reads the row's L int64
     ids (1 MB at 128 k); a table entry costs one thread its prefix compare.
  2. ms per graph replay of the one-stream and 8-stream decode steps (DecodeEngine) and of the 1-slot and 8-slot
     continuous-batching steps (SlotDecodeEngine, every slot admitted with the constraints, against an engine built without
     max_constraint_tokens) with and without constraints (no_repeat_ngram_size=3, 100 bad words, 100 sequence-bias entries,
     min_new_tokens, suppress_tokens), alternated over --rounds rounds (median, min, max).  The slot steps replay
     --steps / 2 times per round: the slots' budget is the cache left after the prompt.

Prints one JSON object (with the GPU name and power limit read in the same run) and writes it to --out if given.
Usage: python scripts/constraints_bench.py [--layers 32] [--steps 100] [--rounds 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

V8B = 128256


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


def options(n_entries: int, ngram: int, g: torch.Generator) -> dict:
    """no_repeat_ngram_size plus n_entries table entries: half bad words (2 ids), half sequence-bias entries (1-3 ids)."""
    ids = torch.randint(1, V8B, (n_entries, 3), generator=g).tolist()
    half = n_entries // 2
    kw = dict(no_repeat_ngram_size=ngram)
    if half:
        kw["bad_words_ids"] = [r[:2] for r in ids[:half]]
        kw["sequence_bias"] = {tuple(r[:1 + i % 3]): 0.5 for i, r in enumerate(ids[half:])}
    return kw


def bench_kernel(iters: int) -> list:
    from ultravox_b200 import ops
    from ultravox_b200.constraints import LogitsConstraints
    g = torch.Generator().manual_seed(0)
    out = []
    logits = torch.randn(1, V8B, device="cuda")
    for L in (1024, 8192, 32768, 131072):
        seq = torch.randint(0, 2000, (1, L + 1), generator=g).cuda()      # 2000 ids: n-grams repeat, so bans are written
        cur = torch.tensor([L], dtype=torch.int32, device="cuda")
        for n in (2, 4):
            for entries in (0, 100, 1000):
                c = LogitsConstraints.build(V8B, [128001], L, **options(entries, n, g))
                tab = c.device_tables("cuda")
                fn = lambda: ops.logits_constraints_(logits, seq, cur, tab)  # noqa: E731
                for _ in range(10):
                    fn()
                ms = time_ms(fn, iters)
                out.append(dict(L=L, n=n, entries=len(c.entries), us=round(ms * 1e3, 2),
                                seq_read_gb_s=round(L * 8 / (ms * 1e-3) / 1e9, 1)))
    return out


def bench_steps(layers: int, steps: int, rounds: int) -> list:
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.constraints import LogitsConstraints
    from ultravox_b200.engine import DecodeEngine, SlotDecodeEngine
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=layers))
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    g = torch.Generator().manual_seed(1)
    S, cap = 512, 512 + 4 * steps + 16
    res = []
    for B in (1, 8):
        ids = torch.randint(0, 2000, (B, S), generator=g).cuda()
        kw = options(200, 3, g)
        kw.update(min_new_tokens=10, suppress_tokens=list(range(100, 110)))
        c = LogitsConstraints.build(V8B, [128001], S, **kw)
        engines = {}
        for name, cons in (("plain", None), ("constrained", c)):
            eng = DecodeEngine(model, B, cap, use_graph=True, eos_token_ids=[128001], constraints=cons)
            first = torch.randn(B, V8B, device="cuda")
            eng.begin(ids, first)
            eng.step()
            engines[name] = eng
        times = {k: [] for k in engines}
        for _ in range(rounds):
            for name, eng in engines.items():
                eng.begin(ids, torch.randn(B, V8B, device="cuda"))
                eng.step()
                times[name].append(time_ms(eng.step, steps))
        row = dict(streams=B, layers=layers, prompt=S, launches={k: e.launches_per_step for k, e in engines.items()})
        for name, t in times.items():
            row[name] = dict(median_ms=round(statistics.median(t), 4), min_ms=round(min(t), 4), max_ms=round(max(t), 4))
        res.append(row)
        del engines
        torch.cuda.empty_cache()
        # the slot step (continuous batching): every slot admitted with the same constraints, or an engine built without
        # them; prompts of 200 tokens, so the admissions prefill at once (not in chunks)
        S2 = 200
        c2 = LogitsConstraints.build(V8B, [128001], S2, **kw)
        slot_engines = {}
        for name, N in (("plain", None), ("constrained", c2.n_ids)):
            eng = SlotDecodeEngine(model, B, cap, eos_token_ids=[128001], max_constraint_tokens=N)
            for j in range(B):
                eng.admit(j, ids[j:j + 1, :S2], cap - S2 - 1, constraints=c2 if N is not None else None)
            eng.step()
            slot_engines[name] = eng
        times = {k: [] for k in slot_engines}
        for _ in range(rounds):
            for name, eng in slot_engines.items():
                times[name].append(time_ms(eng.step, steps // 2))
        row = dict(slots=B, layers=layers, prompt=S2, launches={k: e.launches_per_step for k, e in slot_engines.items()})
        for name, t in times.items():
            row[name] = dict(median_ms=round(statistics.median(t), 4), min_ms=round(min(t), 4), max_ms=round(max(t), 4))
        res.append(row)
        del slot_engines
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("constraints_bench needs a GPU")
    res = dict(info=gpu_info(), kernel=bench_kernel(a.iters), steps=bench_steps(a.layers, a.steps, a.rounds))
    s = json.dumps(res)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
