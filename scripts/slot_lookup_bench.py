"""Prompt lookup inside the slot step (SlotScheduler / SlotDecodeEngine with prompt_lookup_num_tokens = K) on the GPU.

  1. step time of graph replays on the 8B backbone (32 layers, random weights): slots 2 / 4 / 8 with K = 0 (the plain step),
     1 and 3, plus 4 x 7 and 8 x 7 (64 rows, past the decode-form GEMM's 32); every slot busy with a 200-token prompt
     (one B = 1 prefill each).  Each arm is timed with CUDA events over `--steps` replays per round, the arms alternated over `--rounds` rounds; medians with
     [min, max].  break_even = t_K / t_plain - 1: the accepted drafts per slot-step a lookup step needs to pay for itself.
  2. a served run: 64 requests (96-token prompts that quote themselves, 64 new tokens, greedy) through 8 slots, without lookup
     and with K = 3, on the random weights (drafts almost never accepted: the cost of misses) and on a synthetic looping
     construction of the same weights (the LM head reads the embedding table, o / down damped) where replies repeat.  Wall time,
     tokens per slot-step and accepted drafts; the two arms' tokens are compared.

Prints one JSON object (with the GPU name, power limit and max SM clock read in the same run) and writes it to --out if given.
Usage: python scripts/slot_lookup_bench.py [--layers 32] [--rounds 5] [--steps 20] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ARMS = [(2, 0), (2, 1), (2, 3), (4, 0), (4, 1), (4, 3), (4, 7), (8, 0), (8, 1), (8, 3), (8, 7)]


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[0].split(",")] if q else ("?", "?", "?")
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def build(layers: int):
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=layers))
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=0)


def med(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs))


def step_times(model, rounds: int, steps: int, prompt_len: int = 200) -> dict:
    from ultravox_b200.engine import SlotDecodeEngine
    g = torch.Generator().manual_seed(1)
    engines = {}
    for slots, K in ARMS:
        eng = SlotDecodeEngine(model, slots, prompt_len + 1200, eos_token_ids=[], prompt_lookup_num_tokens=K or None)
        for j in range(slots):
            ids = torch.randint(3, 120000, (1, prompt_len), generator=g).cuda()
            eng.admit(j, ids, 1100, lookup=(K, 2) if K else None)
        for _ in range(3):               # captures the arm's graph, warms it up
            eng.step()
        torch.cuda.synchronize()
        engines[(slots, K)] = eng
    times = {a: [] for a in ARMS}
    for _ in range(rounds):
        for a in ARMS:
            eng = engines[a]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                eng.step()
            e1.record()
            torch.cuda.synchronize()
            times[a].append(e0.elapsed_time(e1) / steps)
    out = {}
    for slots, K in ARMS:
        r = med(times[(slots, K)])
        r["rows"] = slots * (K + 1)
        if K:
            r["break_even_accepted_per_slot_step"] = r["median"] / statistics.median(times[(slots, 0)]) - 1
        out[f"{slots}x{K}"] = r
    del engines
    torch.cuda.empty_cache()
    return out


def served(model, K: int, n_req: int = 64, slots: int = 8, S: int = 96, n_new: int = 64) -> dict:
    from ultravox_b200.serving import SlotScheduler
    g = torch.Generator().manual_seed(2)
    reqs = []
    for i in range(n_req):
        ids = torch.randint(3, 120000, (1, S), generator=g)
        ids[0, S - 24:] = ids[0, 8:32]                  # the prompt quotes itself
        reqs.append(ids.cuda())
    sched = SlotScheduler(model, slots=slots, max_len=S + n_new + 8, eos_token_ids=[], prompt_lookup_num_tokens=K or None)
    serve_ids = [sched.submit(dict(input_ids=r), max_new_tokens=n_new) for r in reqs[:slots]]   # warm-up: captures the graphs
    sched.run()
    torch.cuda.synchronize()
    steps0 = sched.steps
    t0 = time.perf_counter()
    serve_ids = [sched.submit(dict(input_ids=r), max_new_tokens=n_new) for r in reqs]
    res = sched.run()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    steps = sched.steps - steps0
    toks = sum(int(res[i].shape[1]) - S for i in serve_ids)
    out = dict(wall_s=wall, steps=steps, tokens=toks, tokens_per_slot_step=toks / (steps * slots))
    if K:
        out["accepted_drafts"] = sum(sched.accepted_drafts[i] for i in serve_ids)
    return out, [res[i].cpu() for i in serve_ids]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slot_lookup_bench.py measures on the GPU; none found")
    res = dict(info=gpu_info(), layers=a.layers)
    cfg, model = build(a.layers)
    res["step_ms"] = step_times(model, a.rounds, a.steps)
    for name in ("random", "looping_synthetic"):
        if name == "looping_synthetic":
            lm = model.language_model
            lm.lm_head.weight.data.copy_(lm.model.embed_tokens.weight.data)
            for layer in lm.model.layers:
                layer.self_attn.o_proj.weight.data.mul_(0.05)
                layer.mlp.down_proj.weight.data.mul_(0.05)
            model._tiled = None
        plain, tp = served(model, 0)
        look, tl = served(model, 3)
        look["same_tokens_as_plain"] = all(torch.equal(x, y) for x, y in zip(tp, tl))
        res[f"served_{name}"] = dict(plain=plain, lookup_k3=look)
    res["info_after"] = gpu_info()
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
