"""FP8 (e4m3) paged KV pool against the bf16 pool on the GPU.

  1. bytes per position and per page at the Llama-3.1-8B and 70B widths (computed from shapes)
  2. paged decode attention (uvx_attention_paged vs _fp8) at the 8B widths, 8 and 32 rows, every row at 1k / 4k / 16k keys, and
     the mixed step's chunk attention (uvx_attention_indexed_paged vs _fp8), 248 queries over past 0 and 4k: each call captured
     20 times into a CUDA graph, timed with CUDA events over graph replays, the two pools' arms alternated
  3. the whole slot step of PagedSlotDecodeEngine on the 8B backbone (random weights), 8 and 32 slots, every row at 4k and 16k
     positions (arms that do not fit in device memory beside the weights are reported as such), alternated the same way
  4. drift over a fixed greedy workload on the same random weights: the share of generated tokens the two pools agree on, and
     the largest logit difference of the first decode step (the first step that reads the pool)

Prints one JSON object (with the GPU name and power limit read in the same run) and writes it to --out if given.
Usage: python scripts/kv_fp8_bench.py [--layers 32] [--rounds 5] [--out FILE]
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

HQ, HKV, D = 32, 8, 128        # Llama-3.1-8B / 70B attention widths (70B: 64 query heads, same Hkv and D)


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[0].split(",")] if q else ("?", "?", "?")
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def pool_bytes() -> dict:
    out = {}
    for name, layers in (("8b", 32), ("70b", 80)):
        for dt, es in (("bf16", 2), ("fp8", 1)):
            pos = layers * HKV * D * 2 * es
            out[f"{name}_{dt}_bytes_per_position"] = pos
            out[f"{name}_{dt}_MiB_per_page"] = pos * 64 / 2 ** 20
    return out


def graph_of(fn, n: int):
    """A CUDA graph of n back-to-back calls of fn (warmed up first)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def replay_ms(g, per_graph: int, reps: int = 5) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        g.replay()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / (reps * per_graph)


def alternate(fa, fb, rounds: int):
    """(median, min, max) of each of two timers, called in turn `rounds` times."""
    a, b = [], []
    for _ in range(rounds):
        a.append(fa())
        b.append(fb())
    st = lambda x: dict(median=round(statistics.median(x), 5), min=round(min(x), 5), max=round(max(x), 5))  # noqa: E731
    return st(a), st(b)


def pools(n_pages: int, seed: int):
    """A bf16 pool layer pair and the e4m3 pair quantized from it, random values, [n_pages, 64, Hkv, D]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    kb = torch.randn(n_pages, 64, HKV, D, device="cuda", generator=g).to(torch.bfloat16)
    vb = torch.randn(n_pages, 64, HKV, D, device="cuda", generator=g).to(torch.bfloat16)
    return (kb, vb), (kb.to(torch.float8_e4m3fn), vb.to(torch.float8_e4m3fn))


def bench_kernels(rounds: int) -> dict:
    from ultravox_b200 import ops
    out = {}
    scale = torch.ones(2, dtype=torch.float32, device="cuda")
    per = 20
    for rows in (8, 32):
        for ctx in (1024, 4096, 16384):
            W = ctx // 64
            (kb, vb), (k8, v8) = pools(rows * W, rows + ctx)
            table = torch.randperm(rows * W, device="cuda").to(torch.int32).view(rows, W)
            q = torch.randn(rows, HQ * D, device="cuda").to(torch.bfloat16)
            o = torch.empty_like(q)
            lens = torch.full((rows,), ctx, dtype=torch.int32, device="cuda")
            gb = graph_of(lambda: ops.attention_paged(q, kb, vb, o, HQ, D ** -0.5, table, lens), per)
            g8 = graph_of(lambda: ops.attention_paged(q, k8, v8, o, HQ, D ** -0.5, table, lens, kv_scale=scale), per)
            a, b = alternate(lambda: replay_ms(gb, per), lambda: replay_ms(g8, per), rounds)
            kv_bytes = rows * ctx * HKV * D * 2
            out[f"decode_attn_rows{rows}_ctx{ctx}"] = dict(
                bf16_us=a["median"] * 1000, fp8_us=b["median"] * 1000, bf16_spread_us=[a["min"] * 1000, a["max"] * 1000],
                fp8_spread_us=[b["min"] * 1000, b["max"] * 1000],
                bf16_kv_GBps=round(2 * kv_bytes / (a["median"] * 1e-3) / 1e9, 1), fp8_kv_GBps=round(kv_bytes / (b["median"] * 1e-3) / 1e9, 1))
            del kb, vb, k8, v8
    C = 248
    for past in (0, 4096):
        W = -(-(past + C) // 64)
        (kb, vb), (k8, v8) = pools(W, past)
        table = torch.arange(W, dtype=torch.int32, device="cuda").view(1, W)
        q = torch.randn(1, C, HQ * D, device="cuda").to(torch.bfloat16)
        o = torch.empty_like(q)
        i32 = dict(dtype=torch.int32, device="cuda")
        args = (torch.zeros(1, **i32), torch.full((1,), past, **i32), torch.full((1,), past + C, **i32))
        gb = graph_of(lambda: ops.attention_indexed_paged(q, kb, vb, o, HQ, D ** -0.5, table, *args), per)
        g8 = graph_of(lambda: ops.attention_indexed_paged(q, k8, v8, o, HQ, D ** -0.5, table, *args, kv_scale=scale), per)
        a, b = alternate(lambda: replay_ms(gb, per), lambda: replay_ms(g8, per), rounds)
        out[f"chunk_attn_q{C}_past{past}"] = dict(bf16_us=a["median"] * 1000, fp8_us=b["median"] * 1000,
                                                  bf16_spread_us=[a["min"] * 1000, a["max"] * 1000],
                                                  fp8_spread_us=[b["min"] * 1000, b["max"] * 1000])
    return out


def build_8b(layers: int):
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.model import UltravoxModel
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=layers))
    return cfg, UltravoxModel(cfg, device="cuda").init_random_(seed=42)


def step_engine(model, slots: int, ctx: int, dtype: str, steps: int):
    """A paged slot engine whose every slot decodes greedily at position ctx over a pool of random K / V (no prefill: the rows
    are placed directly, their pages listed in the table)."""
    from ultravox_b200.engine import PagedSlotDecodeEngine
    max_len = ctx + steps + 64
    per = -(-max_len // 64)
    e = PagedSlotDecodeEngine(model, slots, max_len, slots * per, kv_cache_dtype=dtype)
    for t in (e.pool_k, e.pool_v):
        t.view(torch.uint8).fill_(0x30) if dtype == "fp8_e4m3" else t.normal_(0, 1)
    for j in range(slots):
        e.kv._set_table_row(j, list(range(j * per, (j + 1) * per)))
        e.seq[j, :ctx] = 1000 + j
        e.cur_len[j] = ctx
        e.n_new[j] = 0
        e.max_new[j] = max_len - ctx - 2      # a row finishes (and writes nothing more) before it runs out of positions
        e.active[j] = 1
        e.busy[j] = True
        e._seed(j, ctx + 1)
    return e


def bench_steps(model, rounds: int, steps: int) -> dict:
    out = {}
    free = torch.cuda.mem_get_info()[0]
    for slots in (8, 32):
        for ctx in (4096, 16384):
            per_pos = model.config.text_config.num_hidden_layers * HKV * D * 2
            need = {d: slots * (ctx + steps + 128) * per_pos * es for d, es in (("bf16", 2), ("fp8_e4m3", 1))}
            fits = {d: need[d] + (need["fp8_e4m3"] if d == "bf16" else 0) < 0.9 * free for d in need}
            key = f"slot_step_{slots}_ctx{ctx}"
            if not fits["fp8_e4m3"]:
                out[key] = dict(note="does not fit beside the weights")
                continue
            engines = {d: step_engine(model, slots, ctx, d, steps * (rounds + 2)) for d in need
                       if fits[d] or d == "fp8_e4m3"}
            for e in engines.values():
                for _ in range(3):
                    e.step()
            timers = {d: (lambda e=e: replay_graph_ms(e, steps)) for d, e in engines.items()}
            if len(timers) == 2:
                a, b = alternate(timers["bf16"], timers["fp8_e4m3"], rounds)
                out[key] = dict(bf16_ms=a, fp8_ms=b)
            else:
                _, b = alternate(lambda: 0.0, timers["fp8_e4m3"], rounds)
                out[key] = dict(bf16_ms="pool does not fit beside the weights", fp8_ms=b)
            out[key]["launches_per_step"] = {d: e.launches_per_step for d, e in engines.items()}
            del engines
            torch.cuda.empty_cache()
    return out


def replay_graph_ms(e, steps: int) -> float:
    s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        e.step()
    t.record()
    t.synchronize()
    return s.elapsed_time(t) / steps


def bench_drift(model, n_req: int = 16, new: int = 64) -> dict:
    from ultravox_b200.serving import SlotScheduler
    g = torch.Generator().manual_seed(3)
    reqs = [dict(input_ids=torch.randint(0, 128000, (1, 100 + 7 * i), generator=g).cuda()) for i in range(n_req)]
    seqs, first = {}, {}
    for dt in ("bf16", "fp8_e4m3"):
        sched = SlotScheduler(model, slots=8, max_len=512, kv_pages=8 * 8, kv_cache_dtype=dt)
        ids = [sched.submit(r, max_new_tokens=new) for r in reqs]
        res = sched.run()
        seqs[dt] = [res[i] for i in ids]
        eng = sched.engine           # the first step after 8 admissions: identical first tokens, the pool read for the first time
        for j, r in enumerate(reqs[:8]):
            eng.admit(j, r["input_ids"], 4, pages=list(range(8 * j, 8 * j + 8)))
        eng.step()
        first[dt] = eng.logits.float().clone()
        del sched
        torch.cuda.empty_cache()
    agree = total = 0
    for a, b, r in zip(seqs["bf16"], seqs["fp8_e4m3"], reqs):
        S = r["input_ids"].shape[1]
        n = min(a.shape[1], b.shape[1]) - S
        agree += int((a[0, S:S + n] == b[0, S:S + n]).sum())
        total += max(a.shape[1], b.shape[1]) - S
    return dict(drift_requests=n_req, drift_new_tokens=new, drift_token_agreement=round(agree / total, 4),
                drift_first_step_logits_max_abs_diff=float((first["bf16"] - first["fp8_e4m3"]).abs().max()),
                drift_first_step_logits_max_abs=float(first["bf16"].abs().max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32, help="Llama layers of the 8B backbone (32 = the full model)")
    ap.add_argument("--rounds", type=int, default=5, help="alternations between the bf16 and fp8 arms")
    ap.add_argument("--steps", type=int, default=40, help="slot steps per timed window")
    ap.add_argument("--skip", default="", help="comma-separated parts to skip: kernels,steps,drift")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_fp8_bench.py needs a GPU")
    from ultravox_b200 import _lib
    _lib.lib()
    skip = set(filter(None, args.skip.split(",")))
    res = dict(gpu_info())
    res.update(pool_bytes())
    if "kernels" not in skip:
        res.update(bench_kernels(args.rounds))
        print(json.dumps(res), flush=True)       # partial results, in case a later part fails
    torch.cuda.empty_cache()
    if not skip >= {"steps", "drift"}:
        _, model = build_8b(args.layers)
        res["llm_layers"] = args.layers
        if "steps" not in skip:
            res.update(bench_steps(model, args.rounds, args.steps))
            print(json.dumps(res), flush=True)
        if "drift" not in skip:
            res.update(bench_drift(model))
    res.update(gpu_info_after=gpu_info())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
