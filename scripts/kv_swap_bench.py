"""Host swap of idle sessions: what a move costs and what a host tier buys a multi-turn workload.

  1. move rate: uvx_kv_pages_move device -> pinned host and back at the 8B widths (32 layers, Hkv 8, D 128), bf16 and e4m3,
     1 / 4 / 16 / 64 pages with shuffled page lists, CUDA events over many launches after warm-up, against the copy engine's
     rate in the same run (a contiguous pinned <-> device copy_ of the same bytes)
  2. serving: conversations x turns of text + one 5 s clip each through 8 slots on the 8B backbone (random weights); a
     conversation 'thinks' after each reply (its next turn is submitted once --lag later replies have arrived), so idle
     sessions exist.  Arms: a pool of about 8 conversations' histories plus a host tier; a pool that holds all of them (no
     swaps); the small pool without a host tier (today's behaviour: it waits, or raises).  Wall time, turn latency
     (submit -> reply, host clock) p50 / p95, pages and bytes swapped, and the time of each move (CUDA events).

Prints one JSON object (with the GPU name and power limit read in the same run) and writes it to --out if given.
Usage: python scripts/kv_swap_bench.py [--layers 32] [--conversations 32] [--turns 4] [--skip move,serve] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.kv_fp8_bench import build_8b, gpu_info  # noqa: E402

L, HKV, D = 32, 8, 128          # Llama-3.1-8B KV widths
SR = 16000


def pct(x, q):
    return float(np.percentile(np.asarray(x, dtype=np.float64), q))


def events_ms(fn, reps: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def bench_move(reps: int) -> dict:
    from ultravox_b200 import ops
    out = {}
    n_dev, n_host = 160, 96
    g = torch.Generator().manual_seed(0)
    for name, dtype in (("bf16", torch.bfloat16), ("fp8", torch.float8_e4m3fn)):
        shape = (L, n_dev, 64, HKV, D)
        kd = torch.randint(0, 256, shape[:-1] + (D * torch.empty(0, dtype=dtype).element_size(),), dtype=torch.uint8,
                           device="cuda").view(dtype)
        vd = kd.clone()
        hk = torch.empty(L, n_host, 64, HKV, D, dtype=dtype, pin_memory=True)
        hv = torch.empty(hk.shape, dtype=dtype, pin_memory=True)
        page_bytes = 64 * HKV * D * kd.element_size()
        for n in (1, 4, 16, 64):
            dev = torch.randperm(n_dev, generator=g)[:n].to(torch.int32).cuda()
            host = torch.randperm(n_host, generator=g)[:n].to(torch.int32).cuda()
            nbytes = 2 * L * n * page_bytes
            d2h = lambda: ops.kv_pages_move(kd, vd, hk, hv, dev, host)          # noqa: E731
            h2d = lambda: ops.kv_pages_move(hk, hv, kd, vd, host, dev)          # noqa: E731
            flat_d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
            flat_h = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
            ce_d2h = lambda: flat_h.copy_(flat_d, non_blocking=True)            # noqa: E731
            ce_h2d = lambda: flat_d.copy_(flat_h, non_blocking=True)            # noqa: E731
            r = max(5, min(reps, int(reps * 16 / n)))
            row = {"bytes": nbytes}
            for key, fn in (("kernel_d2h", d2h), ("kernel_h2d", h2d), ("copy_engine_d2h", ce_d2h), ("copy_engine_h2d", ce_h2d)):
                events_ms(fn, 3)
                ms = events_ms(fn, r)
                row[key + "_ms"] = round(ms, 4)
                row[key + "_GBps"] = round(nbytes / (ms * 1e-3) / 1e9, 2)
            row["kernel_over_copy_engine_d2h"] = round(row["kernel_d2h_GBps"] / row["copy_engine_d2h_GBps"], 3)
            row["kernel_over_copy_engine_h2d"] = round(row["kernel_h2d_GBps"] / row["copy_engine_h2d_GBps"], 3)
            out[f"move_{name}_{n}_pages"] = row
        del kd, vd, hk, hv
    return out


# ------------------------------------------------------------------------------------------------ serving
PRE, POST = 16, 8


def make_conversations(cfg, n, turns, budget, seed):
    from ultravox_b200 import ops
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    convs = []
    for _ in range(n):
        conv = []
        for _ in range(turns):
            wave = torch.from_numpy(rng.standard_normal(5 * SR).astype(np.float32)).cuda()
            mel = ops.logmel(wave[None], cfg.audio_config.num_mel_bins)
            tok = -(-mel.shape[-1] // 16)
            ids = torch.randint(0, 128000, (1, PRE + tok + POST), generator=g).cuda()
            conv.append(dict(ids=ids, mel=mel, frames=mel.shape[-1], tok=tok, budget=budget))
        convs.append(conv)
    return convs


def turn_features(prev, t):
    P = 0 if prev is None else prev.shape[1]
    ids = t["ids"] if prev is None else torch.cat([prev, t["ids"]], dim=1)
    return dict(input_ids=ids, audio_values=t["mel"], audio_token_start_idx=torch.tensor([P + PRE]).cuda(),
                audio_lens=torch.tensor([t["frames"]]).cuda(), audio_token_len=torch.tensor([t["tok"]], dtype=torch.int32).cuda(),
                audio_batch_size=torch.tensor([1]).cuda())


def serve(sched, convs, lag):
    """Serves every turn; returns (wall s, [turn latency ms], [(kind, pages, ms)] of every move)."""
    pending, origs = [], {}
    eng = sched.engine
    for kind in ("swap_out", "swap_in"):
        if hasattr(eng, kind):
            orig = origs[kind] = getattr(eng, kind)

            def timed(a, b, _orig=orig, _kind=kind):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _orig(a, b)
                e1.record()
                pending.append((_kind, len(a), e0, e1))
            setattr(eng, kind, timed)
    state, lat, thinking = {}, [], []
    sids = [sched.open_session() for _ in convs]

    def submit(c, t, prev):
        rid = sched.submit(turn_features(prev, convs[c][t]), max_new_tokens=convs[c][t]["budget"], session=sids[c])
        state[rid] = (c, t, time.perf_counter())

    def on_tokens(rid, seq):
        c, t, t0 = state.pop(rid)
        lat.append((time.perf_counter() - t0) * 1e3)
        if t + 1 < len(convs[c]):
            thinking.append((c, t + 1, seq))
        if len(thinking) > lag:
            submit(*thinking.pop(0))

    torch.cuda.synchronize()
    w0 = time.perf_counter()
    for c in range(len(convs)):
        submit(c, 0, None)
    sched.run(on_tokens)
    while thinking:
        submit(*thinking.pop(0))
        sched.run(on_tokens)
    torch.cuda.synchronize()
    wall = time.perf_counter() - w0
    for s in sids:
        sched.close_session(s)
    for kind, orig in origs.items():
        setattr(eng, kind, orig)
    moves = [(k, n, a.elapsed_time(b)) for k, n, a, b in pending]
    return wall, lat, moves


def bench_serve(args) -> dict:
    from ultravox_b200.serving import SlotScheduler, pages_for
    cfg, model = build_8b(args.layers)
    convs = make_conversations(cfg, args.conversations, args.turns, args.budget, 1)
    hist = max(sum(PRE + t["tok"] + POST + t["budget"] for t in c) for c in convs)
    per_conv = pages_for(hist)
    max_len = -(-(hist + 64) // 64) * 64
    small, big = 8 * per_conv, args.conversations * per_conv + 8
    page_bytes = 2 * L * 64 * HKV * D * 2
    out = dict(llm_layers=args.layers, conversations=args.conversations, turns=args.turns, budget=args.budget, lag=args.lag,
               history_positions_max=hist, pages_per_conversation=per_conv, small_pool_pages=small, big_pool_pages=big,
               host_kv_pages=args.conversations * per_conv, page_MiB=page_bytes / 2 ** 20)
    warm = [c[:2] for c in convs[:8]]
    arms = (("small_pool_host_tier", dict(kv_pages=small, host_kv_pages=args.conversations * per_conv)),
            ("big_pool", dict(kv_pages=big)), ("small_pool_no_host_tier", dict(kv_pages=small)))
    for arm, kw in arms:
        sched = SlotScheduler(model, slots=8, max_len=max_len, **kw)
        serve(sched, [[dict(t, budget=8) for t in c] for c in warm], args.lag)
        sched.swapped_out_pages = sched.swapped_in_pages = 0
        try:
            wall, lat, moves = serve(sched, convs, args.lag)
        except RuntimeError as e:
            out[arm] = dict(error=str(e))
            del sched
            torch.cuda.empty_cache()
            continue
        row = dict(wall_s=round(wall, 3), turns_served=len(lat), turn_latency_ms_p50=round(pct(lat, 50), 1),
                   turn_latency_ms_p95=round(pct(lat, 95), 1))
        if kw.get("host_kv_pages"):
            row.update(swapped_out_pages=sched.swapped_out_pages, swapped_in_pages=sched.swapped_in_pages,
                       swapped_bytes=(sched.swapped_out_pages + sched.swapped_in_pages) * page_bytes, moves=len(moves))
            for kind in ("swap_out", "swap_in"):
                ms = [m for k, _, m in moves if k == kind]
                pg = [n for k, n, _ in moves if k == kind]
                if ms:
                    row[kind] = dict(count=len(ms), pages_mean=round(statistics.fmean(pg), 2), ms_p50=round(pct(ms, 50), 3),
                                     ms_max=round(max(ms), 3), ms_total=round(sum(ms), 2),
                                     GBps=round(sum(pg) * page_bytes / (sum(ms) * 1e-3) / 1e9, 2))
        out[arm] = row
        del sched
        torch.cuda.empty_cache()
    del model
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--conversations", type=int, default=32)
    ap.add_argument("--turns", type=int, default=4)
    ap.add_argument("--budget", type=int, default=32, help="new tokens per turn")
    ap.add_argument("--lag", type=int, default=24, help="replies that arrive before a conversation's next turn is submitted")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--skip", default="", help="comma-separated parts to skip: move,serve")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_swap_bench.py measures on the GPU; none found")
    skip = set(filter(None, args.skip.split(",")))
    res = dict(bench="kv_swap", **gpu_info())
    if "move" not in skip:
        res.update(bench_move(args.reps))
    if "serve" not in skip:
        res["serve"] = bench_serve(args)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
