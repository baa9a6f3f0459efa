"""Cost of the stop strings on the GPU (Llama-3.1-8B widths, random init, a synthetic 128256-token byte-level vocabulary).

  1. uvx_stop_strings alone at 1 and 8 rows, for 1 / 3 / 5 stop strings (table sizes in int32 words) and windows (the longest
     string, 4 / 16 / 64 characters), on rows whose ends match the strings, so the chains walk the whole window: 100 launches
     captured in one CUDA graph, CUDA events around its replays, so the figure is the device time per launch.
  2. ms per graph replay of the one-stream decode step (DecodeEngine) and of the 8-slot continuous-batching step
     (SlotDecodeEngine, every slot admitted with the stop strings, against an engine built without max_stop_table), with and
     without stop strings, alternated over --rounds rounds (median, min, max).
  3. The host build of a table (HF's StopStringCriteria constructor + the packing), first and cached.

Prints one JSON object (with the GPU name and power limit read in the same run) and writes it to --out if given.
Usage: python scripts/stop_strings_bench.py [--layers 32] [--steps 100] [--rounds 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

V8B = 128256
GRAPH_LAUNCHES = 100     # kernel launches captured per timed graph
TEXT = " the user: hello there.\nuser: fine, ok! assistant: done. and then some more words follow here"


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[0].split(",")] if q else ("?", "?", "?")
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def time_ms(fn, iters: int) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def tokenizer(V: int, seed: int = 0):
    """A byte-level BPE vocabulary of exactly V ids: the byte alphabet, then distinct random 2-6 letter pieces (40% with Ġ)."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    alpha = sorted(pre_tokenizers.ByteLevel.alphabet())
    letters = list("abcdefghijklmnopqrstuvwxyz:.,!?")
    rng = np.random.default_rng(seed)
    vocab = {c: i for i, c in enumerate(alpha)}
    while len(vocab) < V:
        t = "".join(rng.choice(letters, size=int(rng.integers(2, 7))))
        vocab.setdefault(("Ġ" + t) if rng.random() < 0.4 else t, len(vocab))
    tk = Tokenizer(models.BPE(vocab=vocab, merges=[]))
    tk.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tk.decoder = decoders.ByteLevel()
    return PreTrainedTokenizerFast(tokenizer_object=tk)


def string_sets(n_strings: int, window: int) -> list:
    """n strings cut from TEXT, the first one `window` characters long."""
    out = [TEXT[5:5 + window]]
    for i in range(1, n_strings):
        out.append(TEXT[10 + 7 * i:10 + 7 * i + 1 + i])
    return out


def bench_kernel(tok, iters: int) -> list:
    from ultravox_b200 import ops
    from ultravox_b200.stop_strings import StopStrings
    text_ids = tok(TEXT, add_special_tokens=False)["input_ids"]
    res = []
    for n_strings in (1, 3, 5):
        for window in (4, 16, 64):
            st = StopStrings.build(tok, string_sets(n_strings, window))
            tab = st.device_table("cuda")
            for B in (1, 8):
                L = 4096
                seq = torch.randint(0, V8B, (B, L + 1)).cuda()
                end = torch.tensor(text_ids[:window // 2 + 8]).cuda()
                seq[:, L + 1 - end.numel():] = end            # the window matches the text: chains run long
                cand = seq[:, L].contiguous()
                hit = torch.zeros(B, dtype=torch.int32, device="cuda")
                cur = torch.tensor([L], dtype=torch.int32, device="cuda")
                ops.stop_strings(cand, seq, cur, tab, hit)
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()         # the launches back to back on the device, no host enqueue in the timing
                with torch.cuda.graph(graph):
                    for _ in range(GRAPH_LAUNCHES):
                        ops.stop_strings(cand, seq, cur, tab, hit)
                graph.replay()
                us = 1000 * time_ms(graph.replay, max(1, iters // GRAPH_LAUNCHES)) / GRAPH_LAUNCHES
                res.append(dict(strings=n_strings, window=window, table_words=st.n_words, rows=B, us=round(us, 2)))
    return res


def bench_steps(tok, layers: int, steps: int, rounds: int) -> list:
    from ultravox_b200.config import PRESETS, preset
    from ultravox_b200.engine import DecodeEngine, SlotDecodeEngine
    from ultravox_b200.model import UltravoxModel
    from ultravox_b200.stop_strings import StopStrings
    base = PRESETS["v0_5_8b"]
    cfg = preset("v0_5_8b", audio_config=dict(base["audio_config"], encoder_layers=1),
                 text_config=dict(base["text_config"], num_hidden_layers=layers))
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    stop = StopStrings.build(tok, string_sets(3, 16))
    g = torch.Generator().manual_seed(1)
    S, cap = 512, 512 + 4 * steps + 16
    ids = torch.randint(0, 2000, (1, S), generator=g).cuda()
    res = []
    engines = {}
    for name, st in (("plain", None), ("stop", stop)):
        eng = DecodeEngine(model, 1, cap, use_graph=True, eos_token_ids=[128001], stop=st)
        eng.begin(ids, torch.randn(1, V8B, device="cuda"))
        eng.step()
        engines[name] = eng
    times = {k: [] for k in engines}
    for _ in range(rounds):
        for name, eng in engines.items():
            eng.begin(ids, torch.randn(1, V8B, device="cuda"))
            eng.step()
            times[name].append(time_ms(eng.step, steps))
    row = dict(streams=1, layers=layers, prompt=S, launches={k: e.launches_per_step for k, e in engines.items()})
    for name, t in times.items():
        row[name] = dict(median_ms=round(statistics.median(t), 4), min_ms=round(min(t), 4), max_ms=round(max(t), 4))
    res.append(row)
    del engines
    torch.cuda.empty_cache()
    B, S2 = 8, 200
    ids8 = torch.randint(0, 2000, (B, S2), generator=g).cuda()
    slot_engines = {}
    for name, N in (("plain", None), ("stop", stop.n_words)):
        eng = SlotDecodeEngine(model, B, cap, eos_token_ids=[128001], max_stop_table=N)
        for j in range(B):
            eng.admit(j, ids8[j:j + 1], cap - S2 - 1, stop=stop if N is not None else None)
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
    return res


def bench_host(tok) -> dict:
    from ultravox_b200.stop_strings import StopStrings
    strings = ["\nUser:", "Assistant:", "###"]
    t0 = time.perf_counter()
    st = StopStrings.build(tok, strings)
    t1 = time.perf_counter()
    StopStrings.build(tok, strings)
    t2 = time.perf_counter()
    return dict(strings=strings, table_words=st.n_words, participating_tokens=int(st.table[0]), first_s=round(t1 - t0, 3),
                cached_ms=round(1000 * (t2 - t1), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stop_strings_bench needs a GPU")
    tok = tokenizer(V8B)
    res = dict(info=gpu_info(), host=bench_host(tok), kernel=bench_kernel(tok, a.iters),
               steps=bench_steps(tok, a.layers, a.steps, a.rounds))
    s = json.dumps(res)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
