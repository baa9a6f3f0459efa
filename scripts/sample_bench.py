"""Cost of nucleus (top-p) sampling on the decode path.

1. The sampler kernel alone at V = 128256 for B in {1, 8}, on peaked, Llama-like logits (a broad background plus a few
   dozen strong candidates), in three forms: uvx_sample (top_k 50), uvx_sample_top_p (top_k 50, top_p 0.9) and
   uvx_sample_top_p (top_k 0, top_p 0.9).  CUDA events over `--launches` back-to-back launches after a warm-up, the three
   forms alternated for `--rounds` rounds; the median per launch is reported.
2. One replay of the graph-captured DecodeEngine step of the 8B backbone (Llama-3.1-8B widths, 32 layers, random weights) at 1
   and 8 streams, in three arms: greedy, T 0.6 / top_k 50, and T 0.6 / top_k 50 / top_p 0.9.  The arms run in one process and
   alternate: `--rounds` rounds of `--steps` replays each; the median per step is reported.

Prints the device name and power limit first, then one JSON line per measurement."""
import argparse, json, os, statistics, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ultravox_b200 import ops

V = 128256


def device_info():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return info


def llama_like_logits(B, gen):
    x = torch.randn(B, V, device="cuda", generator=gen) * 2.5
    for b in range(B):
        idx = torch.randperm(V, device="cuda", generator=gen)[:30]
        x[b, idx] = 14.0 + 2.0 * torch.randn(30, device="cuda", generator=gen)
    return x


def time_launches(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_bench(args):
    gen = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8):
        lg = llama_like_logits(B, gen)
        u = torch.rand(B, device="cuda", generator=gen)
        out = torch.empty(B, dtype=torch.int64, device="cuda")
        forms = {"uvx_sample k50": lambda: ops.sample(lg, 0.6, 50, u, out=out),
                 "uvx_sample_top_p k50 p0.9": lambda: ops.sample(lg, 0.6, 50, u, out=out, top_p=0.9),
                 "uvx_sample_top_p k0 p0.9": lambda: ops.sample(lg, 0.6, 0, u, out=out, top_p=0.9)}
        for fn in forms.values():
            time_launches(fn, 50)
        ms = {name: [] for name in forms}
        for _ in range(args.rounds):
            for name, fn in forms.items():
                ms[name].append(time_launches(fn, args.launches))
        for name in forms:
            print(json.dumps({"bench": "sampler kernel", "form": name, "B": B, "V": V, "launches": args.launches,
                              "us_per_launch_median": 1e3 * statistics.median(ms[name]),
                              "us_per_launch_all": [round(1e3 * m, 2) for m in ms[name]]}), flush=True)


def engine_bench(args):
    from ultravox_b200.config import preset
    from ultravox_b200.engine import DecodeEngine
    from ultravox_b200.model import UltravoxModel
    model = UltravoxModel(preset("v0_5_8b"), device="cuda").init_random_(seed=42)
    lm = model.language_model
    S = 64
    ids = torch.randint(0, 128000, (1, S), generator=torch.Generator().manual_seed(1)).cuda()
    arms = {"greedy": dict(), "T0.6 k50": dict(temperature=0.6, top_k=50),
            "T0.6 k50 p0.9": dict(temperature=0.6, top_k=50, top_p=0.9)}
    with torch.no_grad():
        for B in (1, 8):
            emb = ops.embed_splice(ids.expand(B, -1).contiguous(), lm.model.embed_tokens.weight, None, None)
            engines = {}
            for name, kw in arms.items():
                de = DecodeEngine(model, B, S + (args.rounds + 1) * args.steps + 4,
                                  generator=torch.Generator(device="cuda").manual_seed(2), **kw)
                de.prefill(emb.clone())
                for _ in range(args.steps):                     # the first step captures the graph
                    de.step()
                engines[name] = de
            torch.cuda.synchronize()
            ms = {name: [] for name in arms}
            for _ in range(args.rounds):
                for name, de in engines.items():
                    ms[name].append(time_launches(de.step, args.steps))
            base = statistics.median(ms["greedy"])
            for name in arms:
                med = statistics.median(ms[name])
                print(json.dumps({"bench": "DecodeEngine step (8B, 32 layers)", "arm": name, "streams": B,
                                  "ms_per_step_median": med, "vs_greedy_us": 1e3 * (med - base),
                                  "ms_per_step_all": [round(m, 4) for m in ms[name]],
                                  "launches_per_step": engines[name].launches_per_step}), flush=True)
            del engines
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    print(json.dumps({"device": device_info()}), flush=True)
    kernel_bench(args)
    if not args.skip_engine:
        engine_bench(args)


if __name__ == "__main__":
    main()
