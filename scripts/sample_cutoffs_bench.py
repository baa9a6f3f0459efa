"""Cost of the sampling cut-offs (min_p, typical_p, epsilon, eta) on the decode path.

1. The sampler kernel alone at V = 128256 for B in {1, 8}, on peaked, Llama-like logits: top_k 50 / top_p 0.9 as the
   baseline (uvx_sample_top_p), each cut-off alone after it, and all four (uvx_sample_cutoffs).  CUDA events over
   `--launches` back-to-back launches, the forms alternated for `--rounds` rounds; the median per launch is reported.
2. uvx_sample_slots against uvx_sample_slots_cutoffs with every row's cut-offs off (8 sampled rows), alternated likewise.
3. One replay of the graph-captured DecodeEngine step of the 8B backbone (Llama-3.1-8B widths, 32 layers, random weights) at
   1 and 8 streams, T 0.6 / top_k 50 with and without min_p 0.05, and an 8-slot SlotDecodeEngine step whose sampler is
   uvx_sample_slots (the form before the cut-offs) or uvx_sample_slots_cutoffs with every slot off.  Arms alternate:
   `--rounds` rounds of `--steps` replays each; the median per step is reported.

Prints the device name and power limit first, then one JSON line per measurement."""
import argparse, json, os, statistics, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ultravox_b200 import ops
from sample_bench import V, device_info, llama_like_logits, time_launches

CUTS = {"min_p 0.05": (0.05, 1.0, 0.0, 0.0), "typical 0.9": (0.0, 0.9, 0.0, 0.0), "epsilon 3e-4": (0.0, 1.0, 3e-4, 0.0),
        "eta 3e-4": (0.0, 1.0, 0.0, 3e-4), "all four": (0.05, 0.9, 3e-4, 3e-4)}


def alternate(forms, args, n):
    for fn in forms.values():
        time_launches(fn, 20)
    ms = {name: [] for name in forms}
    for _ in range(args.rounds):
        for name, fn in forms.items():
            ms[name].append(time_launches(fn, n))
    return ms


def kernel_bench(args):
    gen = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8):
        lg = llama_like_logits(B, gen)
        u = torch.rand(B, device="cuda", generator=gen)
        out = torch.empty(B, dtype=torch.int64, device="cuda")
        forms = {"k50 p0.9 (uvx_sample_top_p)": lambda: ops.sample(lg, 0.6, 50, u, out=out, top_p=0.9)}
        for name, cf in CUTS.items():
            forms[f"k50 p0.9 + {name}"] = (lambda cf=cf: ops.sample(lg, 0.6, 50, u, out=out, top_p=0.9, cutoffs=cf))
        ms = alternate(forms, args, args.launches)
        base = statistics.median(ms["k50 p0.9 (uvx_sample_top_p)"])
        for name in forms:
            med = statistics.median(ms[name])
            print(json.dumps({"bench": "sampler kernel", "form": name, "B": B, "V": V, "us_per_launch_median": 1e3 * med,
                              "vs_baseline_us": 1e3 * (med - base), "us_per_launch_all": [round(1e3 * m, 2) for m in ms[name]]}),
                  flush=True)
    B = 8
    lg = llama_like_logits(B, gen)
    f32 = dict(dtype=torch.float32, device="cuda")
    temps, top_p = torch.full((B,), 0.6, **f32), torch.full((B,), 0.9, **f32)
    top_k = torch.full((B,), 50, dtype=torch.int32, device="cuda")
    off = torch.tensor([ops.CUTOFFS_OFF] * B, **f32)
    u = torch.rand(B, 4, generator=gen, device="cuda")
    n_new = torch.zeros(B, dtype=torch.int32, device="cuda")
    active = torch.ones(B, dtype=torch.int32, device="cuda")
    out = torch.empty(B, dtype=torch.int64, device="cuda")
    forms = {"uvx_sample_slots": lambda: ops.sample_slots(lg, temps, top_k, top_p, u, n_new, active, out),
             "uvx_sample_slots_cutoffs (all off)": lambda: ops.sample_slots_cutoffs(lg, temps, top_k, top_p, off, u, n_new, active,
                                                                                   out)}
    ms = alternate(forms, args, args.launches)
    for name in forms:
        print(json.dumps({"bench": "slot sampler kernel", "form": name, "B": B, "V": V,
                          "us_per_launch_median": 1e3 * statistics.median(ms[name]),
                          "us_per_launch_all": [round(1e3 * m, 2) for m in ms[name]]}), flush=True)


def engine_bench(args):
    from ultravox_b200.config import preset
    from ultravox_b200.engine import DecodeEngine, SlotDecodeEngine
    from ultravox_b200.model import UltravoxModel
    model = UltravoxModel(preset("v0_5_8b"), device="cuda").init_random_(seed=42)
    lm = model.language_model
    S = 64
    ids = torch.randint(0, 128000, (1, S), generator=torch.Generator().manual_seed(1)).cuda()
    arms = {"T0.6 k50": dict(temperature=0.6, top_k=50), "T0.6 k50 min_p 0.05": dict(temperature=0.6, top_k=50,
                                                                                      cutoffs=(0.05, 1.0, 0.0, 0.0))}
    with torch.no_grad():
        for B in (1, 8):
            emb = ops.embed_splice(ids.expand(B, -1).contiguous(), lm.model.embed_tokens.weight, None, None)
            engines = {}
            for name, kw in arms.items():
                de = DecodeEngine(model, B, S + (args.rounds + 1) * args.steps + 4,
                                  generator=torch.Generator(device="cuda").manual_seed(2), **kw)
                de.prefill(emb.clone())
                for _ in range(args.steps):
                    de.step()
                engines[name] = de
            torch.cuda.synchronize()
            ms = {name: [] for name in arms}
            for _ in range(args.rounds):
                for name, de in engines.items():
                    ms[name].append(time_launches(de.step, args.steps))
            for name in arms:
                print(json.dumps({"bench": "DecodeEngine step (8B, 32 layers)", "arm": name, "streams": B,
                                  "ms_per_step_median": statistics.median(ms[name]),
                                  "ms_per_step_all": [round(m, 4) for m in ms[name]]}), flush=True)
            del engines
            torch.cuda.empty_cache()

        class PlainSlots(SlotDecodeEngine):        # the slot step with the sampler it had before the cut-offs
            def _pick_rows(self, logits, r, n_open):
                real = ops.sample_slots_cutoffs
                ops.sample_slots_cutoffs = lambda lg, t, k, p, c, u, n, a, out: ops.sample_slots(lg, t, k, p, u, n, a, out)
                try:
                    super()._pick_rows(logits, r, n_open)
                finally:
                    ops.sample_slots_cutoffs = real

        slots, steps = 8, args.steps
        cap = S + (args.rounds + 2) * steps + 8
        engines = {}
        for name, cls in (("uvx_sample_slots", PlainSlots), ("uvx_sample_slots_cutoffs (all off)", SlotDecodeEngine)):
            se = cls(model, slots, cap, eos_token_ids=[-1])
            g = torch.Generator(device="cuda").manual_seed(3)
            for j in range(slots):
                se.admit(j, ids, cap - S - 1, temperature=0.6, top_k=50, top_p=1.0,
                         u=torch.rand(cap + 1, device="cuda", generator=g))
            for _ in range(steps):
                se.step()
            engines[name] = se
        torch.cuda.synchronize()
        ms = {name: [] for name in engines}
        for _ in range(args.rounds):
            for name, se in engines.items():
                ms[name].append(time_launches(se.step, steps))
        for name in engines:
            print(json.dumps({"bench": "SlotDecodeEngine step (8B, 32 layers, 8 slots)", "sampler": name,
                              "ms_per_step_median": statistics.median(ms[name]),
                              "ms_per_step_all": [round(m, 4) for m in ms[name]]}), flush=True)


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
