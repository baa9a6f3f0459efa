"""Cost of beam search on the decode path.

1. One replay of the graph-captured decode step of the 8B backbone (Llama-3.1-8B widths, 32 layers, random weights) after a
   prompt of S = 201 positions (the length of a 30 s clip prompt), B = 1, in four arms: greedy DecodeEngine at 1 and at 4
   streams, BeamDecodeEngine with 4 and with 8 beams (no EOS ids, so no beam finishes).  The arms run in one process and
   alternate: `--rounds` rounds of `--steps` replays each; the median per step is reported.
2. The beam-only kernels at V = 128256 (uvx_log_softmax, uvx_beam_select, uvx_beam_update, the Llama-3 EOS triple) for 4 and
   8 beams, CUDA events over `--launches` back-to-back launches.
3. uvx_kv_reorder on the 8B cache (32 layers, 8 KV heads x 128, bf16) of 4 and 8 beams with every beam re-parented, at
   cur_len 256 / 1024 / 4096: time per launch and the bytes moved (each moved row read once, written once) in GB/s.

Prints the device name and power limit first, then one JSON line per measurement."""
import argparse, json, os, statistics, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
from ultravox_b200 import ops
from sample_bench import device_info, time_launches

V = 128256
HBM_GBPS = 3350.0       # H100 SXM data sheet


def engine_bench(args):
    from ultravox_b200.config import preset
    from ultravox_b200.engine import BeamDecodeEngine, DecodeEngine
    from ultravox_b200.model import UltravoxModel
    model = UltravoxModel(preset("v0_5_8b"), device="cuda").init_random_(seed=42)
    lm = model.language_model
    S = 201
    n = (args.rounds + 1) * args.steps + 4
    ids = torch.randint(0, 128000, (1, S), generator=torch.Generator().manual_seed(1)).cuda()
    engines = {}
    with torch.no_grad():
        for name, (streams, beams) in {"greedy x1": (1, 0), "greedy x4": (4, 0), "beams 4": (1, 4), "beams 8": (1, 8)}.items():
            emb = ops.embed_splice(ids.expand(streams, -1).contiguous(), lm.model.embed_tokens.weight, None, None)
            if beams:
                de = BeamDecodeEngine(model, 1, beams, S + n, n)
            else:
                de = DecodeEngine(model, streams, S + n)
            de.prefill(emb)
            for _ in range(args.steps):                     # the first step captures the graph
                de.step()
            engines[name] = de
        torch.cuda.synchronize()
        ms = {name: [] for name in engines}
        for _ in range(args.rounds):
            for name, de in engines.items():
                ms[name].append(time_launches(de.step, args.steps))
        base = statistics.median(ms["greedy x4"])
        for name, de in engines.items():
            med = statistics.median(ms[name])
            print(json.dumps({"bench": "decode step replay (8B, 32 layers, S = 201)", "arm": name, "ms_per_step_median": med,
                              "vs_greedy_x4_us": 1e3 * (med - base), "ms_per_step_all": [round(m, 4) for m in ms[name]],
                              "launches_per_step": de.launches_per_step}), flush=True)
    del engines, model
    torch.cuda.empty_cache()


def kernel_bench(args):
    gen = torch.Generator(device="cuda").manual_seed(0)
    eos = torch.tensor([128001, 128008, 128009], device="cuda")
    for nb in (4, 8):
        K = 4 * nb
        logits = torch.randn(nb, V, device="cuda", generator=gen) * 3
        lp = torch.empty_like(logits)
        sc = -torch.rand(nb, device="cuda", generator=gen) * 20
        out = ops.beam_select(ops.log_softmax(logits), sc, nb, K)
        smax = 4096
        i32 = dict(dtype=torch.int32, device="cuda")
        st = dict(run_score=sc.clone(), run_seq=torch.zeros(nb, smax, dtype=torch.int64, device="cuda"),
                  pool_seq=torch.zeros(nb, smax, dtype=torch.int64, device="cuda"), pool_score=torch.full((nb,), -1e9, device="cuda"),
                  pool_len=torch.zeros(nb, **i32), pool_fin=torch.zeros(nb, **i32), parent=torch.zeros(nb, **i32),
                  tok=torch.zeros(nb, dtype=torch.int64, device="cuda"), heur=torch.ones(1, **i32), flags=torch.zeros(1, **i32),
                  ticket=torch.zeros(1, **i32))
        cnt = dict(cur_len=torch.full((1,), 1024, **i32), step_idx=torch.zeros(1, **i32), done=torch.zeros(1, **i32))
        len_div = torch.ones(smax, device="cuda")

        def update():
            cnt["cur_len"].fill_(1024)      # the same step every launch (a fill kernel is in the timed loop)
            ops.beam_update(out[0], out[1], V, nb, eos, smax, len_div, 0, True, st, cnt)

        forms = {"uvx_log_softmax": lambda: ops.log_softmax(logits, out=lp),
                 "uvx_beam_select": lambda: ops.beam_select(lp, sc, nb, K, out=out),
                 "uvx_beam_update (cur_len 1024, incl. a fill)": update}
        for fn in forms.values():
            time_launches(fn, 20)
        for name, fn in forms.items():
            t = statistics.median(time_launches(fn, args.launches) for _ in range(args.rounds))
            print(json.dumps({"bench": "beam kernel", "form": name, "beams": nb, "K": K, "V": V, "us_per_launch_median": 1e3 * t}),
                  flush=True)


def reorder_bench(args):
    L, hkv, d, smax = 32, 8, 128, 4096
    for nb in (4, 8):
        k = torch.zeros(L, nb, smax, hkv, d, dtype=torch.bfloat16, device="cuda")
        v = torch.zeros_like(k)
        parent = torch.tensor([(j + 1) % nb for j in range(nb)], dtype=torch.int32, device="cuda")
        for cur in (256, 1024, 4096):
            n_pos = torch.tensor([cur], dtype=torch.int32, device="cuda")
            fn = lambda: ops.kv_reorder_(k, v, parent, n_pos, nb)
            time_launches(fn, 5)
            t = statistics.median(time_launches(fn, max(5, args.launches // 20)) for _ in range(args.rounds))
            moved = 2 * 2 * L * nb * cur * hkv * d * 2          # k and v, read + write, every row
            print(json.dumps({"bench": "uvx_kv_reorder (8B cache, every beam re-parented)", "beams": nb, "cur_len": cur,
                              "us_per_launch_median": 1e3 * t, "gb_per_s": moved / (t * 1e-3) / 1e9,
                              "of_hbm_data_sheet": moved / (t * 1e-3) / 1e9 / HBM_GBPS}), flush=True)
        del k, v
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    print(json.dumps({"device": device_info()}), flush=True)
    kernel_bench(args)
    reorder_bench(args)
    if not args.skip_engine:
        engine_bench(args)


if __name__ == "__main__":
    main()
