"""Times the four Llama-prefill GEMMs of the bench step (S = 201 tokens, Llama-3.1-8B widths) in their model forms - row-major
q|k|v with fused RoPE, o_proj and down_proj with split-K + residual + fused RMSNorm, the tiled gate|up image with fused SwiGLU -
under forced tile configurations and thread-block cluster shapes.  This is how the prefill rows of the cluster table in
gemm_tc.cu (pick_cfg) are chosen.

Each (form, configuration) is captured in a CUDA graph of `--calls` back-to-back calls that cycle through enough weight copies
(>= 400 MB) that the weights stream from HBM as they do across the 32 layers of a step, replayed and timed with CUDA events.
Per row: time per call, algorithmic GB/s (W + A + C (+ residual) bytes), and the modelled L2 -> SM ingress: every CTA pulls its
1/cn share of the A box and its 1/cm share of the W box per k-block, so one call moves 2K (n_tiles * M / cn + m_tiles * N / cm)
bytes (TMA does not fetch rows past M; the split count does not change it).  `--encoder` adds the Whisper-large-v3 encoder
GEMMs (T = 1500).  Prints one JSON line per row and the device name and power limit first."""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ultravox_b200 import ops, _lib

BF = torch.bfloat16
S, D, FFN, NQ, NKV, HD = 201, 4096, 14336, 32, 8, 128

# form -> candidates (cfg = MT*1000 + BN, splits, cm, cn); the first one of each form is the tiling before clusters
CANDIDATES = {
    "qkv": [(1128, 1, 1, 1), (1128, 1, 2, 1), (1128, 1, 2, 2), (1128, 1, 1, 2), (1128, 1, 1, 4)],
    "o": [(2128, 4, 1, 1), (2128, 4, 1, 2), (2128, 4, 1, 4), (1128, 2, 2, 1), (1128, 2, 2, 2), (2128, 2, 1, 4)],
    "gate_up": [(1128, 1, 1, 1), (2128, 1, 1, 1), (1128, 1, 2, 1), (1128, 1, 2, 2), (2128, 1, 1, 2),
                (2128, 1, 1, 4)],
    "down": [(2128, 4, 1, 1), (2128, 4, 1, 2), (2128, 4, 1, 4), (1128, 2, 2, 1), (1128, 2, 2, 2), (2128, 2, 1, 4), (1128, 4, 1, 1),
             (1128, 4, 2, 1), (1128, 4, 2, 2)],
    "enc_qkv": [(1256, 1, 1, 1), (1256, 1, 2, 1), (1128, 1, 1, 1), (1128, 1, 2, 1), (1128, 1, 2, 2), (2128, 1, 1, 1), (2128, 1, 1, 2),
                (1208, 1, 1, 1)],
    "enc_o": [(1128, 1, 1, 1), (1128, 1, 2, 1), (1064, 1, 1, 1), (1064, 1, 2, 1), (2064, 1, 1, 1), (2128, 1, 1, 1)],
    "enc_fc1": [(1256, 1, 1, 1), (1256, 1, 2, 1), (1128, 1, 1, 1), (1128, 1, 2, 1), (1128, 1, 2, 2), (2128, 1, 1, 1), (2128, 1, 1, 2)],
    "enc_fc2": [(1128, 1, 1, 1), (1128, 1, 2, 1), (1064, 1, 1, 1), (1064, 1, 2, 1), (2064, 1, 1, 1), (2128, 1, 1, 1)],
}


def device_info():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return info


def rnd(*shape, scale=1.0, gen=None):
    return (torch.randn(*shape, device="cuda", generator=gen) * scale).to(BF)


def build_form(name, gen):
    """-> (M, N, K, calls(i) -> None for weight copy i, n_copies, output bytes per row, has residual)"""
    dev = "cuda"
    if name.startswith("enc_"):
        T, E = 1500, 1280
        N, K, act = {"enc_qkv": (3 * E, E, 0), "enc_o": (E, E, 0), "enc_fc1": (4 * E, E, ops.ACT_GELU), "enc_fc2": (E, 4 * E, 0)}[name]
        x, r = rnd(T, K, gen=gen), rnd(T, N, gen=gen) if name in ("enc_o", "enc_fc2") else None
        ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(2)]
        b, out = rnd(N, gen=gen), torch.empty(T, N, dtype=BF, device=dev)
        return T, N, K, (lambda i: ops.linear(x, ws[i], b, act=act, residual=r, out=out)), 2, 2 * N, r is not None
    N, K = {"qkv": ((NQ + 2 * NKV) * HD, D), "o": (D, D), "gate_up": (2 * FFN, D), "down": (D, FFN)}[name]
    copies = max(2, -(-400_000_000 // (N * K * 2)))
    x = rnd(S, K, gen=gen)
    if name == "qkv":
        inv = ops.llama3_inv_freq(HD, 500000.0, dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                                     original_max_position_embeddings=8192))
        cos, sin = ops.rope_tables(inv, 512, dev)
        rope = (cos, sin, None, S, 0, (NQ + NKV) * HD)
        ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(copies)]
        out = torch.empty(S, N, dtype=BF, device=dev)
        return S, N, K, (lambda i: ops.linear(x, ws[i], out=out, rope=rope)), copies, 2 * N, False
    if name == "gate_up":
        ws = [ops.TiledWeight(rnd(N, K, scale=0.02, gen=gen), 128, swiglu=True) for _ in range(copies)]
        out = torch.empty(S, N // 2, dtype=BF, device=dev)
        return S, N, K, (lambda i: ops.linear_tiled(x, ws[i], out=out, act=ops.ACT_SWIGLU)), copies, N, False
    ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(copies)]
    h, nw, xn = rnd(S, N, gen=gen), rnd(N, gen=gen), torch.empty(S, N, dtype=BF, device=dev)
    return S, N, K, (lambda i: ops.linear(x, ws[i], residual=h, out=h, norm=(nw, 1e-5, xn))), copies, 2 * N, True


def cluster_dims(M, N, mt, bn, cm, cn):
    """the library's rule: a cluster axis that does not divide the tile count on that axis falls back to 1"""
    m_tiles, n_tiles = -(-M // (mt * 128)), -(-N // bn)
    return (cm if m_tiles % cm == 0 else 1), (cn if n_tiles % cn == 0 else 1)


def time_form(name, cand, M, N, K, call, copies, c_row_bytes, has_r, calls, reps):
    cfg, splits, cm, cn = cand
    lib = _lib.lib()
    lib.uvx_debug_gemm_override(cfg, splits)
    lib.uvx_debug_gemm_cluster(cm, cn)
    try:
        for i in range(copies):
            call(i)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for j in range(calls):
                call(j % copies)
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    finally:
        lib.uvx_debug_gemm_override(0, 0)
        lib.uvx_debug_gemm_cluster(0, 0)
    t = e0.elapsed_time(e1) * 1e-3 / (reps * calls)
    mt, bn = cfg // 1000, cfg % 1000
    pcm, pcn = cluster_dims(M, N, mt, bn, cm, cn)
    alg = N * K * 2 + M * K * 2 + M * c_row_bytes + (M * N * 2 if has_r else 0)
    m_tiles, n_tiles = -(-M // (mt * 128)), -(-N // bn)
    ingress = 2 * K * (n_tiles * M / pcn + m_tiles * n_tiles * bn / pcm)
    return {"form": name, "M": M, "N": N, "K": K, "forced": list(cand), "MT": mt, "BN": bn, "splits": splits, "cm": pcm, "cn": pcn,
            "us": round(t * 1e6, 2), "alg_gbs": round(alg / t / 1e9, 1), "ingress_gbs": round(ingress / t / 1e9, 1),
            "ingress_per_w_byte": round(ingress / (N * K * 2), 2), "tflops": round(2.0 * M * N * K / t / 1e12, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--forms", default="qkv,o,gate_up,down")
    ap.add_argument("--encoder", action="store_true", help="also the Whisper encoder GEMMs (T = 1500)")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-cluster", action="store_true", help="only the candidates without a cluster")
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    args = ap.parse_args()
    forms = args.forms.split(",") + (["enc_qkv", "enc_o", "enc_fc1", "enc_fc2"] if args.encoder else [])
    print(json.dumps({"device": device_info(), "calls_per_graph": args.calls, "replays": args.reps}), flush=True)
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name in forms:
        M, N, K, call, copies, c_row_bytes, has_r = build_form(name, gen)
        for cand in CANDIDATES[name]:
            if args.no_cluster and cand[2] * cand[3] > 1:
                continue
            r = time_form(name, cand, M, N, K, call, copies, c_row_bytes, has_r, args.calls, args.reps)
            rows.append(r)
            print(json.dumps(r), flush=True)
        del call
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
