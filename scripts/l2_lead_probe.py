"""Go / no-go for an L2 lead of the M = 201 Llama prefill GEMMs: how much faster is each call when the first `lead` k-blocks of
every CTA's first unit are already in L2?  Each call of a graph of back-to-back calls (cycling weight copies, so L2 cannot serve
the weights) is preceded by a small reduction that reads either that lead region of the call's own weight copy ("warm") or a
region of the same size in an unrelated buffer ("cold"); torch.profiler gives the GEMM kernel's own duration.  Also times the
layer sequence with o / down flagged as static weights (their first ring round issued before griddepcontrol.wait)."""
import json, os, sys, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
from ultravox_b200 import ops
from scripts.gemm_cluster_sweep import device_info, rnd
from scripts import prefill_gemm_ab as ab

BF = torch.bfloat16
M = ab.S


def lead_view(name, w, lead):
    """the boxes the first `lead` k-blocks of every CTA's first unit read, as a strided view of the weight (or image)"""
    N, K = ab.SHAPES[name]
    if name == "qkv":                       # 96 CTAs = all 96 tiles, split 1
        return w.view(N, K // 64, 64)[:, :lead]
    if name in ("o", "down"):               # 32 column tiles x 4 splits = 128 first units
        return w.view(N, 4, K // 256, 64)[:, :, :lead]
    img = w.image.view(-1, K // 64, 128, 64)     # gate|up image: 224 tiles, CTA b's first unit is tile b (132 CTAs)
    return img[:132, :lead]


def build(name, gen):
    N, K = ab.SHAPES[name]
    copies = max(2, -(-400_000_000 // (N * K * 2)))
    x = rnd(M, K, gen=gen)
    if name == "gate_up":
        ws = [ops.TiledWeight(rnd(N, K, scale=0.02, gen=gen), 128, swiglu=True) for _ in range(copies)]
        torch.cuda.synchronize()
        out = torch.empty(M, N // 2, dtype=BF, device="cuda")
        call = lambda i, fl: ops.linear_tiled(x, ws[i], out=out, act=ops.ACT_SWIGLU, flags=ops.GEMM_W_STATIC)
    elif name == "qkv":
        inv = ops.llama3_inv_freq(ab.HD, 500000.0, dict(rope_type="llama3", factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                                                        original_max_position_embeddings=8192))
        cos, sin = ops.rope_tables(inv, 512, "cuda")
        rope = (cos, sin, None, M, 0, (ab.NQ + ab.NKV) * ab.HD)
        ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(copies)]
        out = torch.empty(M, N, dtype=BF, device="cuda")
        call = lambda i, fl: ops.linear(x, ws[i], out=out, rope=rope, flags=fl)
    else:
        ws = [rnd(N, K, scale=0.02, gen=gen) for _ in range(copies)]
        h, nw, xn = rnd(M, N, gen=gen), rnd(N, gen=gen), torch.empty(M, N, dtype=BF, device="cuda")
        call = lambda i, fl: ops.linear(x, ws[i], residual=h, out=h, norm=(nw, 1e-5, xn), flags=fl)
    return call, ws, copies


def kernel_us(step, n, reps):
    """graph of step(j), j < n; per-kernel-name mean duration (us) over `reps` profiled replays"""
    for j in range(n):
        step(j)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for j in range(n):
            step(j)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            g.replay()
        torch.cuda.synchronize()
    agg = collections.defaultdict(list)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            agg[e.name.split("(")[0].split("<")[0][-40:]].append(e.time_range.end - e.time_range.start)
    return {k: round(sum(v) / len(v), 2) for k, v in agg.items()}


def main():
    assert torch.cuda.is_available()
    print(json.dumps({"device": device_info()}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(0)
    scratch = torch.zeros(64 << 20, dtype=BF, device="cuda")
    calls = {f: build(f, gen) for f in ab.FORMS}
    for name in ab.FORMS:
        call, ws, copies = calls[name]
        for lead in (4, 8, 16):
            for arm in ("cold", "warm", "cold", "warm"):
                def step(j):
                    i = j % copies
                    v = lead_view(name, ws[i], lead)
                    if arm == "cold":
                        v = scratch[:v.numel()].view(v.shape)
                    v.amax()
                    call(i, 0)
                r = kernel_us(step, 20, 5)
                gemm = {k: v for k, v in r.items() if "gemm" in k or "splitk" in k}
                lead_mb = lead_view(name, ws[0], lead).numel() * 2 / 1e6
                print(json.dumps({"form": name, "lead": lead, "lead_mb": round(lead_mb, 1), "arm": arm, "kernels_us": gemm}), flush=True)
    # layer sequence with o / down flagged static, CUDA events
    for rnd_i in range(3):
        for fl in (0, ops.GEMM_W_STATIC):
            step = lambda j: [calls[f][0](j % calls[f][2], fl) for f in ab.FORMS]
            us = ab.time_graph(step, 20, 10)
            print(json.dumps({"form": "layer", "static_o_down_qkv": bool(fl), "round": rnd_i, "us": round(us, 2)}), flush=True)


if __name__ == "__main__":
    main()
