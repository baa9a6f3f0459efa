"""The optimizer step of the released recipes on the device (HF Trainer: clip_grad_norm_(max_grad_norm), AdamW, LambdaLR schedule,
gradient accumulation): uvx_grad_norm_clip / uvx_adamw_multi / uvx_grad_accumulate against torch, then AdapterTrainer end to end
on the micro model - accumulation, the parameter trajectory against torch AdamW + clip + scheduler, CUDA-graph replay, resume,
the unchanged default path and two data-parallel ranks."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
PROJ = 50_343_936                      # projector flat buffer of Whisper-large + Llama-3.1-8B
LORA = 32 * 64 * 1280                  # one EncoderLora tensor (A / Bq / Bk) of Whisper-large


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def randn(n, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, generator=g, device="cuda") * scale


def _norm_args(grads):
    from ultravox_b200 import lr_schedule, ops
    dev = grads[0].device
    return dict(workspace=ops.norm_workspace(dev), step=torch.zeros(1, dtype=torch.int64, device=dev),
                lr_table=lr_schedule.lr_table("cosine", 1e-3, 2, 5, device=dev), lr=torch.zeros(1, device=dev))


def _torch_coef(norm, max_norm):
    return torch.clamp(max_norm / (norm + 1e-6), max=1.0)         # torch.nn.utils.clip_grad_norm_'s formula, fp32


# ------------------------------------------------------------------------------------------ uvx_grad_norm_clip
def test_grad_norm_clip_matches_torch_and_is_deterministic():
    from ultravox_b200 import ops
    sizes = [PROJ, LORA, LORA, LORA, 10007, 33, 1, 4099]
    grads = [randn(n, 100 + i, 1e-3 * (i + 1)) for i, n in enumerate(sizes)]
    grads[5] = grads[5][1:]                                    # a tensor that is not 16-byte aligned: the scalar path
    s = torch.tensor([1 / 6], dtype=torch.float32, device="cuda")
    kw = _norm_args(grads)
    want = torch.nn.utils.get_total_norm([(g * s).double() for g in grads])
    for max_norm in (1.0, 0.05, None, 0.0):
        out = ops.grad_norm_clip(grads, s, max_norm, kw["workspace"]).clone()
        again = ops.grad_norm_clip(grads, s, max_norm, kw["workspace"]).clone()
        assert torch.equal(out, again)                          # fixed grid, fixed order: the same bits every launch
        assert rel(out[0], want) < 1e-6, (float(out[0]), float(want))
        if max_norm:
            assert torch.equal(out[1], _torch_coef(out[0], max_norm))
            t_norm = torch.nn.utils.get_total_norm([g * s for g in grads])   # torch's own fp32 norm, and its coef
            assert rel(out[0], t_norm) < 1e-6 and rel(out[1], _torch_coef(t_norm, max_norm)) < 1e-6
        else:
            assert float(out[1]) == 1.0
    assert float(ops.grad_norm_clip(grads, s, 0.05, kw["workspace"])[1]) < 1.0              # clipping is active at 0.05
    # scale folding: the scaled norm is the norm of the pre-scaled gradients, bit for bit
    one = torch.ones(1, device="cuda")
    pre = ops.grad_norm_clip([g * s for g in grads], one, 0.05, kw["workspace"])
    assert torch.equal(ops.grad_norm_clip(grads, s, 0.05, kw["workspace"]), pre)
    # step bookkeeping: step += 1, lr = table[step - 1], clamped to the last entry
    lrs = []
    for _ in range(7):
        ops.grad_norm_clip(grads[4:], s, 1.0, kw["workspace"], step=kw["step"], lr_table=kw["lr_table"], lr=kw["lr"])
        lrs.append(float(kw["lr"]))
    assert int(kw["step"]) == 7
    tab = kw["lr_table"].tolist()
    assert lrs == tab + [tab[-1]] and lrs[0] == 0.0


def test_grad_norm_clip_non_finite_like_torch():
    from ultravox_b200 import ops
    grads = [randn(PROJ, 1, 1e-3), randn(4099, 2)]
    one = torch.ones(1, device="cuda")
    ws = ops.norm_workspace("cuda")
    grads[0][12345] = float("nan")
    out = ops.grad_norm_clip(grads, one, 1.0, ws)
    t_norm = torch.nn.utils.get_total_norm(grads)
    assert math.isnan(float(out[0])) and math.isnan(float(out[1])) and math.isnan(float(t_norm))
    grads[0][12345] = float("inf")
    out = ops.grad_norm_clip(grads, one, 1.0, ws)
    assert math.isinf(float(out[0])) and float(out[1]) == 0.0
    assert float(_torch_coef(torch.tensor(float("inf")), 1.0)) == 0.0


# ------------------------------------------------------------------------------------------ uvx_adamw_multi
def test_adamw_multi_matches_torch_adamw_clip_and_cosine_schedule():
    """6 steps of clip_grad_norm_(1.0) + torch.optim.AdamW(wd 0.01) + get_scheduler("cosine", warmup 2) on fp32 copies of the
    parameters, fed the same gradients; clipping is active on some steps only."""
    import transformers
    from ultravox_b200 import lr_schedule, ops
    sizes = [10007, 4099, 33, 4096]
    base, wd, s = 2e-3, 0.01, 0.5
    ps = [randn(n, 10 + i).to(BF) for i, n in enumerate(sizes)]
    p0 = [p.clone() for p in ps]
    ms = [torch.zeros(n, device="cuda") for n in sizes]
    vs = [torch.zeros(n, device="cuda") for n in sizes]
    gs = [torch.empty(n, device="cuda") for n in sizes]
    pf = [p.float().clone().requires_grad_(True) for p in ps]
    opt = torch.optim.AdamW(pf, lr=base, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
    sch = transformers.get_scheduler("cosine", opt, num_warmup_steps=2, num_training_steps=6)
    kw = _norm_args(gs)
    table = lr_schedule.lr_table("cosine", base, 2, 6, device="cuda")
    scale = torch.tensor([s], device="cuda")
    out = torch.empty(2, device="cuda")
    coefs = []
    for k, amp in enumerate([0.05, 0.001, 0.03, 0.002, 0.1, 0.0005]):
        for i, g in enumerate(gs):
            g.copy_(randn(g.numel(), 1000 * k + i, amp))
        for p, g in zip(pf, gs):
            p.grad = g * s
        t_norm = torch.nn.utils.clip_grad_norm_(pf, 1.0)
        lr_used = opt.param_groups[0]["lr"]
        opt.step()
        sch.step()
        ops.grad_norm_clip(gs, scale, 1.0, kw["workspace"], out=out, step=kw["step"], lr_table=table, lr=kw["lr"])
        ops.adamw_multi_(ps, gs, ms, vs, kw["lr"], kw["step"], scale, coef=out[1:], betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
        assert rel(out[0], t_norm) < 1e-6 and float(kw["lr"]) == np.float32(lr_used)
        coefs.append(float(out[1]))
        if k == 0:                                              # warmup: the first update runs with lr = 0
            assert lr_used == 0.0 and all(torch.equal(a, b) for a, b in zip(ps, p0))
        for p, m, v, ref in zip(ps, ms, vs, pf):
            st = opt.state[ref]
            assert rel(m, st["exp_avg"]) < 1e-5 and rel(v, st["exp_avg_sq"]) < 1e-5, k
            assert rel(p, ref.detach().to(BF)) < 8e-3, k        # bf16 parameter storage, as test_adamw_step_matches_torch
    assert min(coefs) < 1.0 and max(coefs) == 1.0, coefs
    assert int(kw["step"]) == 6


def test_grad_accumulate():
    from ultravox_b200 import ops
    gs = [randn(n, n) for n in (PROJ, LORA, 4099)]
    gs.append(randn(34, 7)[1:])                                 # unaligned: scalar path
    accs = [torch.full_like(g, 7.0) for g in gs]
    ops.grad_accumulate_(accs, gs, assign=True)
    assert all(torch.equal(a, g) for a, g in zip(accs, gs))
    hs = [randn(g.numel(), 99 + i) for i, g in enumerate(gs)]
    ops.grad_accumulate_(accs, hs)
    assert all(torch.equal(a, g + h) for a, g, h in zip(accs, gs, hs))
    with pytest.raises(Exception):
        ops.grad_accumulate_(gs[:1], gs[:1])                   # acc may not alias g


# ------------------------------------------------------------------------------------------ AdapterTrainer end to end
def _setup(lens, seed=7):
    from oracle import logmel as ol
    from ultravox_b200.config import preset
    from ultravox_b200.model import UltravoxModel
    cfg = preset("micro")
    model = UltravoxModel(cfg, device="cuda").init_random_(seed=42)
    with torch.no_grad():   # norm weights away from their constant init so their gradients are exercised
        for n, p in model.multi_modal_projector.named_parameters():
            if "ln_" in n:
                p.add_(torch.randn(p.shape, generator=torch.Generator().manual_seed(3)).to(p.device, p.dtype) * 0.1)
    waves = [np.random.default_rng(1000 + i).standard_normal(n).astype(np.float32) for i, n in enumerate(lens)]
    padded, frames = ol.pad_batch(waves)
    g = torch.Generator().manual_seed(seed)
    tok = [int(-(-int(f) // 16)) for f in frames]
    S = 8 + max(tok) + 5
    ids = torch.randint(0, cfg.vocab_size, (len(waves), S), generator=g)
    labels = ids.clone()
    labels[:, :-5] = -100
    batch = dict(input_ids=ids, audio_token_start_idx=torch.tensor([8] * len(waves)),
                 audio_lens=torch.tensor([int(f) for f in frames]), audio_token_len=torch.tensor(tok, dtype=torch.int32),
                 audio_batch_size=torch.ones(len(waves), dtype=torch.int64), labels=labels)
    return cfg, model, padded, batch


def _micro_batches(n=2, lens=(16000 * 2, 16000 + 77)):
    """``n`` micro-batches of the same shapes (different tokens) on one micro model."""
    from ultravox_b200 import ops
    cfg, model, padded, batch = _setup(list(lens))
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    out = []
    for j in range(n):
        b = dict(batch, audio_values=mel)
        g = torch.Generator().manual_seed(50 + j)
        b["input_ids"] = torch.randint(0, cfg.vocab_size, batch["input_ids"].shape, generator=g)
        b["labels"] = b["input_ids"].clone()
        b["labels"][:, :-5] = -100
        out.append(b)
    return cfg, model, out


def _lora(model):
    from ultravox_b200.autograd import EncoderLora
    lora = EncoderLora(model, r=8, alpha=8.0, seed=3)
    with torch.no_grad():
        lora.Bq[:, :, :8] = (torch.randn(lora.L, lora.d, 8, generator=torch.Generator().manual_seed(9)) * 0.05).to(BF).cuda()
    return lora


@pytest.mark.parametrize("with_lora", [False, True])
def test_accumulated_gradient_is_the_mean_of_micro_batch_gradients(with_lora):
    from ultravox_b200.training import AdapterTrainer
    cfg, model, mbs = _micro_batches(2)
    lora = _lora(model) if with_lora else None
    plain = AdapterTrainer(model, lr=1e-3, encoder_lora=lora)
    refs = []
    for b in mbs:
        plain.forward_backward(**b)
        refs.append([plain.grad.clone()] + ([g.clone().view(-1) for _, g in lora.params_and_grads()] if lora else []))
    tr = AdapterTrainer(model, lr=1e-3, encoder_lora=lora, grad_accum_steps=2, max_grad_norm=1.0)
    flat0 = model.multi_modal_projector.flat.clone()
    tr.train_step(**mbs[0])
    assert tr.phase == 1 and torch.equal(model.multi_modal_projector.flat, flat0) and tr.step_count == 0
    own1 = [g.clone() for g in tr._grads]
    assert all(torch.equal(a, g) for a, g in zip(tr._accs, own1))
    tr.train_step(**mbs[1])
    assert tr.phase == 0 and tr.step_count == 1 and int(tr.opt_step) == 1
    assert float(tr.grad_scale) == 0.5 and len(tr._accs) == (4 if with_lora else 1)
    # exact against this trainer's own micro-batch gradients; against separate plain runs within fp32 rounding (the RMSNorm
    # weight gradients are summed with fp32 atomics, so two backward passes may differ in their last bits)
    assert all(torch.equal(a, g1 + g2) for a, g1, g2 in zip(tr._accs, own1, tr._grads))
    for a, g1, g2 in zip(tr._accs, refs[0], refs[1]):
        assert rel(a * 0.5, (g1.double() + g2.double()) / 2) < 1e-6
    total = torch.cat([((g1 + g2) * 0.5).double() for g1, g2 in zip(own1, tr._grads)]).norm()
    assert rel(tr.last["grad_norm"], total) < 1e-6
    assert not torch.equal(model.multi_modal_projector.flat, flat0)


def test_trainer_trajectory_matches_torch_adamw_clip_and_scheduler():
    """4 optimizer steps (cosine, warmup 1, clip 0.5, wd 0.01, projector + encoder LoRA): the trainer's parameters against
    torch AdamW + clip_grad_norm_ + get_scheduler on fp32 copies fed the same per-step gradients."""
    import transformers
    from ultravox_b200.training import AdapterTrainer
    cfg, model, mbs = _micro_batches(1)
    lora = _lora(model)
    tr = AdapterTrainer(model, lr=2e-3, weight_decay=0.01, encoder_lora=lora, max_grad_norm=0.5, lr_scheduler="cosine",
                        warmup_steps=1, num_training_steps=4)
    params = tr._params
    pf = [p.float().clone().requires_grad_(True) for p in params]
    opt = torch.optim.AdamW(pf, lr=2e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    sch = transformers.get_scheduler("cosine", opt, num_warmup_steps=1, num_training_steps=4)
    norms, losses = [], []
    for k in range(4):
        losses.append(float(tr.train_step(**mbs[0])))
        for p, g in zip(pf, tr._grads):
            p.grad = g.clone()
        norms.append((float(torch.nn.utils.clip_grad_norm_(pf, 0.5)), float(tr.last["grad_norm"])))
        assert float(tr.last["lr"]) == np.float32(opt.param_groups[0]["lr"])
        opt.step()
        sch.step()
        for p, ref in zip(params, pf):
            assert rel(p, ref.detach().to(BF)) < 8e-3, (k, rel(p, ref.detach().to(BF)))
        for m, ref in zip(tr._m, pf):
            assert rel(m, opt.state[ref]["exp_avg"]) < 1e-5
    assert all(abs(a - b) <= 1e-5 * a for a, b in norms), norms
    assert max(a for a, _ in norms) > 0.5                        # clipping was active
    with pytest.raises(RuntimeError):
        tr.train_step(**mbs[0])                                 # past num_training_steps


def test_recipe_training_reduces_loss():
    from ultravox_b200.training import AdapterTrainer
    cfg, model, mbs = _micro_batches(2, lens=(16000, 16000))
    tr = AdapterTrainer(model, lr=2e-3, max_grad_norm=1.0, lr_scheduler="cosine_with_min_lr", warmup_steps=0.2,
                        num_training_steps=6, scheduler_kwargs={"min_lr_rate": 0.1}, grad_accum_steps=2)
    losses = []
    for _ in range(6):
        for b in mbs:
            tr.train_step(**b)
        losses.append(float(tr.last["loss"]))
    assert all(math.isfinite(x) for x in losses) and losses[-1] < losses[0], losses


def test_optimizer_step_graph_replay_equals_eager():
    from ultravox_b200.training import AdapterTrainer
    cfg, model, mbs = _micro_batches(1)
    lora = _lora(model)
    tr = AdapterTrainer(model, lr=2e-3, weight_decay=0.01, encoder_lora=lora, max_grad_norm=0.5, lr_scheduler="cosine",
                        warmup_steps=2, num_training_steps=10)
    tr.forward_backward(**mbs[0])
    p0, sd0 = [p.clone() for p in tr._params], tr.state_dict()
    for _ in range(5):
        tr.optimizer_step_device()
    eager = [t.clone() for t in tr._params + tr._m + tr._v + [tr.opt_step, tr.opt_lr, tr.norm_coef]]
    for p, q in zip(tr._params, p0):
        p.copy_(q)
    tr.load_state_dict(sd0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        tr.optimizer_step_device()
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    got = tr._params + tr._m + tr._v + [tr.opt_step, tr.opt_lr, tr.norm_coef]
    assert int(tr.opt_step) == 5
    assert all(torch.equal(a, b) for a, b in zip(got, eager))


def test_resume_from_state_dict_is_bit_identical():
    """state_dict() after optimizer step 2 plus one micro-batch, a fresh trainer with load_state_dict, steps 3-4: the same bits
    as the uninterrupted run.  The micro-batch gradients are fed from a seed so that the two runs see identical gradients."""
    from ultravox_b200.training import AdapterTrainer

    class Fed(AdapterTrainer):
        def forward_backward(self, k, **_):
            self.grad.copy_(randn(self.grad.numel(), 500 + k, 1e-3))
            return torch.tensor(float(k), device="cuda")

    kw = dict(lr=2e-3, weight_decay=0.01, max_grad_norm=0.5, lr_scheduler="linear", warmup_steps=1, num_training_steps=4,
              grad_accum_steps=2)
    cfg, model, _ = _micro_batches(1)
    flat0 = model.multi_modal_projector.flat.clone()
    tr = Fed(model, **kw)
    for k in range(8):
        tr.train_step(k=k)
    want = [model.multi_modal_projector.flat.clone(), tr.m.clone(), tr.v.clone(), tr.opt_lr.clone()]
    assert float(tr.last["loss"]) == 6.5 and tr.step_count == 4
    model.multi_modal_projector.flat.copy_(flat0)
    tr2 = Fed(model, **kw)
    for k in range(5):                                          # 2 optimizer steps + one micro-batch of the third
        tr2.train_step(k=k)
    sd, flat = tr2.state_dict(), model.multi_modal_projector.flat.clone()
    model.multi_modal_projector.flat.copy_(flat)                # a fresh trainer on the restored parameters
    tr3 = Fed(model, **kw)
    tr3.load_state_dict(sd)
    assert tr3.phase == 1 and tr3.step_count == 2
    for k in range(5, 8):
        tr3.train_step(k=k)
    assert tr3.step_count == 4 and int(tr3.opt_step) == 4
    got = [model.multi_modal_projector.flat, tr3.m, tr3.v, tr3.opt_lr]
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    with pytest.raises(ValueError):
        Fed(model, **dict(kw, grad_accum_steps=4)).load_state_dict(sd)
    with pytest.raises(RuntimeError):
        tr3.train_step(k=8)                                     # past num_training_steps


def test_default_trainer_is_the_plain_adamw_path():
    """AdapterTrainer(model, lr) driven as bench.py drives it (forward_backward, all_reduce, optimizer_step) == ops.adamw_ called
    directly on a shadow copy with the same gradients: the new arguments change nothing at their defaults."""
    from ultravox_b200 import ops
    from ultravox_b200.training import AdapterTrainer
    cfg, model, mbs = _micro_batches(1)
    flat = model.multi_modal_projector.flat
    tr = AdapterTrainer(model, lr=2e-3)
    assert not tr.recipe
    shadow, m, v = flat.clone(), torch.zeros_like(tr.m), torch.zeros_like(tr.v)
    for step in (1, 2, 3):
        tr.forward_backward(**mbs[0])
        scale = tr.all_reduce()
        ops.adamw_(shadow, tr.grad, m, v, step, 2e-3, (0.9, 0.999), 1e-8, 0.0, scale)
        tr.optimizer_step(scale)
        assert torch.equal(flat, shadow) and torch.equal(m, tr.m) and torch.equal(v, tr.v)
    with pytest.raises(RuntimeError):
        tr.optimizer_step_device()


# ------------------------------------------------------------------------------------------ two data-parallel ranks
def _rank(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ultravox_b200 import ops
    from ultravox_b200.training import AdapterTrainer
    cfg, model, padded, batch = _setup([16000 * 2] * 4)
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    tr = AdapterTrainer(model, lr=1e-3, max_grad_norm=1e-3, grad_accum_steps=2)
    for j in range(2):                                          # rank r: clips 2r, 2r + 1 as two micro-batches
        i = 2 * rank + j
        tr.train_step(audio_values=mel[i:i + 1], **{k: v[i:i + 1] for k, v in batch.items()})
    torch.cuda.synchronize()
    q.put((rank, model.multi_modal_projector.flat.cpu(), float(tr.last["grad_norm"]), float(tr.norm_coef[1]), float(tr.grad_scale)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_accumulated_clipped_step_matches_single_process():
    import socket
    import torch.multiprocessing as mp
    from ultravox_b200 import ops
    from ultravox_b200.training import AdapterTrainer
    with socket.socket() as sck:
        sck.bind(("127.0.0.1", 0))
        port = sck.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in range(2)], key=lambda t: t[0])
    for p_ in procs:
        p_.join(timeout=60)
        assert p_.exitcode == 0
    (_, flat0, norm0, coef0, scale0), (_, flat1, norm1, _, _) = res
    assert torch.equal(flat0, flat1) and norm0 == norm1
    assert scale0 == 0.25 and coef0 < 1.0                        # 1 / (world * accumulation steps); clipping active
    cfg, model, padded, batch = _setup([16000 * 2] * 4)
    mel = ops.logmel(torch.from_numpy(padded).cuda(), cfg.audio_config.num_mel_bins)
    tr = AdapterTrainer(model, lr=1e-3)
    tr.forward_backward(audio_values=mel, **batch)
    want = float(tr.grad.double().norm())
    assert abs(norm0 - want) < 2e-2 * want, (norm0, want)
