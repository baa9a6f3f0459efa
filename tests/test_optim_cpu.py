"""Optimizer-step semantics of the released recipes that need no GPU: the learning-rate table against transformers' own
schedulers, and the claim that every tensor AdapterTrainer trains is in HF Trainer's weight-decay group."""
import math
import types

import pytest
import torch

transformers = pytest.importorskip("transformers")

from ultravox_b200 import lr_schedule  # noqa: E402

CASES = [
    ("constant", {}),
    ("constant_with_warmup", {}),
    ("linear", {}),
    ("cosine", {}),
    ("cosine", {"num_cycles": 0.25}),
    ("cosine_with_min_lr", {"min_lr_rate": 0.1}),
    ("cosine_with_min_lr", {"min_lr": 3e-4}),
]


def _hf_lrs(name, base, warmup_steps, total, kwargs):
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.AdamW([p], lr=base)
    sch = transformers.get_scheduler(name, opt, num_warmup_steps=warmup_steps, num_training_steps=total,
                                     scheduler_specific_kwargs=dict(kwargs))
    out = []
    for _ in range(total + 1):
        out.append(opt.param_groups[0]["lr"])
        opt.step()
        sch.step()
    return out


@pytest.mark.parametrize("name,kwargs", CASES)
@pytest.mark.parametrize("warmup,total", [(0, 10), (3, 10), (1000, 1200), (0.1, 57), (0.03, 1000), (0.5, 7)])
def test_lr_table_equals_transformers_get_scheduler(name, kwargs, warmup, total):
    base = 2e-3
    w = math.ceil(total * warmup) if warmup < 1 else warmup    # TrainingArguments.get_warmup_steps
    args = types.SimpleNamespace(warmup_steps=warmup)   # the method reads only this field
    assert transformers.TrainingArguments.get_warmup_steps(args, total) == w == lr_schedule.warmup_steps_for(warmup, total)
    want = _hf_lrs(name, base, w, total, kwargs)
    got = lr_schedule.lr_values(name, base, warmup, total, **kwargs)
    assert got == want                                                     # exact, in double
    table = lr_schedule.lr_table(name, base, warmup, total, **kwargs)
    assert table.dtype == torch.float32 and table.numel() == total + 1
    assert torch.equal(table, torch.tensor(want, dtype=torch.float64).to(torch.float32))


def test_cosine_with_min_lr_warmup_example():
    got = [v / 2e-3 for v in lr_schedule.lr_values("cosine_with_min_lr", 2e-3, 3, 10, min_lr_rate=0.1)]
    want = [0, .333, .667, 1, .955, .831, .650, .450, .269, .145]
    assert all(abs(a - b) < 6e-4 for a, b in zip(got, want)), got
    assert got[0] == 0.0                                                   # HF's first update runs with lr = 0


def test_constant_schedules_without_total():
    assert lr_schedule.lr_values("constant", 1e-3) == [1e-3]
    assert lr_schedule.lr_values("constant_with_warmup", 1e-3, 4) == [0.0, 2.5e-4, 5e-4, 7.5e-4, 1e-3]


@pytest.mark.parametrize("name", ["polynomial", "cosine_with_restarts", "inverse_sqrt", "reduce_lr_on_plateau",
                                  "warmup_stable_decay", "nonsense"])
def test_unsupported_scheduler_raises(name):
    with pytest.raises(ValueError):
        lr_schedule.lr_values(name, 1e-3, 0, 10)


def test_decaying_schedule_needs_total_and_min_lr_args():
    with pytest.raises(ValueError):
        lr_schedule.lr_values("cosine", 1e-3, 2)
    with pytest.raises(ValueError):
        lr_schedule.lr_values("cosine_with_min_lr", 1e-3, 2, 10)
    with pytest.raises(ValueError):
        lr_schedule.lr_values("cosine_with_min_lr", 1e-3, 2, 10, min_lr=1e-4, min_lr_rate=0.1)
    with pytest.raises(ValueError):
        lr_schedule.warmup_steps_for(0.1, None)


def test_every_trained_tensor_is_in_hf_weight_decay_group():
    """Trainer.get_decay_parameter_names on a module carrying the projector's names (its norms are LlamaRMSNorm subclasses,
    as in the reference's UltravoxProjector) and the encoder-LoRA names: nothing is excluded, so every trained tensor is in one
    decay group, as AdapterTrainer applies weight decay."""
    from transformers import Trainer
    from transformers.models.llama.modeling_llama import LlamaRMSNorm

    class RMSNorm(LlamaRMSNorm):
        pass

    proj = torch.nn.Module()
    proj.ln_pre = RMSNorm(16)
    proj.linear_1 = torch.nn.Linear(16, 8, bias=False)
    proj.ln_mid = RMSNorm(4)
    proj.ln_post = RMSNorm(4)
    proj.linear_2 = torch.nn.Linear(4, 4, bias=False)
    attn = torch.nn.Module()
    for name in ("q_proj", "k_proj"):
        lin = torch.nn.Module()
        lin.lora_A = torch.nn.ModuleDict({"default": torch.nn.Linear(8, 2, bias=False)})
        lin.lora_B = torch.nn.ModuleDict({"default": torch.nn.Linear(2, 8, bias=False)})
        setattr(attn, name, lin)
    layer = torch.nn.Module()
    layer.self_attn = attn
    tower = torch.nn.Module()
    tower.layers = torch.nn.ModuleList([layer])
    root = torch.nn.Module()
    root.multi_modal_projector = proj
    root.audio_tower = torch.nn.Module()
    root.audio_tower.base_model = torch.nn.Module()
    root.audio_tower.base_model.model = tower
    names = [n for n, _ in root.named_parameters()]
    assert len(names) == 9 and "multi_modal_projector.ln_mid.weight" in names
    assert "audio_tower.base_model.model.layers.0.self_attn.q_proj.lora_A.default.weight" in names
    assert sorted(Trainer.get_decay_parameter_names(None, root)) == sorted(names)
