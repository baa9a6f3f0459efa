"""Learning-rate schedules of the released recipes, as a per-step table the optimizer kernel reads on the device.

The reference trains through HF ``Seq2SeqTrainer`` (ref:ultravox/training/train.py:250-307): ``lr_scheduler`` (default
``"cosine"``, ref config_base.py:151; ``"cosine_with_min_lr"`` with ``min_lr_rate: 0.1`` in meta_config.yaml:29-30) and
``lr_warmup_steps`` (a value < 1 is a warmup ratio, ref train.py:292-293) go to ``transformers.get_scheduler``, a ``LambdaLR``
stepped once after every optimizer step.  ``LambdaLR`` sets lr = base * lambda(0) before the first step, so optimizer step k
(1-based) runs with base * lambda(k - 1).  The lambdas below restate transformers 5.5's (``optimization.py``) operation for
operation in double; the table rounds each value to fp32 once.
"""
from __future__ import annotations

import math
from typing import Optional, Union

import torch

SCHEDULERS = ("constant", "constant_with_warmup", "linear", "cosine", "cosine_with_min_lr")


def warmup_steps_for(warmup: Union[int, float], num_training_steps: Optional[int]) -> int:
    """``TrainingArguments.get_warmup_steps``: a value >= 1 is a step count, a value < 1 a ratio of the total, rounded up."""
    if warmup >= 1:
        return int(warmup)
    if warmup == 0:
        return 0
    if num_training_steps is None:
        raise ValueError("a warmup ratio needs num_training_steps")
    return math.ceil(num_training_steps * warmup)


def lr_lambda(name: str, warmup: int, num_training_steps: Optional[int], base_lr: float, num_cycles: float = 0.5,
              min_lr: Optional[float] = None, min_lr_rate: Optional[float] = None):
    """lambda(step) of ``transformers.get_scheduler(name, ...)``; raises ``ValueError`` for any other scheduler name."""
    if name not in SCHEDULERS:
        raise ValueError(f"lr_scheduler {name!r} is not supported (supported: {', '.join(SCHEDULERS)})")
    if name == "constant":
        return lambda s: 1
    if name == "constant_with_warmup":
        return lambda s: float(s) / float(max(1.0, warmup)) if s < warmup else 1.0
    if num_training_steps is None:
        raise ValueError(f"lr_scheduler {name!r} needs num_training_steps")
    T = num_training_steps
    if name == "linear":
        return lambda s: (float(s) / float(max(1, warmup)) if s < warmup
                          else max(0.0, float(T - s) / float(max(1, T - warmup))))
    rate = 0.0
    if name == "cosine_with_min_lr":
        if (min_lr is None) == (min_lr_rate is None):
            raise ValueError("cosine_with_min_lr needs exactly one of min_lr / min_lr_rate")
        rate = min_lr / base_lr if min_lr is not None else min_lr_rate

    def cosine(s):
        if s < warmup:
            return float(s) / float(max(1, warmup))
        progress = float(s - warmup) / float(max(1, T - warmup))
        factor = 0.5 * (1.0 + math.cos(math.pi * float(num_cycles) * 2.0 * progress))
        factor = factor * (1 - rate) + rate
        return max(0, factor)
    return cosine


def lr_values(name: str, base_lr: float, warmup: Union[int, float] = 0, num_training_steps: Optional[int] = None,
              **scheduler_kwargs) -> list:
    """The scheduler's lr (double) after 0, 1, ... scheduler steps: entry k is what optimizer step k + 1 uses.  Length
    num_training_steps + 1; without num_training_steps (constant schedules only) the warmup plus one constant entry, which the
    device lookup repeats for every later step."""
    w = warmup_steps_for(warmup, num_training_steps)
    lam = lr_lambda(name, w, num_training_steps, base_lr, **scheduler_kwargs)
    n = num_training_steps + 1 if num_training_steps is not None else w + 1
    return [base_lr * lam(k) for k in range(n)]


def lr_table(name: str, base_lr: float, warmup: Union[int, float] = 0, num_training_steps: Optional[int] = None, device=None,
             **scheduler_kwargs) -> torch.Tensor:
    """``lr_values`` rounded once to fp32: the ``lr_table`` of ``uvx_grad_norm_clip``."""
    return torch.tensor(lr_values(name, base_lr, warmup, num_training_steps, **scheduler_kwargs), dtype=torch.float32,
                        device=device)
