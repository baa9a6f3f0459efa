"""Adapter-only training step (SURVEY.md 8a-14, 8a-16, cfg3): encoder and LLM frozen, projector trained.

What the reference does with HF Trainer + autograd + DDP (``ref:ultravox/training/train.py:250-330``:
``model(**batch)`` -> ``loss.backward()`` -> DDP bucket all-reduce -> AdamW), written out explicitly over libuvx kernels:

  forward   encoder (no grad) -> projector (activations kept) -> splice -> Llama layers (per-layer inputs kept) ->
            final norm -> logits ONLY for rows that carry a label (the reference computes all rows) -> fp32 CE
  backward  CE -> lm_head dgrad (row-scattered) -> per layer {down, SwiGLU, gate/up, RMSNorm, o_proj, attention,
            RoPE, qkv, RMSNorm} data gradients against pre-transposed frozen weights (no weight gradients - the LLM
            is frozen, ref apply_lora r=0) -> gather at the audio positions -> projector dgrad + the four weight
            gradients (fp32, written straight into one flat buffer)
  exchange  ONE all-reduce (NCCL over NVLink / NVSwitch via torch.distributed) on the flat projector gradient,
            averaged over ranks - the only collective on the path (SURVEY.md 8e)
  update    one AdamW launch over the flat parameter buffer (fp32 moments, bf16 parameters)

With any of ``max_grad_norm`` / ``lr_scheduler`` / ``warmup_steps`` / ``num_training_steps`` / ``scheduler_kwargs`` /
``grad_accum_steps`` set, ``train_step`` runs the optimizer step of the released recipes (HF ``Trainer``: ``max_grad_norm`` 1.0,
warmup + cosine schedules, ``grad_accum_steps`` 2-6): micro-batch gradients are accumulated in fp32, and every
``grad_accum_steps``-th call does one all-reduce, ``uvx_grad_norm_clip`` (global L2 norm of the averaged gradient, clip
coefficient, device step += 1, lr from the schedule table) and ``uvx_adamw_multi`` over every trained tensor - two launches that
read every per-step scalar from device memory (``optimizer_step_device``, CUDA-graph capturable).
"""
from __future__ import annotations

from typing import Optional, Union

import torch

from . import lr_schedule, ops
from .model import BF16, UltravoxModel


class AdapterTrainer:
    def __init__(self, model: UltravoxModel, lr: float = 2e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, process_group=None, encoder_lora=None, max_grad_norm: Optional[float] = None,
                 lr_scheduler: str = "constant", warmup_steps: Union[int, float] = 0, num_training_steps: Optional[int] = None,
                 scheduler_kwargs: Optional[dict] = None, grad_accum_steps: int = 1):
        """``encoder_lora`` (``autograd.EncoderLora``): also train LoRA adapters on the encoder's q / k projections - the
        ``audio_model_lora_config: {r: 8}`` of the released recipes (ref:ultravox/training/configs/v0.5_config.yaml:5-6); the
        encoder then runs its training forward (activations kept) and a full data-gradient backward.

        The HF ``TrainingArguments`` of the recipes' optimizer step (ref train.py:250-307): ``max_grad_norm`` (None = no clipping;
        HF's default is 1.0), ``lr_scheduler`` (``lr_schedule.SCHEDULERS``; others raise ``ValueError``) with ``warmup_steps``
        (steps, or a ratio of ``num_training_steps`` if < 1) and ``scheduler_kwargs`` (``num_cycles``, ``min_lr`` /
        ``min_lr_rate``), ``num_training_steps`` (needed by the decaying schedules; a step past it raises) and
        ``grad_accum_steps`` (micro-batches per optimizer step, each loss divided by it).  With all of them at their defaults
        every method behaves as it did without them: constant lr, no clipping, one batch per step, and ``optimizer_step``
        always runs that plain per-tensor AdamW."""
        self.model = model
        self.lora = encoder_lora
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.pg = process_group
        pj = model.multi_modal_projector
        n = pj.flat.numel()
        dev = pj.flat.device
        self.grad = torch.zeros(n, dtype=torch.float32, device=dev)     # flat fp32 gradient (all-reduced)
        self.m = torch.zeros(n, dtype=torch.float32, device=dev)
        self.v = torch.zeros(n, dtype=torch.float32, device=dev)
        self.lora_state = []
        if encoder_lora is not None:
            for prm, _ in encoder_lora.params_and_grads():
                self.lora_state.append((torch.zeros(prm.numel(), dtype=torch.float32, device=dev),
                                        torch.zeros(prm.numel(), dtype=torch.float32, device=dev)))
        self.step_count = 0
        self.last = {}
        self._comm_stream: Optional[torch.cuda.Stream] = None
        self._pending: list = []
        self.max_grad_norm = max_grad_norm
        self.grad_accum_steps = int(grad_accum_steps)
        if self.grad_accum_steps < 1:
            raise ValueError("grad_accum_steps must be >= 1")
        self.schedule = dict(name=lr_scheduler, warmup_steps=warmup_steps, num_training_steps=num_training_steps,
                             kwargs=dict(scheduler_kwargs or {}))
        self.recipe = (max_grad_norm is not None or lr_scheduler != "constant" or warmup_steps != 0 or num_training_steps is not None
                       or bool(scheduler_kwargs) or self.grad_accum_steps != 1)
        if self.recipe:
            self._init_recipe_step(dev)

    def _init_recipe_step(self, dev):
        from .dist_utils import group_world_size
        sch = self.schedule
        self.lr_table = lr_schedule.lr_table(sch["name"], self.lr, sch["warmup_steps"], sch["num_training_steps"], device=dev,
                                             **sch["kwargs"])
        self.opt_step = torch.zeros(1, dtype=torch.int64, device=dev)     # device step (torch's state["step"])
        self.opt_lr = torch.zeros(1, dtype=torch.float32, device=dev)     # lr of the last optimizer step
        self.norm_coef = torch.zeros(2, dtype=torch.float32, device=dev)  # [total grad norm, clip coefficient] of the last step
        self._norm_ws = ops.norm_workspace(dev)
        self._scale_host = 1.0 / (group_world_size(self.pg) * self.grad_accum_steps)
        self.grad_scale = torch.full((1,), self._scale_host, dtype=torch.float32, device=dev)
        lora_pg = self.lora.params_and_grads() if self.lora is not None else []
        self._params = [self.model.multi_modal_projector.flat] + [prm.data.view(-1) for prm, _ in lora_pg]
        self._grads = [self.grad] + [g.view(-1) for _, g in lora_pg]
        self._m = [self.m] + [m1 for m1, _ in self.lora_state]
        self._v = [self.v] + [v1 for _, v1 in self.lora_state]
        self.phase = 0                 # micro-batches accumulated towards the next optimizer step
        self._losses: list = []
        if self.grad_accum_steps > 1:  # one flat fp32 accumulator (projector | LoRA): one all-reduce per optimizer step
            self.acc = torch.zeros(sum(g.numel() for g in self._grads), dtype=torch.float32, device=dev)
            self._accs = list(torch.split(self.acc, [g.numel() for g in self._grads]))
        self._step_grads = self._accs if self.grad_accum_steps > 1 else self._grads

    def grad_view(self, name: str) -> torch.Tensor:
        off, n, shape = self.model.multi_modal_projector.slices[name]
        return self.grad[off:off + n].view(*shape)

    # -- forward + backward --------------------------------------------------------------------------
    def forward_backward(self, input_ids, audio_values, audio_token_start_idx, audio_lens, audio_token_len,
                         audio_batch_size, labels, audio_tm: Optional[torch.Tensor] = None, alt_input_ids=None,
                         alt_labels=None, alt_attention_mask=None, attention_mask=None, audio_waveforms=None,
                         audio_num_frames=None, audio_pad_frames=None, **_) -> torch.Tensor:
        """Accumulates d(loss)/d(projector) into ``self.grad`` (zeroed first) and returns the loss (device scalar).  Drives the
        same forward / backward pieces as the autograd path (``autograd.py``) without building a graph; labels follow the HF
        convention; ``attention_mask`` may carry right padding."""
        from . import autograd as ag
        m, cfg = self.model, self.model.config
        lm, pj = m.language_model, m.multi_modal_projector
        dev = m.device
        input_ids = input_ids.to(dev)
        B, S = input_ids.shape
        Dm = m.config.text_config.hidden_size
        kv_start, kv_len = m._pad_bounds(attention_mask.to(dev) if attention_mask is not None else None)
        if kv_start is not None:
            raise NotImplementedError("training batches are right-padded (ref ultravox_processing.py:43-51); left padding is for generation")
        self.grad.zero_()
        with torch.no_grad():
            # ---- forward: audio tower (frozen, nothing kept) + projector (kept)
            if audio_tm is None and audio_waveforms is not None:
                audio_tm = m.mel_chunks_from_waveforms(audio_waveforms, audio_num_frames, audio_pad_frames=audio_pad_frames)
            if audio_tm is None:
                audio_tm = ops.mel_to_timemajor(audio_values.to(dev, torch.float32))
            sv_e = None
            if self.lora is not None:
                self.lora.merge_into(m)                                            # q|k|v weights <- base + s B A (this step's adapters)
                enc, sv_e = ag.encoder_forward_train(m, audio_tm, audio_lens)
            else:
                enc = m.encode_audio(audio_tm, audio_lens).clone()                 # [N, T2, d]
            aud, sv_p = ag.projector_forward(m, enc)
            src = ops.splice_plan(audio_token_start_idx.to(dev, torch.int64).contiguous(),
                                  audio_token_len.to(dev, torch.int32).contiguous(),
                                  audio_batch_size.to(dev, torch.int64).reshape(-1).contiguous(), B, S, sv_p["rows_a"])
            h = ops.embed_splice(input_ids, lm.model.embed_tokens.weight, aud, src).view(B * S, Dm)
            # ---- forward: Llama with per-layer activations kept, loss on the labelled rows
            hn, sv_l = ag.llama_stack_forward(m, h, B, S, kv_len)
            loss, keep = ag.head_loss_forward(m, hn, labels, alt_input_ids, alt_labels)
            # ---- backward: head -> frozen LLM (data gradients only) -> splice rows -> projector (fp32 weight gradients
            #      straight into the flat buffer)
            dh = ag.llama_stack_backward(m, sv_l, ag.head_loss_backward(m, keep))
            d_aud = ops.gather_rows(dh, ops.splice_inverse(src, sv_p["N"] * sv_p["rows_a"]))
            names = ag.projector_param_names(cfg)
            d_enc = ag.projector_backward(m, sv_p, d_aud, {n: self.grad_view(n) for n in names}, want_d_enc=sv_e is not None)
            if sv_e is not None:
                self.lora.zero_grad()
                ag.encoder_backward(m, sv_e, d_enc, self.lora)
        self.last = dict(loss=loss, rows=keep["n_rows"])
        return loss

    # -- exchange + update ---------------------------------------------------------------------------
    def all_reduce(self) -> float:
        """The single data-path collective: SUM of the flat projector gradient over the data-parallel ranks (NCCL over NVLink /
        NVSwitch when launched with one process per GPU).  Returns the scale (1 / world) the optimizer kernel applies - the
        mean is folded into ``uvx_adamw(grad_scale)`` instead of a separate pass over the 201 MB buffer."""
        from .dist_utils import allreduce_sum_
        if self.lora is not None:
            for _, g in self.lora.params_and_grads():
                allreduce_sum_(g, self.pg)
        return allreduce_sum_(self.grad, self.pg)

    def optimizer_step(self, grad_scale: float = 1.0):
        self.step_count += 1
        ops.adamw_(self.model.multi_modal_projector.flat, self.grad, self.m, self.v, self.step_count, self.lr, self.betas,
                   self.eps, self.wd, grad_scale)
        if self.lora is not None:
            for (prm, g), (m1, v1) in zip(self.lora.params_and_grads(), self.lora_state):
                ops.adamw_(prm.data.view(-1), g.view(-1), m1, v1, self.step_count, self.lr, self.betas, self.eps, self.wd, grad_scale)

    def optimizer_step_device(self) -> None:
        """The recipes' optimizer step on the gradients of this step (the accumulators with ``grad_accum_steps`` > 1, else
        ``grad`` and the LoRA gradients), already all-reduced: ``uvx_grad_norm_clip`` (norm of ``grad_scale`` x gradient,
        clip coefficient, device step += 1, lr = schedule[step - 1]) then ``uvx_adamw_multi`` over every trained tensor.  Two
        launches, no host sync and no host value that changes between steps, so it can be captured in a CUDA graph.  The host
        mirror ``step_count`` is advanced by ``train_step``, not here."""
        if not self.recipe:
            raise RuntimeError("optimizer_step_device needs the recipe optimizer (max_grad_norm / lr_scheduler / grad_accum_steps ...)")
        ops.grad_norm_clip(self._step_grads, self.grad_scale, self.max_grad_norm, self._norm_ws, out=self.norm_coef,
                           step=self.opt_step, lr_table=self.lr_table, lr=self.opt_lr)
        ops.adamw_multi_(self._params, self._step_grads, self._m, self._v, self.opt_lr, self.opt_step, self.grad_scale,
                         coef=self.norm_coef[1:], betas=self.betas, eps=self.eps, weight_decay=self.wd)

    def train_step(self, **batch) -> torch.Tensor:
        """One micro-batch: forward + backward, and (every ``grad_accum_steps``-th call with the recipe optimizer) the exchange
        and the optimizer step.  Returns this micro-batch's loss; after an optimizer step ``last`` also holds ``grad_norm``
        (total norm before clipping), ``lr`` (the lr that step used) and ``loss`` (mean over its micro-batches), as device
        scalars."""
        if not self.recipe:
            loss = self.forward_backward(**batch)
            scale = self.all_reduce()
            self.optimizer_step(scale)
            return loss
        total = self.schedule["num_training_steps"]
        if self.phase == 0 and total is not None and self.step_count >= total:
            raise RuntimeError(f"optimizer step {self.step_count + 1} is past num_training_steps = {total}")
        loss = self.forward_backward(**batch)
        k = self.grad_accum_steps
        if k > 1:
            ops.grad_accumulate_(self._accs, self._grads, assign=self.phase == 0)
        self._losses.append(loss)
        self.phase += 1
        if self.phase < k:
            return loss
        from .dist_utils import allreduce_sum_
        inv_world = allreduce_sum_(self.acc, self.pg) if k > 1 else self.all_reduce()
        scale = inv_world / k
        if scale != self._scale_host:
            self.grad_scale.fill_(scale)
            self._scale_host = scale
        self.optimizer_step_device()
        self.step_count += 1
        self.phase = 0
        mean_loss = torch.stack(self._losses).sum() / k
        self._losses = []
        self.last.update(loss=mean_loss, grad_norm=self.norm_coef[0].clone(), lr=self.opt_lr[0].clone())
        return loss

    # -- checkpoint ----------------------------------------------------------------------------------
    def state_dict(self) -> dict:
        """Optimizer state for resuming (what HF's ``resume_from_checkpoint`` restores): moments, step, and with the recipe
        optimizer the device step, the schedule, the clip norm and the accumulation phase (with the partial accumulator).
        Parameters are the model's (``model.state_dict()`` / ``EncoderLora``)."""
        sd = dict(step_count=self.step_count, m=self.m.clone(), v=self.v.clone(),
                  lora_m=[m1.clone() for m1, _ in self.lora_state], lora_v=[v1.clone() for _, v1 in self.lora_state])
        if self.recipe:
            sd.update(device_step=self.opt_step.clone(), schedule=dict(self.schedule, kwargs=dict(self.schedule["kwargs"])),
                      lr=self.lr, max_grad_norm=self.max_grad_norm, grad_accum_steps=self.grad_accum_steps, phase=self.phase,
                      losses=[l.clone() for l in self._losses], acc=self.acc.clone() if self.grad_accum_steps > 1 else None)
        return sd

    def load_state_dict(self, sd: dict) -> None:
        """Restore ``state_dict()`` into a trainer built with the same arguments; training then continues bit-identically."""
        if ("device_step" in sd) != self.recipe:
            raise ValueError("state_dict and trainer disagree on the recipe optimizer (max_grad_norm / lr_scheduler / ...)")
        if self.recipe:
            mine = dict(schedule=self.schedule, lr=self.lr, max_grad_norm=self.max_grad_norm, grad_accum_steps=self.grad_accum_steps)
            for key, val in mine.items():
                if sd[key] != val:
                    raise ValueError(f"state_dict {key} = {sd[key]!r}, trainer has {val!r}")
        if len(sd["lora_m"]) != len(self.lora_state):
            raise ValueError("state_dict and trainer disagree on encoder_lora")
        self.step_count = int(sd["step_count"])
        self.m.copy_(sd["m"])
        self.v.copy_(sd["v"])
        for (m1, v1), m0, v0 in zip(self.lora_state, sd["lora_m"], sd["lora_v"]):
            m1.copy_(m0)
            v1.copy_(v0)
        if self.recipe:
            self.opt_step.copy_(sd["device_step"])
            self.phase = int(sd["phase"])
            self._losses = [l.to(self.m.device) for l in sd["losses"]]
            if sd["acc"] is not None:
                self.acc.copy_(sd["acc"])
