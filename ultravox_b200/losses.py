"""Losses of the hot path (CUDA, through libuvx)."""
from __future__ import annotations

import torch

from ._lib import check, lib
from .ops import _cuda, _stream


def causal_lm_loss(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100, keep: dict | None = None,
                   shift: bool = True):
    """Next-token cross entropy, fp32 (hf:loss/loss_utils.py:28-67).  logits [B, S, V] fp32, labels [B, S]; with
    ``shift=False`` logits are [R, V] pre-gathered rows and labels [R] their targets."""
    _cuda(logits, torch.float32, "logits"), _cuda(labels, torch.int64, "labels")
    if logits.dim() == 2:
        logits = logits[None]
        labels = labels.reshape(1, -1)
    B, S, V = logits.shape
    if labels.shape != (B, S):
        raise ValueError(f"labels {tuple(labels.shape)} do not match logits {tuple(logits.shape)}")
    lg = logits.reshape(B * S, V)
    if lg.stride(-1) != 1 or lg.stride(0) % 4 != 0 or lg.data_ptr() % 16 != 0:
        lg = lg.contiguous()                      # the kernels read unit-stride rows with 128-bit loads
    labels = labels.contiguous()
    row_loss = torch.empty(B * S, dtype=torch.float32, device=logits.device)
    row_lse = torch.empty_like(row_loss)
    out = torch.empty(2, dtype=torch.float32, device=logits.device)
    check(lib().uvx_ce_loss(lg.data_ptr(), lg.stride(0), labels.data_ptr(), B, S, V, ignore_index, int(shift),
                            row_loss.data_ptr(), row_lse.data_ptr(), out.data_ptr(), _stream()), "uvx_ce_loss")
    if keep is not None:
        keep.update(row_lse=row_lse, loss2=out, logits2d=lg, labels=labels, B=B, S=S, V=V, shift=int(shift),
                    ignore_index=ignore_index)
    return out[0]


def causal_lm_loss_bwd(keep: dict, grad_scale: float = 1.0) -> torch.Tensor:
    """d(loss)/d(logits) as bf16 [B*S, V] for the rows/labels recorded by ``causal_lm_loss(keep=...)``."""
    lg = keep["logits2d"]
    d = torch.empty(lg.shape, dtype=torch.bfloat16, device=lg.device)
    check(lib().uvx_ce_bwd(lg.data_ptr(), lg.stride(0), keep["labels"].data_ptr(), keep["B"], keep["S"], keep["V"],
                           keep["ignore_index"], keep["shift"], keep["row_lse"].data_ptr(), keep["loss2"].data_ptr(),
                           grad_scale, d.data_ptr(), _stream()), "uvx_ce_bwd")
    return d


def prediction_rows(labels: torch.Tensor, ignore_index: int = -100):
    """Host-side index bookkeeping of ``_get_prediction_mask`` (ref ultravox_model.py:158-200): flat row indices
    (b*S + s) where the model predicts a labelled token (label mask shifted by one) and, per sequence, whether the row is
    the last such position (the EOT prediction)."""
    lab = labels.to("cpu")
    B, S = lab.shape
    pred = torch.zeros(B, S, dtype=torch.bool)
    pred[:, :-1] = lab[:, 1:] != ignore_index
    rows = torch.nonzero(pred.reshape(-1)).reshape(-1)
    is_eot = torch.zeros(rows.numel(), dtype=torch.bool)
    b_of = rows // S
    for b in range(B):
        idx = torch.nonzero(b_of == b).reshape(-1)
        if idx.numel() > 0:
            is_eot[idx[-1]] = True
    return rows, is_eot


def kl_distill_loss(student: torch.Tensor, teacher: torch.Tensor, is_eot: torch.Tensor, temperature: float = 2.0,
                    eot_loss_weight: float = 1.0, keep: dict | None = None) -> torch.Tensor:
    """KL(teacher || student) at temperature T, "batchmean" over the rows, + eot_loss_weight x the same over the EOT rows
    (ref ultravox_model.py:228-255).  student / teacher: [R, V] fp32 rows gathered at the prediction positions."""
    _cuda(student, torch.float32, "student"), _cuda(teacher, torch.float32, "teacher")
    if student.dim() != 2 or teacher.shape != student.shape:
        raise ValueError(f"student {tuple(student.shape)} and teacher {tuple(teacher.shape)} must be the same [R, V]")
    # the kernels take ONE row stride for both: hand them contiguous rows (a no-op for the lm_head outputs of training)
    student, teacher = student.contiguous(), teacher.contiguous()
    R, V = student.shape
    n_eot = int(is_eot.sum())
    w = torch.full((R,), 1.0 / R, dtype=torch.float32)
    if eot_loss_weight > 0 and n_eot > 0:
        w[is_eot] += eot_loss_weight / n_eot
    w = w.to(student.device)
    row_kl = torch.empty(R, dtype=torch.float32, device=student.device)
    lse_s, lse_t = torch.empty_like(row_kl), torch.empty_like(row_kl)
    out = torch.empty(1, dtype=torch.float32, device=student.device)
    check(lib().uvx_kl_loss(student.data_ptr(), teacher.data_ptr(), student.stride(0), R, V, temperature, w.data_ptr(),
                            row_kl.data_ptr(), lse_s.data_ptr(), lse_t.data_ptr(), out.data_ptr(), _stream()), "uvx_kl_loss")
    if keep is not None:
        keep.update(kind="kl", student=student, teacher=teacher, w=w, lse_s=lse_s, lse_t=lse_t, T=temperature)
    return out[0]


def kl_distill_loss_bwd(keep: dict, grad_scale: float = 1.0) -> torch.Tensor:
    s, t = keep["student"], keep["teacher"]
    d = torch.empty(s.shape, dtype=torch.bfloat16, device=s.device)
    check(lib().uvx_kl_bwd(s.data_ptr(), t.data_ptr(), s.stride(0), s.shape[0], s.shape[1], keep["T"], keep["w"].data_ptr(),
                           keep["lse_s"].data_ptr(), keep["lse_t"].data_ptr(), grad_scale, d.data_ptr(), _stream()), "uvx_kl_bwd")
    return d
