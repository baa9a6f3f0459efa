"""Prefill engine: the whole hot path (waveform -> log-mel -> Whisper encoder -> projector -> splice -> Llama prefill
-> last-position logits -> greedy token) recorded once into a CUDA graph and replayed per request.

This is the serving-side caller of ``UltravoxModel`` for fixed request shapes (what ``LocalInference.infer`` +
``model.generate(max_new_tokens=1)`` does in the reference, ref:ultravox/inference/infer.py:125-153,309-342), with the
host work (processor bookkeeping) hoisted out: per request only the waveform changes.  One engine per process / GPU;
multi-GPU inference is independent replicas (SURVEY.md 8e) - no collective.
"""
from __future__ import annotations

import dataclasses
import numbers
from typing import Optional

import torch

import os

from . import _lib, ops
from .model import KVCache, UltravoxModel

GEMV_MAX_B = int(os.environ.get("UVX_GEMV_MAX_B", "1"))     # decode streams up to which the linears run as matrix-vector kernels
# Rows up to which the LLM GEMMs stay on the weight-bound tiling (gemm_tc.cu pick_cfg: more rows take the tensor-bound tiles).
# SlotDecodeEngine prefills a prompt of more rows in chunks of PREFILL_ROWS - slots rows inside a mixed decode step.
PREFILL_ROWS = 256


class PrefillEngine:
    def __init__(self, model: UltravoxModel, clip_samples: int, input_ids: torch.Tensor,
                 audio_token_start_idx: torch.Tensor, audio_token_len: torch.Tensor, audio_batch_size: torch.Tensor,
                 n_clips: Optional[int] = None, use_graph: bool = True):
        """All index tensors follow the processor's output contract (one entry per encoder CHUNK: a clip longer than the encoder
        context of 3000 frames = 30 s is cut into chunks exactly like ``UltravoxProcessor._chunk_and_pad_audio``, ref
        ultravox_processing.py:153-215; ``n_clips`` waveforms of ``clip_samples`` samples each)."""
        from .processing import frame_chunks
        self.model = model
        dev = model.device
        hop = 160
        L = -(-clip_samples // hop) * hop
        T = L // hop
        ctx = model.audio_tower.max_context_length
        frames_clip = -(-clip_samples // hop)
        chunks_per_clip = -(-frames_clip // ctx)
        N = int(n_clips if n_clips is not None else audio_token_start_idx.numel() // chunks_per_clip)
        self.chunked = chunks_per_clip > 1
        self.N, self.L, self.T = N, L, T
        plan, _ = frame_chunks([frames_clip] * N, ctx)
        if len(plan) != audio_token_start_idx.numel():
            raise ValueError(f"{audio_token_start_idx.numel()} audio index entries for {len(plan)} encoder chunks")
        self.frames_host = torch.full((N,), frames_clip, dtype=torch.int64)
        self.n_mels = model.audio_tower.n_mels
        self.wave = torch.zeros(N, L, dtype=torch.float32, device=dev)          # static input buffer
        self.input_ids = input_ids.to(dev).contiguous()
        self.start = audio_token_start_idx.to(dev, torch.int64).contiguous()
        self.tok_len = audio_token_len.to(dev, torch.int32).contiguous()
        self.abs = audio_batch_size.to(dev, torch.int64).reshape(-1).contiguous()
        frames = torch.tensor([p[2] for p in plan], dtype=torch.int64)          # valid frames of every chunk
        self.kv_len = ((frames - 1) // 2 + 1).to(torch.int32).to(dev)             # encoder key lengths
        self.audio_lens_host = frames
        self.token = torch.zeros(self.input_ids.shape[0], dtype=torch.int64, device=dev)
        self.logits = None
        self.graph = None
        self.launches_per_step = 0
        self._host_token = torch.zeros(self.input_ids.shape[0], dtype=torch.int64).pin_memory()
        # warm-up outside capture: builds device tables, sets func attributes, sizes the allocator pools
        for _ in range(2):
            self._step()
        torch.cuda.synchronize()
        if use_graph:
            before = _lib.launch_count()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._step()
            self.launches_per_step = _lib.launch_count() - before
            self.graph = g
        else:
            before = _lib.launch_count()
            self._step()
            self.launches_per_step = _lib.launch_count() - before
        torch.cuda.synchronize()

    # the hot path, in order (each call is one libuvx kernel or a short sequence of them)
    def _step(self):
        m = self.model
        if self.chunked:     # log-mel once per clip (its max is per CLIP), then cut into 3000-frame chunks, continuation chunks zero-padded
            tm = m.mel_chunks_from_waveforms(self.wave, self.frames_host)
        else:
            tm = ops.logmel(self.wave, self.n_mels, want_f32=False, want_tm=True)
        enc = m.encode_audio(tm, None, kv_len=self.kv_len)
        aud = m.project_audio(enc)
        B, S = self.input_ids.shape
        src = ops.splice_plan(self.start, self.tok_len, self.abs, B, S, aud.shape[1])
        emb = ops.embed_splice(self.input_ids, m.language_model.model.embed_tokens.weight, aud, src)
        hidden = m.llama_hidden(emb)
        self.logits = ops.lm_head(hidden[:, -1, :], m.language_model.lm_head.weight)
        ops.argmax(self.logits, out=self.token)

    def run(self) -> torch.Tensor:
        """One prefill over whatever is in ``self.wave``; returns the device token tensor (no sync)."""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._step()
        return self.token

    def run_e2e(self, wave_host_pinned: torch.Tensor) -> torch.Tensor:
        """Host waveform (pinned fp32 [N, L]) in, host token out: H2D + prefill + D2H + sync."""
        self.wave.copy_(wave_host_pinned, non_blocking=True)
        self.run()
        self._host_token.copy_(self.token, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._host_token


@dataclasses.dataclass
class TokenLogprobs:
    """Log-probabilities of a request's generated tokens under the model's raw distribution (log_softmax of the LM-head logits,
    before the repetition penalty, temperature, top-k and top-p - what OpenAI-style ``logprobs`` report), one entry per new
    token: ``token_logprobs`` [n] fp32 of the chosen tokens, ``top_ids`` [n, k] int64 / ``top_logprobs`` [n, k] fp32 the k most
    likely tokens of each step (value descending, lower id first on a tie).  Device tensors."""
    token_logprobs: torch.Tensor
    top_ids: torch.Tensor
    top_logprobs: torch.Tensor


class _RowKV:
    """The KV cache as one ``[S_max]`` row per decode row (stream, beam or slot): ``cache`` [L, rows, S_max, Hkv, D]."""

    keeps_kv = False        # whether a request's KV cache can outlive its slot (conversation sessions)

    def __init__(self, cache: KVCache):
        self.cache = cache

    def map_rows(self, e: "_Decoder", R: int, mode: str) -> None:
        """Before the embedding of a step over R rows: a row's cache row is its own (or ``_mrow``'s / ``_lk_wrow``'s), nothing
        to map."""

    def attend(self, e: "_Decoder", li: int, qkv: torch.Tensor, mode: str) -> torch.Tensor:
        """The cache-touching calls of layer ``li`` of a step over the R rows of ``qkv``: RoPE on q / k + the KV append, then
        attention -> [R, Hq * D].  ``mode`` "plain": row b appends at ``pos[b]`` of cache row b and attends to it; "mixed": the
        B decode rows as in a plain step, the chunk rows appended through ``_mrow`` and attending to the prefilling slot's row;
        "lookup" (``SlotDecodeEngine``'s lookup step): row r appends through ``_lk_wrow`` / ``_lk_pos`` and attends to cache row
        ``_lk_slot[r]``, so a slot's draft rows see the positions its earlier rows appended in the same step."""
        nq, nkv, hd = e.heads
        B, R = e.B, qkv.shape[0]
        kc, vc = self.cache.k[li], self.cache.v[li]
        smax = kc.shape[1]
        att = torch.empty(R, nq * hd, dtype=torch.bfloat16, device=qkv.device)
        if mode == "lookup":
            ops.rope_kv_append_map_(qkv, nq, nkv, hd, e.cos, e.sin, e._lk_rope, kc, vc, e._lk_wrow, e._lk_pos)
            return ops.attention_rows(qkv[:, :nq * hd], kc, vc, att, nq, hd ** -0.5, e._lk_lens, e._lk_slot)
        if mode == "plain":
            ops.rope_kv_append_(qkv, nq, nkv, hd, e.cos, e.sin, e.rope_pos, kc, vc, e.pos)
        else:
            ops.rope_kv_append_map_(qkv, nq, nkv, hd, e.cos, e.sin, e._mrope, kc, vc, e._mrow, e._mpos)
        rs = qkv.stride(0)
        ops.attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), att, B, nq, nkv, 1, smax, hd,
                      (rs, rs, nkv * hd, smax * nkv * hd, nkv * hd, smax * nkv * hd, nq * hd, nq * hd), hd ** -0.5, False,
                      e.lens, 0, e.kv_start)
        if mode == "mixed":
            ops.attention_indexed(qkv[B:, :nq * hd].unsqueeze(0), kc, vc, att[B:].unsqueeze(0), nq, hd ** -0.5, *e._mscal.split(1))
        return att

    def prefill(self, model: UltravoxModel, j: int, input_ids: torch.Tensor, past: int, features: dict) -> torch.Tensor:
        """B = 1 prefill of a whole prompt into cache row ``j`` -> its last position's logits [1, V]."""
        row = KVCache(self.cache.k[:, j:j + 1], self.cache.v[:, j:j + 1])
        return model.forward(input_ids, past_key_values=row, logits_to_keep=1, **features).logits.view(1, -1)

    def install(self, j: int, S: int, n: int, pages) -> None:
        if pages is not None:
            raise ValueError("this engine keeps its KV cache in slot rows, not pages (pages must be None)")

    def release(self, j: int) -> None:
        pass


def check_kv_scales(kv_scales, layers: int) -> torch.Tensor:
    """The FP8 pool's per-layer K / V scales as a new fp32 [layers, 2] tensor (None: all 1); ValueError unless that shape with
    positive, finite values.  Always a copy: pages already written must be read back with the scales they were written with,
    whatever the caller does with its own tensor later."""
    if kv_scales is None:
        return torch.ones(layers, 2, dtype=torch.float32)
    t = torch.as_tensor(kv_scales).to(torch.float32, copy=True)
    if tuple(t.shape) != (layers, 2):
        raise ValueError(f"kv_scales must have shape [{layers}, 2] (one K and one V scale per layer), got {tuple(t.shape)}")
    if not bool((torch.isfinite(t) & (t > 0)).all()):
        raise ValueError("kv_scales must be positive and finite")
    return t


def check_lookup_k(slots: int, k) -> int:
    """The engine-wide draft maximum K of ``prompt_lookup_num_tokens`` (None -> 0, off); ValueError unless None or an integer
    in [1, LOOKUP_MAX_K] with slots * (K + 1) <= PREFILL_ROWS."""
    if k is None:
        return 0
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or not 1 <= k <= ops.LOOKUP_MAX_K:
        raise ValueError(f"prompt_lookup_num_tokens must be an integer in [1, {ops.LOOKUP_MAX_K}] (k + 1 rows of the decode "
                         f"step), got {k!r}")
    if slots * (int(k) + 1) > PREFILL_ROWS:
        raise ValueError(f"{slots} slots x (prompt_lookup_num_tokens = {k} + 1) = {slots * (int(k) + 1)} rows per step; at most "
                         f"{PREFILL_ROWS}")
    return int(k)


def check_stop_table(n) -> Optional[int]:
    """The slot engines' ``max_stop_table`` (None: off); ValueError unless None or an integer >= the table header."""
    if n is None:
        return None
    if isinstance(n, bool) or not isinstance(n, numbers.Integral) or n < ops.STOP_HEADER:
        raise ValueError(f"max_stop_table must be None or an integer >= {ops.STOP_HEADER} (int32 words per slot), got {n!r}")
    return int(n)


def check_constraint_tokens(n) -> Optional[int]:
    """The slot engines' ``max_constraint_tokens`` (None: off); ValueError unless None or an integer >= 0."""
    if n is None:
        return None
    if isinstance(n, bool) or not isinstance(n, numbers.Integral) or n < 0:
        raise ValueError(f"max_constraint_tokens must be None or an integer >= 0, got {n!r}")
    return int(n)


class _PagedKV:
    """The KV cache as a shared pool of 64-position pages, so a request's K / V can outlive its slot.  K and V are
    ``[L, kv_pages + slots, 64, Hkv, D]``: the ``kv_pages`` shareable pages, then one private idle page per slot (an idle row
    writes its pad token at position 0 there, as a contiguous idle row does in its own row).  The page table
    ``[slots, ceil(max_len / 64)]`` int32 lives on the device; the host writes a slot's row between replays (its pages at
    ``install``, its idle page at ``release``).  A page is exactly one key tile of both attention kernels, so every step computes
    the same bits as with ``_RowKV``: one ``uvx_kv_page_map`` launch per step turns each row's (slot, position) into
    (page, offset) for the unchanged mapped RoPE + append, and the attention kernels read their key tiles through the table.
    Rows that are done (finished, not yet retired) write nothing, so the last position a conversation keeps stays intact.

    ``cache`` is the one-row admission scratch ``[L, 1, max_len, Hkv, D]``: a prompt prefilled at B = 1 gathers its
    conversation's first ``past`` positions there, is prefilled like ``generate(past_key_values=...)``, and its new positions
    are scattered into its pages.

    ``kv_cache_dtype="fp8_e4m3"`` makes the pool ``float8_e4m3fn`` with per-layer K / V scales ``kv_scales`` [L, 2] fp32 on the
    device (default all 1): every write into the pool (the step's append, the admission scatter) quantizes, every read (both
    attention kernels, the admission gather into the bf16 scratch) dequantizes, as include/uvx.h states.  This class is the
    only place that knows the pool's element type.

    ``host_kv_pages`` > 0 adds a second tier: ``host_k`` / ``host_v`` ``[L, host_kv_pages, 64, Hkv, D]`` in pinned host memory,
    the device pool's dtype, allocated once here.  ``swap_out(dev_pages, host_pages)`` / ``swap_in(host_pages, dev_pages)`` move
    whole pages between the tiers with one ``uvx_kv_pages_move`` launch on the current stream, the SMs reading or writing the
    host pages over PCIe; an e4m3 page moves as its bytes, under the same per-layer scales.  Nothing waits on the host.  That is
    correct as long as every kernel that touches either tier runs on one stream (the scheduler's): a page freed by a move and
    taken by the next move, admission or step is then written only after the move has read it.  With 0 (the default) nothing is
    allocated."""

    keeps_kv = True

    def __init__(self, model: UltravoxModel, slots: int, max_len: int, kv_pages: int, kv_cache_dtype: str = "bf16",
                 kv_scales: Optional[torch.Tensor] = None, host_kv_pages: int = 0):
        lm, tc = model.language_model, model.config.text_config
        dev = model.device
        if int(kv_pages) < 1:
            raise ValueError(f"kv_pages must be >= 1, got {kv_pages}")
        L, nkv, hd = tc.num_hidden_layers, tc.num_key_value_heads, lm.head_dim
        dtype = {"bf16": torch.bfloat16, "fp8_e4m3": ops.FP8}.get(kv_cache_dtype)
        if dtype is None:
            raise ValueError(f"kv_cache_dtype must be 'bf16' or 'fp8_e4m3', got {kv_cache_dtype!r}")
        self.kv_scales = None
        if dtype == ops.FP8:
            self.kv_scales = check_kv_scales(kv_scales, L).to(dev).contiguous()
        elif kv_scales is not None:
            raise ValueError("kv_scales are for kv_cache_dtype='fp8_e4m3'")
        self.kv_pages = int(kv_pages)
        self.table_width = -(-int(max_len) // ops.PAGE)
        self.pool_k = torch.empty(L, self.kv_pages + slots, ops.PAGE, nkv, hd, dtype=dtype, device=dev)
        self.pool_v = torch.empty_like(self.pool_k)
        self.table = torch.full((slots, self.table_width), -1, dtype=torch.int32, device=dev)
        R = max(slots, PREFILL_ROWS)        # the rows of a mixed step (slots decode rows + PREFILL_ROWS - slots chunk rows)
        self.page = torch.zeros(R, dtype=torch.int32, device=dev)      # the page map's output: page / offset of every row
        self.off = torch.zeros(R, dtype=torch.int32, device=dev)
        self.cache = model.new_cache(1, max_len)
        self.pages = None                   # the admitted request's pages on the device
        if isinstance(host_kv_pages, bool) or not isinstance(host_kv_pages, numbers.Integral) or host_kv_pages < 0:
            raise ValueError(f"host_kv_pages must be an integer >= 0, got {host_kv_pages!r}")
        self.host_kv_pages = int(host_kv_pages)
        self.host_k = self.host_v = None
        if self.host_kv_pages:
            self.host_k = torch.empty(L, self.host_kv_pages, ops.PAGE, nkv, hd, dtype=dtype, pin_memory=True)
            self.host_v = torch.empty(self.host_k.shape, dtype=dtype, pin_memory=True)

    def swap_out(self, dev_pages, host_pages) -> None:
        """Device page dev_pages[j] -> host page host_pages[j], every layer, K and V (stream-ordered, no sync)."""
        self._move(self.pool_k, self.pool_v, dev_pages, self.kv_pages, self.host_k, self.host_v, host_pages, self.host_kv_pages)

    def swap_in(self, host_pages, dev_pages) -> None:
        """Host page host_pages[j] -> device page dev_pages[j], every layer, K and V (stream-ordered, no sync)."""
        self._move(self.host_k, self.host_v, host_pages, self.host_kv_pages, self.pool_k, self.pool_v, dev_pages, self.kv_pages)

    def _move(self, sk, sv, src, n_src, dk, dv, dst, n_dst) -> None:
        src, dst = [int(p) for p in src], [int(p) for p in dst]
        if not self.host_kv_pages:
            raise ValueError("no host tier: create the engine with host_kv_pages > 0")
        if len(src) != len(dst) or len(set(dst)) != len(dst) or not all(0 <= p < n_src for p in src) or \
                not all(0 <= p < n_dst for p in dst):
            raise ValueError(f"bad page lists for a move: {src} -> {dst}")
        if not src:
            return
        # one pinned buffer per move (the host allocator keeps it until its copy has run)
        lists = torch.tensor(src + dst, dtype=torch.int32).pin_memory().to(self.table.device, non_blocking=True)
        ops.kv_pages_move(sk, sv, dk, dv, lists[:len(src)], lists[len(src):])

    def map_rows(self, e: "_Decoder", R: int, mode: str) -> None:
        if mode == "lookup":        # done and prefilling slots already map to -1 (uvx_lookup_draft_slots)
            ops.kv_page_map(self.table, e._lk_wrow, e._lk_pos, self.page[:R], self.off[:R])
        else:
            ops.kv_page_map(self.table, e._mrow[:R], e._mpos[:R], self.page[:R], self.off[:R], frozen=e.done)

    def attend(self, e: "_Decoder", li: int, qkv: torch.Tensor, mode: str) -> torch.Tensor:
        """``_RowKV.attend`` through the page map and the table: every row appends at its (page, offset)."""
        nq, nkv, hd = e.heads
        B, R = e.B, qkv.shape[0]
        kp, vp = self.pool_k[li], self.pool_v[li]
        sc = None if self.kv_scales is None else self.kv_scales[li]
        rope = e._lk_rope if mode == "lookup" else e._mrope[:R]
        ops.rope_kv_append_map_(qkv, nq, nkv, hd, e.cos, e.sin, rope, kp, vp, self.page[:R], self.off[:R], kv_scale=sc)
        att = torch.empty(R, nq * hd, dtype=torch.bfloat16, device=qkv.device)
        if mode == "lookup":
            return ops.attention_paged(qkv[:, :nq * hd], kp, vp, att, nq, hd ** -0.5, self.table, e._lk_lens, kv_scale=sc,
                                       kv_row=e._lk_slot)
        ops.attention_paged(qkv[:B, :nq * hd], kp, vp, att[:B], nq, hd ** -0.5, self.table, e.lens, kv_scale=sc)
        if mode == "mixed":
            ops.attention_indexed_paged(qkv[B:, :nq * hd].unsqueeze(0), kp, vp, att[B:].unsqueeze(0), nq, hd ** -0.5, self.table,
                                        *e._mscal.split(1), kv_scale=sc)
        return att

    def prefill(self, model: UltravoxModel, j: int, input_ids: torch.Tensor, past: int, features: dict) -> torch.Tensor:
        """Gather [0, past) into the scratch row, prefill [past, S) there exactly as ``generate(past_key_values=...)`` does, scatter
        [past, S) into the pages ``install`` gave slot ``j``."""
        S = int(input_ids.shape[1])
        row = self.cache
        if past:
            ops.kv_pages_copy(row.k, row.v, self.pool_k, self.pool_v, self.pages, 0, past, to_pages=False, kv_scales=self.kv_scales)
            emb = model.prompt_embeds(input_ids, **features)       # embed + splice the whole prompt, prefill only the new suffix
            out = model.forward(input_ids[:, past:], None, emb[:, past:].contiguous(), past_key_values=KVCache(row.k, row.v, past),
                                logits_to_keep=1)
        else:
            out = model.forward(input_ids, past_key_values=KVCache(row.k, row.v), logits_to_keep=1, **features)
        ops.kv_pages_copy(row.k, row.v, self.pool_k, self.pool_v, self.pages, past, S, to_pages=True, kv_scales=self.kv_scales)
        return out.logits.view(1, -1)

    def install(self, j: int, S: int, n: int, pages) -> None:
        """Slot ``j``'s table row <- ``pages`` (page ids for positions 0, 64, 128, ...), which must cover its S + n positions."""
        pages = list(pages or [])
        if len(pages) * ops.PAGE < S + n or len(pages) > self.table_width:
            raise ValueError(f"{len(pages)} pages for a prompt of {S} tokens plus max_new_tokens={n}")
        self._set_table_row(j, pages)
        self.pages = torch.tensor(pages, dtype=torch.int32).to(self.table.device, non_blocking=True)

    def release(self, j: int) -> None:
        self._set_table_row(j, [self.kv_pages + j])

    def _set_table_row(self, j: int, pages) -> None:
        row = torch.full((self.table_width,), -1, dtype=torch.int32)
        row[:len(pages)] = torch.tensor(list(pages), dtype=torch.int32)
        self.table[j].copy_(row.pin_memory(), non_blocking=True)


class _Decoder:
    """What every decode engine shares: the KV cache ``kv`` (``_RowKV`` or ``_PagedKV``; ``cache`` is its contiguous part), the
    B decode rows' fed token, sequence, done flag and positions, the EOS ids, the RoPE tables, the step loop and its CUDA-graph
    capture.  ``extra`` rows after the decode rows carry a prompt chunk in a mixed step: ``_mpos`` / ``_mrope`` hold the cache
    position and the RoPE position of every row, ``pos`` / ``rope_pos`` are their decode part."""

    def __init__(self, model: UltravoxModel, rows: int, kv, eos_token_ids, pad_token_id: int, use_graph: bool, extra: int = 0):
        lm, tc = model.language_model, model.config.text_config
        dev = model.device
        i32 = dict(dtype=torch.int32, device=dev)
        self.model, self.B, self.kv = model, rows, kv
        self.cache = kv.cache
        self.max_len = self.cache.capacity
        self.heads = (tc.num_attention_heads, tc.num_key_value_heads, lm.head_dim)
        self._mpos = torch.zeros(rows + extra, **i32)
        self.pos = self._mpos[:rows]            # cache slot of the token being fed
        self.lens = torch.zeros(rows, **i32)    # keys visible to it (= pos + 1)
        self._mrope = torch.zeros(rows + extra, **i32)
        self.rope_pos = self._mrope[:rows]      # its RoPE position (= pos - left padding)
        self.kv_start: Optional[torch.Tensor] = None
        self.token = torch.zeros(rows, 1, dtype=torch.int64, device=dev)
        self.seq = torch.zeros(rows, self.max_len + 1, dtype=torch.int64, device=dev)
        self.done = torch.zeros(rows, **i32)
        eos = sorted(set([eos_token_ids] if isinstance(eos_token_ids, int) else (eos_token_ids or [])))
        self.eos = torch.tensor(eos, dtype=torch.int64, device=dev) if eos else None
        self.pad_id = int(pad_token_id)
        self.cos, self.sin = model._rope_tables(self.max_len + 1)
        self.graph = None
        self.use_graph = use_graph
        self.launches_per_step = 0
        self.captures = 0
        self.logits = None

    def _seed(self, rows, S: int, pad=0) -> None:
        """Positions of ``rows`` whose first new token is picked next from a prompt of S positions: the pick's finish kernel
        bumps pos, lens and rope_pos by one, so the token sits at slot S, sees S + 1 keys and has RoPE position S - pad."""
        self.pos[rows] = S - 1
        self.lens[rows] = S
        self.rope_pos[rows] = (S - 1) - pad

    # -- one step ------------------------------------------------------------------------------------------
    def _forward(self, mixed_in: Optional[torch.Tensor] = None, head_rows: Optional[torch.Tensor] = None,
                 lookup: bool = False) -> torch.Tensor:
        """Embedding -> layers -> final norm -> LM head of a step -> fp32 logits.  A plain step (``mixed_in`` None) feeds the B
        rows of ``token``.  A mixed step feeds ``mixed_in`` [R, D]: the token embedding is written into its first B rows, the
        prompt-chunk rows follow, and the LM head runs over rows ``head_rows`` only.  A lookup step (``lookup``,
        ``SlotDecodeEngine``) feeds the R rows of ``_lk_tok``."""
        m = self.model
        lm, tc = m.language_model, m.config.text_config
        B = self.B
        mode = "lookup" if lookup else ("plain" if mixed_in is None else "mixed")
        tokens = self._lk_tok if lookup else self.token
        R = tokens.shape[0] if mixed_in is None else mixed_in.shape[0]
        # one stream: matrix-vector kernels (fp32 FMAs on the CUDA cores keep up with the weight stream) with RMSNorm / SwiGLU fused
        # into their prologues; more streams: the tensor-core GEMM (at B = 8 the FMA work per weight byte is 8x and the GEMV is
        # instruction-bound)
        one = mode == "plain" and B <= GEMV_MAX_B
        eps = tc.rms_norm_eps
        self.kv.map_rows(self, R, mode)
        if mixed_in is None:
            h = ops.embed_splice(tokens, lm.model.embed_tokens.weight, None, None).view(R, tc.hidden_size)
        else:
            h = mixed_in
            ops.embed_splice(self.token, lm.model.embed_tokens.weight, None, None, out=h[:B])
        for li, layer in enumerate(lm.model.layers):
            sa, mlp = layer.self_attn, layer.mlp
            if one:     # RMSNorm rides in the matrix-vector kernel's prologue
                qkv = ops.gemv(h, sa.qkv_w, norm=(layer.input_layernorm.weight, eps))
            else:
                qkv = ops.linear(ops.rmsnorm(h, layer.input_layernorm.weight, eps), sa.qkv_w)
            att = self.kv.attend(self, li, qkv, mode)
            if one:
                h = ops.gemv(att, sa.o_proj.weight, residual=h)
                gu = ops.gemv(h, mlp.gate_up_w, norm=(layer.post_attention_layernorm.weight, eps))
                h = ops.gemv(gu, mlp.down_proj.weight, residual=h, swiglu=True)         # act_fn(gate) * up in the prologue
            else:
                h = ops.linear(att, sa.o_proj.weight, residual=h)
                x = ops.rmsnorm(h, layer.post_attention_layernorm.weight, eps)
                act = ops.swiglu(ops.linear(x, mlp.gate_up_w), gate_first=True)
                h = ops.linear(act, mlp.down_proj.weight, residual=h)
        if head_rows is not None:
            h = ops.gather_rows(h, head_rows)
        hn = ops.rmsnorm(h, lm.model.norm.weight, eps)
        return ops.lm_head(hn, lm.lm_head.weight)

    def _step(self):
        self._pick(self._forward())

    def step(self) -> torch.Tensor:
        """Feeds ``self.token`` (the previous output), writes the next token into it; returns the device tensor."""
        if self.use_graph and self.graph is None:
            self._step_warm()
        if self.graph is not None:
            self.graph.replay()
        else:
            self._step()
        return self.token

    def _step_warm(self):
        self.graph, self.launches_per_step = self._capture(self._step)

    def _capture(self, step):
        # warm-up on a scratch copy of the state, then capture; the state is restored so no token is lost (the cache row and the
        # sequence column the two trial steps write are rewritten with the same values by the first real step)
        self.captures += 1
        saved = [t.clone() for t in self._state()]
        step()
        torch.cuda.synchronize()
        for t, s0 in zip(self._state(), saved):
            t.copy_(s0)
        before = _lib.launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            step()
        launches = _lib.launch_count() - before
        for t, s0 in zip(self._state(), saved):
            t.copy_(s0)
        torch.cuda.synchronize()
        return g, launches


class DecodeEngine(_Decoder):
    """Token-by-token decoding after a prefill, the whole step (embedding -> 32/80 layers -> lm head -> logits processing ->
    greedy / sampled pick -> EOS + sequence bookkeeping -> position bump) captured ONCE in a CUDA graph and replayed per token:
    positions, KV lengths, the current token, the output sequence and the step counter all live on the device, so nothing in
    the graph changes between steps and the host never has to synchronise inside the loop.  Linear layers are weight-streaming
    matrix-vector kernels (uvx_gemv_bf16, slabs of 8 streams).  This is the serving loop of ``LocalInference._generate``
    (ref:ultravox/inference/infer.py:309-342 -> ``GenerationMixin.generate``): greedy when ``temperature in {None, 0}``,
    multinomial sampling otherwise (top-k, then top-p when ``top_p < 1``); repetition penalty as the reference pipeline sets it
    (ref ultravox_pipeline.py:95-113); left-padded batches (``kv_start`` + mask-derived RoPE positions,
    hf:generation/utils.py:707-729)."""

    def __init__(self, model: UltravoxModel, batch: int, max_len: int, use_graph: bool = True, cache=None,
                 eos_token_ids=None, pad_token_id: int = 0, temperature: float = 0.0, top_k: int = 0,
                 repetition_penalty: float = 1.0, generator: Optional[torch.Generator] = None, top_p: Optional[float] = None,
                 output_scores: bool = False, output_logits: bool = False, max_new_tokens: Optional[int] = None,
                 constraints=None, cutoffs=None, stop=None):
        """``output_scores`` / ``output_logits``: every pick (the first one, in ``begin``, is step 0) also records HF's processed
        scores / the raw logits of its rows into ``scores`` / ``raw_logits`` [max_new_tokens, batch, V] fp32, at the device
        step counter (``uvx_record_scores``).  That is one [batch, V] fp32 tensor per generated token, which is what HF's
        ``generate(output_scores=True / output_logits=True)`` holds too.  Without them nothing is allocated and the step is
        unchanged.

        ``constraints`` (``constraints.LogitsConstraints``): every pick first runs ``uvx_logits_constraints`` over the rows'
        sequences, before the repetition penalty.  None (the default): nothing is allocated and the step is unchanged.

        ``cutoffs``: (min_p, typical_p, epsilon, eta) after top-p (``uvx_sample_cutoffs`` / ``uvx_record_scores_cutoffs``), off
        encoded as (0, 1, 0, 0).  With none on (or None) the step launches exactly the kernels it launches without them.

        ``stop`` (``stop_strings.StopStrings``): every pick runs ``uvx_stop_strings`` on the picked tokens and finishes with
        ``uvx_token_finish_stop``, so a row whose token ends a stop string finishes as on an EOS id; ``fin_len`` [batch] holds
        each finished row's length at the step it finished.  None (the default): nothing is allocated and the step is unchanged."""
        super().__init__(model, batch, _RowKV(cache if cache is not None else model.new_cache(batch, max_len)), eos_token_ids,
                         pad_token_id, use_graph)
        dev = model.device
        self.cur_len = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step_idx = torch.zeros(1, dtype=torch.int32, device=dev)
        self.all_done = torch.zeros(1, dtype=torch.int32, device=dev)
        self.temperature, self.top_k = float(temperature or 0.0), int(top_k or 0)
        self.top_p = 1.0 if top_p is None else float(top_p)         # a kernel argument of the captured step, like top_k
        if not 0.0 <= self.top_p <= 1.0:
            raise ValueError(f"top_p must be in [0, 1], got {top_p}")
        self.penalty = float(repetition_penalty or 1.0)
        self.u = None
        if self.temperature > 0:
            # one uniform per (step, stream), drawn up front from the caller's (seedable) generator: the graph reads row step_idx
            self.u = torch.rand(self.max_len + 1, batch, device=dev, dtype=torch.float32, generator=generator)
        self.scratch = torch.empty(batch, self.max_len + 1, dtype=torch.float32, device=dev) if self.penalty != 1.0 else None
        self.scores = self.raw_logits = None
        if output_scores or output_logits:
            steps = int(max_new_tokens or 0)
            if not 1 <= steps <= self.max_len:
                raise ValueError(f"recording scores / logits needs max_new_tokens in [1, {self.max_len}], got {max_new_tokens}")
            shape = (steps, batch, model.language_model.lm_head.weight.shape[0])
            self.scores = torch.empty(shape, dtype=torch.float32, device=dev) if output_scores else None
            self.raw_logits = torch.empty(shape, dtype=torch.float32, device=dev) if output_logits else None
        self.constraints = None if constraints is None else constraints.device_tables(dev)
        self.cutoffs = tuple(float(v) for v in cutoffs) if ops.cutoffs_on(cutoffs) else None
        self.stop = None
        if stop is not None:
            self.stop = stop.device_table(dev)
            self.stop_hit = torch.zeros(batch, dtype=torch.int32, device=dev)
            self.fin_len = torch.zeros(batch, dtype=torch.int32, device=dev)

    # -- state ---------------------------------------------------------------------------------------------
    def begin(self, input_ids: torch.Tensor, first_logits: torch.Tensor, kv_start: Optional[torch.Tensor] = None) -> torch.Tensor:
        """After the prompt has been prefilled into ``self.cache`` (S = input_ids.shape[1] positions): seeds the sequence buffer
        and the counters, picks the first new token from ``first_logits`` [B, V] fp32.  Returns the device token tensor [B]."""
        B, S = input_ids.shape
        if S + 1 > self.max_len + 1:
            raise ValueError("prompt longer than the KV cache")
        self.seq[:, :S].copy_(input_ids)
        self.cur_len.fill_(S)
        self.step_idx.zero_()
        self.done.zero_()
        self.all_done.zero_()
        if self.stop is not None:
            self.fin_len.zero_()
        self.kv_start = kv_start
        self._seed(slice(None), S, 0 if kv_start is None else kv_start.to(torch.int32))
        self._pick(first_logits.contiguous())
        return self.token.view(-1)

    def prefill(self, inputs_embeds: torch.Tensor) -> torch.Tensor:
        """Runs the prompt through the LLM, fills the cache, returns the first generated token [B] (greedy or sampled)."""
        m = self.model
        B, S, _ = inputs_embeds.shape
        self.cache.length = 0
        hid = m.llama_hidden(inputs_embeds, self.cache)
        logits = ops.lm_head(hid[:, -1, :], m.language_model.lm_head.weight)
        self.seq[:, :S].zero_()
        return self.begin(self.seq[:, :S], logits).clone()

    def _pick(self, logits: torch.Tensor):
        """logits [B, V] fp32 -> self.token (+ sequence / EOS / counter bookkeeping), all on the device."""
        self.logits = logits
        rec = (self.temperature, self.top_k, self.top_p, self.step_idx)
        raw_first = self.raw_logits is not None and (self.penalty != 1.0 or self.constraints is not None)
        if raw_first:       # the constraints and the penalty rewrite the logits in place: take the raw copy before them
            ops.record_scores(logits, *rec, raw=self.raw_logits)
        if self.constraints is not None:
            ops.logits_constraints_(logits, self.seq, self.cur_len, self.constraints)
        if self.penalty != 1.0:
            ops.repetition_penalty_(logits, self.seq, self.cur_len, self.penalty, self.scratch)
        if self.scores is not None or (self.raw_logits is not None and not raw_first):
            ops.record_scores(logits, *rec, scores=self.scores, raw=None if raw_first else self.raw_logits, cutoffs=self.cutoffs)
        tok = self.token.view(-1)
        if self.temperature > 0:
            ops.sample(logits, self.temperature, self.top_k, self.u, self.step_idx, out=tok, top_p=self.top_p, cutoffs=self.cutoffs)
        else:
            ops.argmax(logits, out=tok)
        stop = None
        if self.stop is not None:
            ops.stop_strings(tok, self.seq, self.cur_len, self.stop, self.stop_hit)
            stop = (self.stop_hit, self.fin_len)
        ops.token_finish(tok, self.done, self.eos, self.pad_id, self.seq, self.cur_len, self.step_idx,
                         (self.pos, self.lens, self.rope_pos), self.all_done, stop=stop)

    def _state(self):
        fin = [self.fin_len] if self.stop is not None else []
        return [self.pos, self.lens, self.rope_pos, self.token, self.cur_len, self.step_idx, self.done, self.all_done] + fin


class _SeqKV(_RowKV):
    """The KV cache of ONE sequence, ``cache`` [L, 1, S_max, Hkv, D], fed by several rows of a step that are consecutive
    positions of it (prompt lookup): row i appends its K / V at ``pos[i]`` of the one cache row and attends to its first
    ``lens[i]`` positions, through a K / V batch stride of 0.  The append writes every row before the attention reads, so row i
    sees the positions rows 0..i-1 wrote in the same step, as a plain decode step of its own would have."""

    def attend(self, e: "_Decoder", li: int, qkv: torch.Tensor, mode: str) -> torch.Tensor:
        nq, nkv, hd = e.heads
        R = qkv.shape[0]
        kc, vc = self.cache.k[li], self.cache.v[li]
        smax = kc.shape[1]
        ops.rope_kv_append_(qkv, nq, nkv, hd, e.cos, e.sin, e.rope_pos, kc.expand(R, -1, -1, -1), vc.expand(R, -1, -1, -1), e.pos)
        att = torch.empty(R, nq * hd, dtype=torch.bfloat16, device=qkv.device)
        rs = qkv.stride(0)
        ops.attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), att, R, nq, nkv, 1, smax, hd,
                      (rs, rs, nkv * hd, 0, nkv * hd, 0, nq * hd, nq * hd), hd ** -0.5, False, e.lens, 0, None)
        return att


class LookupDecodeEngine(_Decoder):
    """Prompt lookup decoding of one sequence (hf:generation/utils.py ``_assisted_decoding`` with
    hf:generation/candidate_generator.py ``PromptLookupCandidateGenerator``, transformers 5.5).  Every step is one CUDA graph
    replay over k + 1 rows: ``uvx_lookup_draft`` drafts up to k tokens from the sequence's own earlier n-grams and feeds the
    last token followed by the drafts, the forward runs the k + 1 rows as positions of the one cache row (``_SeqKV``; the
    linears on the decode-form GEMM, whose output rows do not depend on each other), each row is picked exactly as plain
    decoding picks that position (penalty over the sequence up to it, uniform and score index n_new + i), and
    ``uvx_lookup_accept`` keeps the picks that agree with the drafts plus one.  So the tokens are those of ``DecodeEngine``
    for the same call, sampled ones included; a step yields 1 to k + 1 of them.

    ``cache`` needs S + max_new_tokens + k positions: the last check writes up to k positions past the budget.  ``accepted``
    [max_new_tokens] int32 logs each step's accepted draft count (``step_idx`` steps so far); ``cur_len`` / ``n_new`` /
    ``done`` are the device counters the host reads."""

    def __init__(self, model: UltravoxModel, prompt_len: int, max_new_tokens: int, num_tokens: int, ngram: int = 2,
                 use_graph: bool = True, cache=None, eos_token_ids=None, pad_token_id: int = 0, temperature: float = 0.0,
                 top_k: int = 0, top_p: Optional[float] = None, repetition_penalty: float = 1.0,
                 generator: Optional[torch.Generator] = None, output_scores: bool = False, output_logits: bool = False,
                 uniforms: Optional[int] = None, constraints=None, cutoffs=None, stop=None):
        """``uniforms``: how many uniforms to draw when sampling, default S + max_new_tokens + 1 - the count ``DecodeEngine``
        draws (its cache capacity + 1) for the same call, so that a seeded ``generator`` gives the same tokens.
        ``constraints``: as ``DecodeEngine``'s, row i over the sequence up to its position (``uvx_logits_constraints_rows``).
        ``cutoffs``: as ``DecodeEngine``'s, on every row.
        ``stop``: as ``DecodeEngine``'s; row i is checked after the sequence up to its position (``uvx_stop_strings_rows``) and
        the accept is cut at the first row that ends a stop string (``uvx_lookup_accept_stop``), which finishes the sequence."""
        k, n, S, N = int(num_tokens), int(ngram), int(prompt_len), int(max_new_tokens)
        if not 1 <= k <= ops.LOOKUP_MAX_K:
            raise ValueError(f"prompt_lookup_num_tokens must be in [1, {ops.LOOKUP_MAX_K}], got {num_tokens}")
        if n < 1:
            raise ValueError(f"max_matching_ngram_size must be >= 1, got {ngram}")
        if N < 1 or S < 1:
            raise ValueError(f"need a prompt and max_new_tokens >= 1, got S = {S}, max_new_tokens = {N}")
        need = S + N + k
        if cache is None:
            cache = model.new_cache(1, need)
        if cache.k.shape[1] != 1 or cache.capacity < need:
            raise ValueError(f"the cache must be one row of at least {need} positions, got {tuple(cache.k.shape[1:3])}")
        super().__init__(model, k + 1, _SeqKV(cache), eos_token_ids, pad_token_id, use_graph)
        dev = model.device
        i32 = dict(dtype=torch.int32, device=dev)
        self.k, self.ngram, self.prompt_len, self.max_new = k, n, S, N
        self.seq = torch.zeros(self.max_len + 1, dtype=torch.int64, device=dev)       # the one sequence
        self.cur_len = torch.zeros(1, **i32)
        self.n_new = torch.zeros(1, **i32)
        self.step_idx = torch.zeros(1, **i32)
        self.done = torch.zeros(1, **i32)
        self.n_draft = torch.zeros(1, **i32)
        self.accepted = torch.zeros(N, **i32)
        self.pen_len = torch.zeros(k + 1, **i32)
        self.idx = torch.zeros(k + 1, **i32)
        self.pick = torch.zeros(k + 1, dtype=torch.int64, device=dev)
        self.temperature, self.top_k = float(temperature or 0.0), int(top_k or 0)
        self.top_p = 1.0 if top_p is None else float(top_p)
        if not 0.0 <= self.top_p <= 1.0:
            raise ValueError(f"top_p must be in [0, 1], got {top_p}")
        self.penalty = float(repetition_penalty or 1.0)
        self.u = None
        if self.temperature > 0:
            # the uniforms DecodeEngine draws for this call (one per new token), padded for the rows past the budget: row i of a
            # step reads u[n_new + i] through uvx_sample's (step, row) indexing at a row stride of 1
            u = torch.rand(int(uniforms or S + N + 1), 1, device=dev, dtype=torch.float32, generator=generator)
            self.u = torch.cat([u, torch.zeros(k + 1, 1, device=dev, dtype=torch.float32)])
        self.scratch = torch.empty(k + 1, self.max_len + 1, dtype=torch.float32, device=dev) if self.penalty != 1.0 else None
        V = model.language_model.lm_head.weight.shape[0]
        self.scores = torch.empty(N, 1, V, dtype=torch.float32, device=dev) if output_scores else None
        self.raw_logits = torch.empty(N, 1, V, dtype=torch.float32, device=dev) if output_logits else None
        self.constraints = None if constraints is None else constraints.device_tables(dev)
        self.cutoffs = tuple(float(v) for v in cutoffs) if ops.cutoffs_on(cutoffs) else None
        self.stop = None if stop is None else stop.device_table(dev)
        self.stop_hit = torch.zeros(k + 1, **i32) if stop is not None else None

    def begin(self, input_ids: torch.Tensor, first_logits: torch.Tensor) -> None:
        """After the prompt input_ids [1, S] has been prefilled into the cache: seeds the sequence and the counters and picks the
        first new token from ``first_logits`` [1, V] fp32 (one row, no drafts)."""
        S = self.prompt_len
        if tuple(input_ids.shape) != (1, S):
            raise ValueError(f"input_ids must be [1, {S}], got {tuple(input_ids.shape)}")
        self.seq[:S].copy_(input_ids[0])
        self.cur_len.fill_(S)
        for t in (self.n_new, self.step_idx, self.done, self.n_draft, self.accepted, self.idx):
            t.zero_()
        self.pen_len.fill_(S)
        self._pick(first_logits.contiguous(), log=False)

    def _pick(self, logits: torch.Tensor, log: bool = True) -> None:
        """logits [R, V] fp32 of rows 0..R-1 (R = 1: the first token) -> picks, then the accepted tokens and the counters."""
        R = logits.shape[0]
        self.logits = logits
        idx = self.idx[:R]
        rec = (self.temperature, self.top_k, self.top_p, idx)
        scores = None if self.scores is None else self.scores.view(self.max_new, -1)
        raw = None if self.raw_logits is None else self.raw_logits.view(self.max_new, -1)
        raw_first = raw is not None and (self.penalty != 1.0 or self.constraints is not None)
        if raw_first:       # the constraints and the penalty rewrite the logits in place: take the raw copy before them
            ops.record_scores_rows(logits, *rec, raw=raw)
        if self.constraints is not None:
            ops.logits_constraints_rows_(logits, self.seq.view(1, -1).expand(R, -1), self.pen_len[:R], self.constraints)
        if self.penalty != 1.0:
            ops.repetition_penalty_rows_(logits, self.seq.view(1, -1).expand(R, -1), self.pen_len[:R], self.penalty,
                                         self.scratch[:R])
        if scores is not None or (raw is not None and not raw_first):
            ops.record_scores_rows(logits, *rec, scores=scores, raw=None if raw_first else raw, cutoffs=self.cutoffs)
        pick = self.pick[:R]
        if self.temperature > 0:
            ops.sample(logits, self.temperature, self.top_k, self.u, self.n_new, out=pick, top_p=self.top_p, cutoffs=self.cutoffs)
        else:
            ops.argmax(logits, out=pick)
        hit = None
        if self.stop is not None:
            hit = ops.stop_strings_rows(pick, self.seq.view(1, -1).expand(R, -1), self.pen_len[:R], self.stop, self.stop_hit[:R])
        ops.lookup_accept(pick, self.token.view(-1)[:R], self.n_draft, self.eos, self.seq, self.cur_len, self.n_new, self.max_new,
                          self.done, self.step_idx if log else None, self.accepted if log else None, hit=hit)

    def _step(self):
        ops.lookup_draft(self.seq, self.cur_len, self.n_new, self.max_new, self.k, self.ngram, self.eos, self.done,
                         self.token.view(-1), self.n_draft, self.pos, self.lens, self.rope_pos, self.pen_len, self.idx)
        self._pick(self._forward())

    def _state(self):
        return [self.pos, self.lens, self.rope_pos, self.token, self.cur_len, self.n_new, self.step_idx, self.done, self.n_draft,
                self.pen_len, self.idx, self.pick]


class BeamDecodeEngine(DecodeEngine):
    """Beam search over ``batch`` prompts with ``num_beams`` beams each (row b * num_beams + j), as
    hf:generation/utils.py ``_beam_search``: the forward of ``DecodeEngine._step`` runs unchanged over the batch * num_beams
    rows, and the pick becomes log_softmax -> token constraints (if any) -> repetition penalty on the log-probs -> top-K
    continuations per prompt -> running beams / finished pool / early-stop heuristic -> KV cache rows gathered by parent beam,
    all on the device, so a
    step is still one CUDA graph replay.  ``all_done`` is HF's loop condition (negated); ``logprobs`` holds the last step's
    processed log-probs [batch * num_beams, V] and ``logits`` the raw ones.  The cache must have batch * num_beams rows with
    each prompt prefilled into row b * num_beams (``begin`` broadcasts it to the other beams)."""

    def __init__(self, model: UltravoxModel, batch: int, num_beams: int, max_len: int, max_new_tokens: int, use_graph: bool = True,
                 cache=None, eos_token_ids=None, length_penalty: float = 1.0, early_stopping=False, repetition_penalty: float = 1.0,
                 constraints=None, stop=None):
        """``stop`` (``stop_strings.StopStrings``): every step checks each candidate's sequence (its parent's running sequence
        plus its token, ``uvx_stop_strings_beam``) and a hit finishes the candidate as an EOS id does (``uvx_beam_update_stop``),
        as HF's ``_beam_search`` does with ``StopStringCriteria``.  None: the step is unchanged."""
        nb = int(num_beams)
        if not 1 <= nb <= ops.BEAM_MAX:
            raise ValueError(f"num_beams must be in [1, {ops.BEAM_MAX}], got {num_beams}")
        if early_stopping not in (False, True, "never"):
            raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
        eos_list = [eos_token_ids] if isinstance(eos_token_ids, int) else list(eos_token_ids or [])
        super().__init__(model, batch * nb, max_len, use_graph=use_graph, cache=cache, eos_token_ids=eos_list,
                         repetition_penalty=repetition_penalty, constraints=constraints)
        dev = model.device
        R = batch * nb
        self.prompts, self.nb = batch, nb
        self.K = max(2, 1 + len(eos_list)) * nb                 # HF's beams_to_keep
        if self.K > ops.BEAM_MAX_K:
            raise ValueError(f"max(2, 1 + {len(eos_list)} EOS ids) * {nb} beams = {self.K} candidates; at most {ops.BEAM_MAX_K}")
        self.max_new = int(max_new_tokens)
        if not 1 <= self.max_new <= self.max_len:
            raise ValueError(f"max_new_tokens must be in [1, {self.max_len}], got {max_new_tokens}")
        self.length_penalty = float(length_penalty)
        self.es = 2 if early_stopping == "never" else int(early_stopping is True)
        # divisor of a hypothesis of n generated tokens: HF divides by the Python float n ** length_penalty, which torch rounds
        # once to fp32 (entry 0 is never read)
        self.len_div = torch.tensor([1.0] + [float(n) ** self.length_penalty for n in range(1, self.max_len + 2)],
                                    dtype=torch.float32, device=dev)
        self.V = model.language_model.lm_head.weight.shape[0]
        i32 = dict(dtype=torch.int32, device=dev)
        self.run_score = torch.zeros(R, dtype=torch.float32, device=dev)
        self.pool_seq = torch.zeros_like(self.seq)
        self.pool_score = torch.full((R,), -1e9, dtype=torch.float32, device=dev)
        self.pool_len = torch.zeros(R, **i32)
        self.pool_fin = torch.zeros(R, **i32)
        self.parent = torch.arange(R, **i32)
        self.heur = torch.ones(batch, **i32)
        self.flags = torch.zeros(batch, **i32)
        self.ticket = torch.zeros(1, **i32)
        self.n_pos = torch.zeros(1, **i32)
        self.logprobs = torch.empty(R, self.V, dtype=torch.float32, device=dev)
        self.row_buf = (torch.empty(R * self.K, dtype=torch.float32, device=dev), torch.empty(R * self.K, dtype=torch.int64, device=dev))
        self.cand = (torch.empty(batch, self.K, dtype=torch.float32, device=dev), torch.empty(batch, self.K, dtype=torch.int64, device=dev))
        self._beam = dict(run_score=self.run_score, run_seq=self.seq, pool_seq=self.pool_seq, pool_score=self.pool_score,
                          pool_len=self.pool_len, pool_fin=self.pool_fin, parent=self.parent, tok=self.token.view(-1),
                          heur=self.heur, flags=self.flags, ticket=self.ticket)
        self._counters = dict(cur_len=self.cur_len, step_idx=self.step_idx, done=self.all_done)
        self.beam_stop = None if stop is None else stop.device_table(dev)
        self.beam_hit = torch.zeros(batch * self.K, **i32) if stop is not None else None

    def begin(self, input_ids: torch.Tensor, first_logits: torch.Tensor, kv_start: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``input_ids`` [batch, S] prompts prefilled into cache rows b * num_beams, ``first_logits`` [batch, V] their last
        positions: broadcasts both to the beams and runs the first beam step (HF's running scores [0, -1e9, ...] and a pool of
        -1e9 entries).  Returns the device token tensor [batch * num_beams]."""
        B, S = input_ids.shape
        nb = self.nb
        rows = input_ids.repeat_interleave(nb, 0)
        self.pool_seq[:, :S].copy_(rows)
        self.run_score.view(B, nb).fill_(-1e9)
        self.run_score.view(B, nb)[:, 0] = 0.0
        self.pool_score.fill_(-1e9)
        self.pool_len.zero_()
        self.pool_fin.zero_()
        self.heur.fill_(1)
        self.flags.zero_()
        self.ticket.zero_()
        self.parent.copy_(torch.arange(B * nb, dtype=torch.int32, device=self.parent.device) // nb * nb)
        self.n_pos.fill_(S)
        ops.kv_reorder_(self.cache.k, self.cache.v, self.parent, self.n_pos, nb)
        kv = kv_start.repeat_interleave(nb) if kv_start is not None else None
        return super().begin(rows, first_logits.repeat_interleave(nb, 0), kv)

    def prefill(self, inputs_embeds: torch.Tensor) -> torch.Tensor:
        """Prefills the batch prompts [batch, S, D] once each into rows b * num_beams, then ``begin`` (prompt ids taken as 0)."""
        m = self.model
        B, S, _ = inputs_embeds.shape
        L, _, smax, hkv, d = self.cache.k.shape
        view = type(self.cache)(self.cache.k.view(L, B, self.nb * smax, hkv, d), self.cache.v.view(L, B, self.nb * smax, hkv, d))
        hid = m.llama_hidden(inputs_embeds, view)
        logits = ops.lm_head(hid[:, -1, :], m.language_model.lm_head.weight)
        ids = torch.zeros(B, S, dtype=torch.int64, device=logits.device)
        return self.begin(ids, logits).clone()

    def _pick(self, logits: torch.Tensor):
        """logits [batch * nb, V] fp32 -> the next running beams in ``token`` / ``seq``, the pool, the cache rows reordered."""
        self.logits = logits
        lp = ops.log_softmax(logits, out=self.logprobs)
        if self.constraints is not None:        # HF applies the processors to each running beam's log-probs
            ops.logits_constraints_(lp, self.seq, self.cur_len, self.constraints)
        if self.penalty != 1.0:
            ops.repetition_penalty_(lp, self.seq, self.cur_len, self.penalty, self.scratch)
        s, i = ops.beam_select(lp, self.run_score, self.nb, self.K, scratch=self.row_buf, out=self.cand)
        hit = None
        if self.beam_stop is not None:      # before the update rewrites the running sequences
            hit = ops.stop_strings_beam(i, self.V, self.nb, self.seq, self.cur_len, self.beam_stop, self.beam_hit)
        ops.beam_update(s, i, self.V, self.nb, self.eos, self.max_new, self.len_div, self.es, self.length_penalty > 0.0, self._beam,
                        self._counters, (self.pos, self.lens, self.rope_pos), hit=hit)
        # the update advanced pos to the slot of the token fed next: the cache holds positions [0, pos)
        ops.kv_reorder_(self.cache.k, self.cache.v, self.parent, self.pos, self.nb)

    def _step_warm(self):
        # the warm-up and capture steps run with the search marked done, so they leave the beams, the pool and the cache rows
        # alone (the update then only sets the identity parent map)
        prev = self.all_done.clone()
        self.all_done.fill_(1)
        super()._step_warm()
        self.all_done.copy_(prev)

    def result(self, prompt_len: int, num_return_sequences: int, fill_value: int):
        """(sequences [batch * n, prompt_len + longest], scores [batch * n]) of the n best finished hypotheses per prompt, cropped
        to the longest of them and filled with ``fill_value`` past each one's end (HF's output)."""
        dev = self.pool_seq.device
        idx = (torch.arange(self.prompts, device=dev)[:, None] * self.nb
               + torch.arange(num_return_sequences, device=dev)[None, :]).reshape(-1)
        lens = self.pool_len[idx].to(torch.int64)
        width = prompt_len + int(lens.max())
        seq = self.pool_seq[idx, :width]
        keep = torch.arange(width, device=dev)[None, :] < (prompt_len + lens)[:, None]
        return torch.where(keep, seq, torch.full_like(seq, fill_value)), self.pool_score[idx].clone()


class SlotDecodeEngine(_Decoder):
    """Continuous batching: ``slots`` decode rows that each carry their own request.  The step is the shared step loop over
    all rows followed by three per-row kernels (``uvx_repetition_penalty_slots``, ``uvx_sample_slots_cutoffs``, ``uvx_slot_finish``);
    every per-request value - positions, lengths, budget, active / done flags, sampling settings, the uniforms - lives in a
    device array [slots], so the step is captured once per engine and admission and retirement only write into those arrays
    between replays.

    An idle slot holds ``pos = 0``, ``lens = 1`` and the pad token: it writes its own K / V at position 0 and attends to that
    alone, so it stays finite whatever its cache row held.  A finished slot is frozen (no sequence writes, no position bumps)
    until ``retire``.  ``n_open[0]`` counts the active slots still decoding after each step.

    A prompt of more than ``PREFILL_ROWS`` rows is prefilled in chunks instead of one B = 1 prefill that would stall every
    other slot: ``admit`` runs the audio side and the splice and parks the slot as prefilling, and each following ``step``
    is a mixed step - a second graph, captured on the first such admission - whose GEMMs carry the ``slots`` decode rows
    followed by ``chunk = PREFILL_ROWS - slots`` prompt rows (so they stay on the weight-bound tiling).  The chunk rows take
    RoPE + the KV append through a per-row map and attend to the prefilling slot's cache row through the device-indexed
    attention; the LM head runs over the decode rows plus the chunk's last valid row.  While it prefills, the slot's own
    decode row writes nothing to the cache and picks nothing; after the last chunk its first token is picked from that row's
    logits and the slot becomes active.  One slot prefills at a time.  A chunk's rows are independent of the decode rows
    (every kernel is row-independent at the fixed row count), so a chunked request gets the same bits whatever else is
    decoding; the decode rows of a mixed step run at 256 rows instead of ``slots`` and are not bit-identical to a plain step.

    ``max_logprobs`` (0..20) > 0 adds per-token log-probabilities: every pick (the step's, the mixed step's and the one-row
    admission pick) copies the raw logits rows aside before the penalty and runs ``uvx_token_logprobs`` after the sampler, which
    writes each row's chosen-token log-prob and its ``n_top[b]`` most likely alternatives at index ``n_new[b]`` of
    ``lp_token`` [slots, max_len + 1] / ``lp_ids``, ``lp_top`` [slots, max_len + 1, max_logprobs].  A request asks with
    ``admit(..., logprobs=k)``.  With 0 (the default) nothing is allocated and the step is unchanged.

    ``prompt_lookup_num_tokens`` = K (1..31, with slots * (K + 1) <= ``PREFILL_ROWS``) adds prompt lookup decoding: a request
    admitted with ``lookup=(k, n)``, 1 <= k <= K, drafts up to k tokens per step from its own earlier n-grams
    (``uvx_lookup_draft``'s rule, capped so it never passes its budget) and keeps the picks that agree plus one, so its tokens
    are those of plain slot decoding and a step yields 1 to k + 1 of them.  While no chunked prompt is in flight and some
    active slot has k > 0, ``step`` replays a third graph, the lookup step (captured on first use), over R = slots * (K + 1)
    rows, slot s owning rows s * (K + 1) + i: ``uvx_lookup_draft_slots`` lays out the rows, the forward runs them with the
    row-mapped RoPE + append and attention (a slot's rows all read its cache row; rows past its drafts write nothing), the
    row-mapped penalty / sampler / log-prob kernels pick each row as plain decoding would pick that position, and
    ``uvx_lookup_accept_slots`` appends the accepted tokens and leaves every counter as ``uvx_slot_finish`` would.  So the
    plain and the mixed step can follow any lookup step.  ``accepted`` [slots] int32 counts each request's accepted drafts.
    The linears of a lookup step run at R rows: a request's bits are those of a plain engine of R slots (the decode-form GEMM
    keeps rows independent at a fixed row count).  None (the default) allocates and captures nothing.

    ``max_constraint_tokens`` = N (None, the default: off) adds the token constraints of ``generate()``
    (``constraints.LogitsConstraints``) per slot: settings ``ck_cfg`` [slots, 4] and a table of N ids per slot (``ck_ids``,
    ``ck_end``, ``ck_bias``, ``ck_kind`` [slots, max(N, 1)]), written by ``admit(..., constraints=...)`` between replays and
    cleared when the slot goes idle.  Every pick (the plain, mixed and lookup steps' and the admission pick) then runs
    ``uvx_logits_constraints_slots`` (``_rows_map`` in the lookup step) after the raw copy for log-probs and before the penalty.
    None allocates nothing and launches nothing: the steps are unchanged.

    ``max_stop_table`` = N (None, the default: off) adds ``generate()``'s stop strings per slot: ``stop_tab`` [slots, N] int32
    holds each slot's packed table (``stop_strings.StopStrings``, written by ``admit(..., stop=...)``; a slot without stop
    strings has an all-zero header).  Every pick then runs ``uvx_stop_strings_slots`` after the sampler and finishes with
    ``uvx_slot_finish_stop`` (the lookup step: ``uvx_stop_strings_rows_map`` and ``uvx_lookup_accept_slots_stop``), so a slot
    whose token ends a stop string finishes as on an EOS id.  None allocates and launches nothing."""

    def __init__(self, model: UltravoxModel, slots: int, max_len: int, eos_token_ids=None, pad_token_id: int = 0,
                 use_graph: bool = True, cache=None, max_logprobs: int = 0, prompt_lookup_num_tokens: Optional[int] = None,
                 max_constraint_tokens: Optional[int] = None, max_stop_table: Optional[int] = None):
        check_lookup_k(int(slots), prompt_lookup_num_tokens)      # before the cache is allocated
        kv = _RowKV(cache if cache is not None else model.new_cache(slots, max_len))
        self._setup(model, int(slots), kv, eos_token_ids, pad_token_id, use_graph, max_logprobs, prompt_lookup_num_tokens,
                    max_constraint_tokens, max_stop_table)

    def _setup(self, model: UltravoxModel, slots: int, kv, eos_token_ids, pad_token_id: int, use_graph: bool, max_logprobs: int = 0,
               lookup_k: Optional[int] = None, max_constraint_tokens: Optional[int] = None, max_stop_table: Optional[int] = None):
        if isinstance(max_logprobs, bool) or not isinstance(max_logprobs, numbers.Integral) or \
                not 0 <= max_logprobs <= ops.LOGPROBS_MAX:
            raise ValueError(f"max_logprobs must be an integer in [0, {ops.LOGPROBS_MAX}], got {max_logprobs!r}")
        self.max_constraint_tokens = check_constraint_tokens(max_constraint_tokens)
        self.max_stop_table = check_stop_table(max_stop_table)
        self.K = check_lookup_k(slots, lookup_k)
        self.max_logprobs = int(max_logprobs)
        self.slots = slots
        self.chunk = PREFILL_ROWS - slots
        # mixed-step rows: [0, slots) decode rows, [slots, slots + chunk) prompt-chunk rows.  The host writes the chunk part of
        # the per-row position arrays (_mpos, _mrope), the cache-row map, the attention scalars (cache row, past, past + valid)
        # and the LM-head row list between replays.
        super().__init__(model, slots, kv, eos_token_ids, pad_token_id, use_graph, extra=max(self.chunk, 0))
        dev = model.device
        i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
        self.cur_len = torch.zeros(slots, **i32)
        self.n_new = torch.zeros(slots, **i32)
        self.max_new = torch.ones(slots, **i32)
        self.active = torch.zeros(slots, **i32)
        self.temps = torch.zeros(slots, **f32)
        self.top_ks = torch.zeros(slots, **i32)
        self.top_ps = torch.ones(slots, **f32)
        self.cutoffs = torch.tensor([ops.CUTOFFS_OFF] * slots, **f32)   # per slot (min_p, typical_p, epsilon, eta), off = (0, 1, 0, 0)
        self.penalties = torch.ones(slots, **f32)
        self.u = torch.zeros(slots, self.max_len + 1, **f32)
        self.scratch = torch.empty(slots, self.max_len + 1, **f32)
        self.n_open = torch.zeros(1, **i32)
        self._admit_open = torch.zeros(1, **i32)     # the count an admission's one-row pick writes (not the step's)
        self._mrow = torch.arange(self._mpos.shape[0], **i32)
        self._mscal = torch.zeros(3, **i32)
        self._head_rows = torch.arange(slots + 1, **i32)
        self._mixed_in = None
        self._mixed_graph = None
        self._chunk_logits = None
        self._prefill: Optional[dict] = None
        self.launches_per_mixed_step = 0
        if self.max_logprobs:
            V = model.language_model.lm_head.weight.shape[0]
            self.n_top = torch.full((slots,), -1, **i32)                # per slot: alternatives asked for, -1 = none
            self._raw = torch.empty(slots, V, **f32)                    # the picked rows' logits before the penalty
            self.lp_token = torch.zeros(slots, self.max_len + 1, **f32)
            self.lp_ids = torch.zeros(slots, self.max_len + 1, self.max_logprobs, dtype=torch.int64, device=dev)
            self.lp_top = torch.zeros(slots, self.max_len + 1, self.max_logprobs, **f32)
        self._lookup_graph = None
        self.launches_per_lookup_step = 0
        # host copy of lk_k: the host picks the graph of each step from it without a sync.  It is cleared at retirement, so a
        # slot that has finished on the device but is not retired yet (up to the scheduler's sync_every steps) keeps the lookup
        # step running even when no open slot drafts: the same tokens, at the R-row step's cost for that window
        self._slot_k = [0] * slots
        if self.K:
            R = slots * (self.K + 1)
            self.lk_k = torch.zeros(slots, **i32)      # per slot: drafts per step (0: none) and n-gram size
            self.lk_n = torch.full((slots,), 2, **i32)
            self.accepted = torch.zeros(slots, **i32)
            self.n_draft = torch.zeros(slots, **i32)
            # the prefilling mask of uvx_lookup_draft_slots: set while a slot's prompt is chunked, but step() only replays the
            # lookup step when no prompt is in flight, so it is all zero whenever the lookup step runs
            self._pf = torch.zeros(slots, **i32)
            self._lk_tok = torch.zeros(R, 1, dtype=torch.int64, device=dev)
            self._lk_pick = torch.zeros(R, dtype=torch.int64, device=dev)
            self._lk_pos, self._lk_lens, self._lk_rope, self._lk_pen, self._lk_idx, self._lk_slot, self._lk_wrow = (
                torch.zeros(R, **i32) for _ in range(7))
            self._lk_scratch = torch.empty(R, self.max_len + 1, **f32)
            if self.max_logprobs:
                self._lk_raw = torch.empty(R, model.language_model.lm_head.weight.shape[0], **f32)
        self.ck = None
        if self.max_constraint_tokens is not None:
            T = max(self.max_constraint_tokens, 1)
            self.ck_cfg = torch.zeros(slots, 4, **i32)
            self.ck_ids = torch.zeros(slots, T, dtype=torch.int64, device=dev)
            self.ck_end, self.ck_kind = torch.zeros(slots, T, **i32), torch.zeros(slots, T, **i32)
            self.ck_bias = torch.zeros(slots, T, **f32)
            self.ck = (self.ck_cfg, self.ck_ids, self.ck_end, self.ck_bias, self.ck_kind)
        self.stop_tab = None
        if self.max_stop_table is not None:
            self.stop_tab = torch.zeros(slots, self.max_stop_table, **i32)
            self.stop_hit = torch.zeros(slots, **i32)
            if self.K:
                self._lk_hit = torch.zeros(slots * (self.K + 1), **i32)
        self.busy = [False] * slots
        for j in range(slots):
            self._idle(j)
        if use_graph:
            self._step_warm()

    def _idle(self, j: int) -> None:
        self.active[j] = 0
        self.done[j] = 0
        self.cur_len[j] = 0
        self.n_new[j] = 0
        self.pos[j] = 0
        self.lens[j] = 1
        self.rope_pos[j] = 0
        self.token[j] = self.pad_id
        self.busy[j] = False
        if self.max_logprobs:
            self.n_top[j] = -1
        if self.K:
            self.lk_k[j] = 0
            self._slot_k[j] = 0
        if self.ck is not None:
            self.ck_cfg[j] = 0          # no n-gram size and no entries: the kernel leaves the row alone
        if self.stop_tab is not None:
            self.stop_tab[j, :ops.STOP_HEADER] = 0      # no stop strings: no hit
        self.kv.release(j)

    def _state(self):
        lk = [self.accepted, self.n_draft] if self.K else []
        return [self.pos, self.lens, self.rope_pos, self.token, self.cur_len, self.n_new, self.done, self.n_open] + lk

    def _lookup_step(self):
        """The lookup step: drafts and row layout, the forward over R rows, the row-mapped pick, the accept."""
        R = self._lk_tok.shape[0]
        ops.lookup_draft_slots(self.seq, self.token.view(-1), self.cur_len, self.n_new, self.max_new, self.lk_k, self.lk_n, self.done,
                               self.active, self._pf, self.pos, self.lens, self.rope_pos, self.K, self.eos, self._lk_tok.view(-1),
                               self.n_draft, self._lk_pos, self._lk_lens, self._lk_rope, self._lk_pen, self._lk_idx, self._lk_slot,
                               self._lk_wrow)
        logits = self._forward(lookup=True)
        self.logits = logits
        rows = (self._lk_slot, self._lk_idx)
        if self.max_logprobs:
            self._lk_raw.copy_(logits)
        if self.ck is not None:
            ops.logits_constraints_rows_map_(logits, self.seq, self.active, self._lk_slot, self._lk_pen, self._lk_idx, self.ck)
        ops.repetition_penalty_rows_map_(logits, self.seq, self.penalties, self.active, self._lk_slot, self._lk_pen, self._lk_idx,
                                         self._lk_scratch[:R])
        ops.sample_rows_cutoffs(logits, self.temps, self.top_ks, self.top_ps, self.cutoffs, self.u, self.active, *rows, self._lk_pick)
        if self.max_logprobs:       # at n_new + i, before the accept advances n_new; rows past the drafts (idx -1) record nothing
            ops.token_logprobs_rows(self._lk_raw, self._lk_pick, self.n_top, *rows, self.lp_token, self.lp_ids, self.lp_top)
        hit = None
        if self.stop_tab is not None:
            hit = ops.stop_strings_rows_map(self._lk_pick, self.seq, self.active, self._lk_slot, self._lk_pen, self._lk_idx,
                                            self.stop_tab, self._lk_hit)
        ops.lookup_accept_slots(self._lk_pick, self._lk_tok.view(-1), self.n_draft, self.K, self.eos, self.seq, self.token.view(-1),
                                self.done, self.cur_len, self.n_new, self.max_new, self.active, self.pos, self.lens, self.rope_pos,
                                self.accepted, self.n_open, hit=hit)

    def _pick_rows(self, logits: torch.Tensor, r: slice, n_open: torch.Tensor) -> None:
        tok = self.token.view(-1)[r]
        if self.max_logprobs:
            raw = self._raw[r]
            raw.copy_(logits)
        if self.ck is not None:
            ops.logits_constraints_slots_(logits, self.seq[r], self.cur_len[r], self.active[r], tuple(t[r] for t in self.ck))
        ops.repetition_penalty_slots_(logits, self.seq[r], self.cur_len[r], self.penalties[r], self.active[r], self.scratch[r])
        ops.sample_slots_cutoffs(logits, self.temps[r], self.top_ks[r], self.top_ps[r], self.cutoffs[r], self.u[r], self.n_new[r],
                                 self.active[r], tok)
        if self.max_logprobs:       # at n_new, before the finish kernel advances it
            ops.token_logprobs(raw, tok, self.n_top[r], self.n_new[r], self.lp_token[r], self.lp_ids[r], self.lp_top[r])
        hit = None
        if self.stop_tab is not None:
            hit = ops.stop_strings_slots(tok, self.seq[r], self.cur_len[r], self.active[r], self.stop_tab[r], self.stop_hit[r])
        ops.slot_finish(tok, self.done[r], self.eos, self.seq[r], self.cur_len[r], self.n_new[r], self.max_new[r], self.active[r],
                        self.pos[r], self.lens[r], self.rope_pos[r], n_open, hit=hit)

    def _pick(self, logits: torch.Tensor):
        self.logits = logits
        self._pick_rows(logits, slice(None), self.n_open)

    def _mixed_step(self):
        logits = self._forward(self._mixed_in, self._head_rows)
        self._chunk_logits = logits[self.B:]
        self._pick(logits[:self.B])

    @property
    def prefilling(self) -> Optional[int]:
        """The slot whose prompt is being prefilled in chunks, or None."""
        return None if self._prefill is None else self._prefill["slot"]

    def step(self) -> torch.Tensor:
        """A plain decode step, or a mixed step while a chunked prompt is pending (whose last chunk activates its slot)."""
        pf = self._prefill
        if pf is None and any(self._slot_k):
            if not self.use_graph:
                self._lookup_step()
            else:
                if self._lookup_graph is None:
                    self._lookup_graph, self.launches_per_lookup_step = self._capture(self._lookup_step)
                self._lookup_graph.replay()
            return self.token
        if pf is None:
            return super().step()
        j, S, a, C, B = pf["slot"], pf["S"], pf["done"], self.chunk, self.slots
        n = min(C, S - a)
        self._mixed_in[B:B + n].copy_(pf["embeds"][a:a + n])
        # cache row per chunk row (-1: padding, no write) | its position (padding: 0, inside the RoPE tables) | attention scalars
        # | the LM head's chunk row; one pinned buffer per step (the host allocator keeps it until its copies have run)
        hv = torch.tensor([j] * n + [-1] * (C - n) + list(range(a, a + n)) + [0] * (C - n) + [j, a, a + n, B + n - 1],
                          dtype=torch.int32).pin_memory()
        self._mrow[B:].copy_(hv[:C], non_blocking=True)
        self._mpos[B:].copy_(hv[C:2 * C], non_blocking=True)
        self._mrope[B:].copy_(hv[C:2 * C], non_blocking=True)
        self._mscal.copy_(hv[2 * C:2 * C + 3], non_blocking=True)
        self._head_rows[B:].copy_(hv[2 * C + 3:], non_blocking=True)
        if self.use_graph:
            if self._mixed_graph is None:
                self._mixed_graph, self.launches_per_mixed_step = self._capture(self._mixed_step)
            self._mixed_graph.replay()
        else:
            self._mixed_step()
        pf["done"] = a + n
        if a + n == S:
            self._prefill = None
            self.active[j] = 1
            if self.K:
                self._pf[j] = 0
            if self.max_logprobs:
                self.n_top[j] = pf["n_top"]
            self._seed(j, S)
            self._mrow[j] = j
            self._pick_rows(self._chunk_logits, slice(j, j + 1), self._admit_open)
        return self.token

    def admit(self, slot: int, input_ids: torch.Tensor, max_new_tokens: int, temperature: float = 0.0, top_k: int = 0,
              top_p: float = 1.0, repetition_penalty: float = 1.0, u: Optional[torch.Tensor] = None, past: int = 0,
              pages=None, logprobs: Optional[int] = None, lookup: Optional[tuple] = None, constraints=None, cutoffs=None,
              stop=None, **features) -> torch.Tensor:
        """Prefills one request (``input_ids`` [1, S] plus the processor's audio features, passed to ``model.forward``) at B = 1
        into cache row ``slot``, sets the slot's state and picks its first token from the prefill logits with the slot kernels.
        ``temperature <= 0`` is greedy; a sampled request reads ``u`` (its uniforms, one per step, as ``generate()`` draws them
        for a batch of one).  Returns the device token tensor [slots] (no sync).

        A prompt of more than ``PREFILL_ROWS`` rows is only embedded here (audio encoder, projector, splice); its LLM prefill
        runs in chunks inside the following steps, and its first token is picked after the last one (``prefilling`` is the
        slot until then).  Only one slot prefills at a time.

        ``past`` > 0 (engines that keep a conversation's KV cache, ``PagedSlotDecodeEngine``): the slot's cache already holds the
        first ``past`` positions of ``input_ids``, so only the suffix is prefilled, as ``generate(past_key_values=...)`` does; the
        chunked form then starts at ``past`` and is taken when the suffix has more than ``PREFILL_ROWS`` rows.  ``pages``
        (``PagedSlotDecodeEngine`` only): the request's page ids for positions 0, 64, 128, ...; they must cover
        S + max_new_tokens positions, and the first ceil(past / 64) of them hold the conversation's first ``past`` positions.

        ``logprobs`` (engines with ``max_logprobs`` > 0): None records nothing, 0 the chosen tokens' log-probs, 1..max_logprobs
        also that many alternatives per token (``token_logprobs_of``).

        ``lookup`` (engines with ``prompt_lookup_num_tokens`` = K): (k, n) with 0 <= k <= K drafts per step from n-grams of up
        to n >= 1 tokens; None or k = 0 drafts nothing.

        ``constraints`` (engines with ``max_constraint_tokens`` = N): the request's ``constraints.LogitsConstraints`` (built
        with its whole prompt's length), at most N ids; None: no constraints.

        ``cutoffs``: the request's (min_p, typical_p, epsilon, eta), as ``generate()`` checks them, off = (0, 1, 0, 0) (None:
        all off).  Every pick reads them from ``cutoffs`` [slots, 4] (``uvx_sample_slots_cutoffs`` / ``_rows_cutoffs``).

        ``stop`` (engines with ``max_stop_table`` = N): the request's ``stop_strings.StopStrings``, a table of at most N words;
        None: no stop strings."""
        n_top = self.check_logprobs(logprobs)
        ck_rows = self.check_constraints(constraints)
        self.check_stop(stop)
        lk, ln = (0, 2) if lookup is None else (int(lookup[0]), int(lookup[1]))
        if lookup is not None and not self.K:
            raise ValueError("this engine has no prompt lookup: create it with prompt_lookup_num_tokens = K")
        if not 0 <= lk <= self.K or ln < 1:
            raise ValueError(f"lookup = {lookup!r}: need 0 <= k <= {self.K} and n >= 1")
        j = int(slot)
        if not 0 <= j < self.slots:
            raise ValueError(f"slot {slot} out of range [0, {self.slots})")
        if self.busy[j]:
            raise ValueError(f"slot {j} is busy; retire it first")
        if input_ids.dim() != 2 or input_ids.shape[0] != 1:
            raise ValueError(f"admit() takes one request: input_ids [1, S], got {tuple(input_ids.shape)}")
        S, n, P = int(input_ids.shape[1]), int(max_new_tokens), int(past)
        if n < 1 or S < 1 or S + n > self.max_len:
            raise ValueError(f"a prompt of {S} tokens plus max_new_tokens={n} does not fit a slot of {self.max_len} positions")
        if not 0 <= P < S:
            raise ValueError(f"past = {P}: the prompt of {S} tokens must extend the cached prefix")
        if P and not self.kv.keeps_kv:
            raise ValueError("this engine keeps no KV cache between requests (past must be 0)")
        if temperature > 0 and (u is None or u.numel() < S + n):
            raise ValueError(f"a sampled request needs at least {S + n} uniforms")
        chunked = S - P > PREFILL_ROWS
        if chunked and self.chunk < 1:
            raise ValueError(f"a prompt of {S} > {PREFILL_ROWS} rows is prefilled in chunks of {PREFILL_ROWS} - slots rows; "
                             f"{self.slots} slots leave none")
        if chunked and self._prefill is not None:
            raise ValueError(f"slot {self._prefill['slot']} is still prefilling; one long prompt at a time")
        self.kv.install(j, S, n, pages)
        dev = self.pos.device
        input_ids = input_ids.to(dev)
        if chunked:
            embeds = self.model.prompt_embeds(input_ids, **features).view(S, -1)
            if self._mixed_in is None:
                self._mixed_in = torch.zeros(self.slots + self.chunk, embeds.shape[1], dtype=embeds.dtype, device=dev)
            self._prefill = dict(slot=j, S=S, done=P, embeds=embeds, n_top=n_top)
            self._mrow[j] = -1          # the slot's idle decode row must not overwrite position 0 of the prompt
            if self.K:
                self._pf[j] = 1
        else:
            logits = self.kv.prefill(self.model, j, input_ids, P, features)
        self.seq[j, :S].copy_(input_ids[0])
        self.cur_len[j] = S
        self.n_new[j] = 0
        self.max_new[j] = n
        self.done[j] = 0
        if not chunked:
            self.active[j] = 1
            self._seed(j, S)
        self.temps[j] = float(temperature) if temperature > 0 else 0.0
        self.top_ks[j] = int(top_k or 0)
        self.top_ps[j] = float(top_p)
        self.cutoffs[j] = torch.tensor(ops.CUTOFFS_OFF if cutoffs is None else [float(v) for v in cutoffs])
        self.penalties[j] = float(repetition_penalty or 1.0)
        if u is not None:
            w = min(u.numel(), self.max_len + 1)
            self.u[j, :w].copy_(u.reshape(-1)[:w])
        self.busy[j] = True
        if self.K:
            self.lk_k[j], self.lk_n[j], self.accepted[j] = lk, ln, 0
            self._slot_k[j] = lk
        if self.ck is not None:
            if ck_rows is None:
                self.ck_cfg[j] = 0
            else:
                for t, a in zip(self.ck, ck_rows):
                    t[j].copy_(torch.from_numpy(a))
        if self.stop_tab is not None:
            if stop is None:
                self.stop_tab[j, :ops.STOP_HEADER] = 0
            else:
                self.stop_tab[j, :stop.n_words].copy_(stop.device_table(self.stop_tab.device))     # device to device
        if not chunked:
            if self.max_logprobs:
                self.n_top[j] = n_top
            self._pick_rows(logits, slice(j, j + 1), self._admit_open)
        return self.token.view(-1)

    def check_constraints(self, constraints):
        """A request's constraint tables at this engine's width (None for None); ValueError when the engine has no constraints or
        the request needs more than ``max_constraint_tokens`` ids."""
        if constraints is None:
            return None
        if self.ck is None:
            raise ValueError("this engine has no token constraints: create it with max_constraint_tokens = N")
        if constraints.n_ids > self.max_constraint_tokens:
            raise ValueError(f"the request's constraints need a table of {constraints.n_ids} ids; max_constraint_tokens = "
                             f"{self.max_constraint_tokens}")
        return constraints.tables(self.ck_ids.shape[1])

    def check_stop(self, stop) -> None:
        """ValueError when a request has stop strings (``stop_strings.StopStrings``) and the engine has no stop tables or the
        request's table is longer than ``max_stop_table`` words."""
        if stop is None:
            return
        if self.stop_tab is None:
            raise ValueError("this engine has no stop strings: create it with max_stop_table = N")
        if stop.n_words > self.max_stop_table:
            raise ValueError(f"the request's stop strings need a table of {stop.n_words} int32 words; max_stop_table = "
                             f"{self.max_stop_table}")

    def check_logprobs(self, logprobs) -> int:
        """The slot kernels' n_top of a request's ``logprobs`` argument (None -> -1); ValueError unless it is None or an integer
        in [0, max_logprobs]."""
        if logprobs is None:
            return -1
        if isinstance(logprobs, bool) or not isinstance(logprobs, numbers.Integral):
            raise ValueError(f"logprobs must be None or an integer, got {logprobs!r}")
        if not self.max_logprobs:
            raise ValueError("this engine records no log-probabilities: create it with max_logprobs > 0")
        if not 0 <= logprobs <= self.max_logprobs:
            raise ValueError(f"logprobs must be in [0, max_logprobs = {self.max_logprobs}], got {logprobs}")
        return int(logprobs)

    def token_logprobs_of(self, slot: int, n: int, k: int) -> TokenLogprobs:
        """Copies of slot ``slot``'s log-probs of its first ``n`` new tokens with ``k`` alternatives each (read before
        ``retire``)."""
        j = int(slot)
        return TokenLogprobs(self.lp_token[j, :n].clone(), self.lp_ids[j, :n, :k].clone(), self.lp_top[j, :n, :k].clone())

    def retire(self, slot: int, length: Optional[int] = None) -> torch.Tensor:
        """The slot's sequence [1, prompt + new tokens] (a copy; ``length`` = its ``cur_len`` if the caller already read it, else
        one sync), then the slot goes back to idle."""
        j = int(slot)
        if j == self.prefilling:
            raise ValueError(f"slot {j} is still prefilling")
        n = int(self.cur_len[j]) if length is None else int(length)
        out = self.seq[j:j + 1, :n].clone()
        self._idle(j)
        return out


class PagedSlotDecodeEngine(SlotDecodeEngine):
    """``SlotDecodeEngine`` whose KV cache is a shared pool of ``kv_pages`` 64-position pages (``_PagedKV``) instead of one
    ``[max_len]`` row per slot, so a request's K / V can outlive its slot: a conversation keeps its pages between turns and
    each turn prefills only its new suffix.  Every step computes the same bits as the contiguous engine's.

    ``admit`` takes the request's ``pages``.  A prompt of at most ``PREFILL_ROWS`` new rows is prefilled at B = 1 in the
    one-row scratch ``cache`` ``[L, 1, max_len, Hkv, D]`` and scattered into its pages; longer suffixes go through the mixed
    step from ``past`` on.  Page ownership (which pages a request or a conversation holds) is the caller's bookkeeping
    (``serving.PagePool``).

    ``kv_cache_dtype="fp8_e4m3"`` (with ``kv_scales`` [L, 2], default all 1) keeps the pool in e4m3: half the bytes per page
    (``_PagedKV``).  Every step then computes the bits the bf16 engine would on a pool holding the dequantized values.

    ``host_kv_pages`` > 0 adds ``host_kv_pages`` pinned host pages (``host_k`` / ``host_v``) and ``swap_out`` / ``swap_in``,
    which move whole pages between them and the device pool between replays (``_PagedKV``)."""

    def __init__(self, model: UltravoxModel, slots: int, max_len: int, kv_pages: int, eos_token_ids=None, pad_token_id: int = 0,
                 use_graph: bool = True, max_logprobs: int = 0, kv_cache_dtype: str = "bf16", kv_scales=None, host_kv_pages: int = 0,
                 prompt_lookup_num_tokens: Optional[int] = None, max_constraint_tokens: Optional[int] = None,
                 max_stop_table: Optional[int] = None):
        check_lookup_k(int(slots), prompt_lookup_num_tokens)      # before the pool is allocated
        kv = _PagedKV(model, int(slots), max_len, kv_pages, kv_cache_dtype, kv_scales, host_kv_pages)
        self.kv_pages, self.pool_k, self.pool_v, self.kv_scales = kv.kv_pages, kv.pool_k, kv.pool_v, kv.kv_scales
        self.host_kv_pages, self.host_k, self.host_v = kv.host_kv_pages, kv.host_k, kv.host_v
        self.swap_out, self.swap_in = kv.swap_out, kv.swap_in
        self._setup(model, int(slots), kv, eos_token_ids, pad_token_id, use_graph, max_logprobs, prompt_lookup_num_tokens,
                    max_constraint_tokens, max_stop_table)
