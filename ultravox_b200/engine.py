"""Prefill engine: the whole hot path (waveform -> log-mel -> Whisper encoder -> projector -> splice -> Llama prefill
-> last-position logits -> greedy token) recorded once into a CUDA graph and replayed per request.

This is the serving-side caller of ``UltravoxModel`` for fixed request shapes (what ``LocalInference.infer`` +
``model.generate(max_new_tokens=1)`` does in the reference, ref:ultravox/inference/infer.py:125-153,309-342), with the
host work (processor bookkeeping) hoisted out: per request only the waveform changes.  One engine per process / GPU;
multi-GPU inference is independent replicas (SURVEY.md 8e) - no collective.
"""
from __future__ import annotations

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


class _RowKV:
    """The KV cache as one ``[S_max]`` row per decode row (stream, beam or slot): ``cache`` [L, rows, S_max, Hkv, D]."""

    keeps_kv = False        # whether a request's KV cache can outlive its slot (conversation sessions)

    def __init__(self, cache: KVCache):
        self.cache = cache

    def map_rows(self, e: "_Decoder", R: int) -> None:
        """Before the embedding of a step over R rows: a row's cache row is its own (or ``_mrow``'s), nothing to map."""

    def attend(self, e: "_Decoder", li: int, qkv: torch.Tensor) -> torch.Tensor:
        """The cache-touching calls of layer ``li`` of a step over the R rows of ``qkv``: RoPE on q / k + the KV append, then
        attention of the B decode rows over their cache rows and, in a mixed step (R > B), of the chunk rows over the prefilling
        slot's row -> [R, Hq * D].  A plain step appends row b at ``pos[b]`` of cache row b, a mixed step through ``_mrow``."""
        nq, nkv, hd = e.heads
        B, R = e.B, qkv.shape[0]
        kc, vc = self.cache.k[li], self.cache.v[li]
        smax = kc.shape[1]
        if R == B:
            ops.rope_kv_append_(qkv, nq, nkv, hd, e.cos, e.sin, e.rope_pos, kc, vc, e.pos)
        else:
            ops.rope_kv_append_map_(qkv, nq, nkv, hd, e.cos, e.sin, e._mrope, kc, vc, e._mrow, e._mpos)
        att = torch.empty(R, nq * hd, dtype=torch.bfloat16, device=qkv.device)
        rs = qkv.stride(0)
        ops.attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), att, B, nq, nkv, 1, smax, hd,
                      (rs, rs, nkv * hd, smax * nkv * hd, nkv * hd, smax * nkv * hd, nq * hd, nq * hd), hd ** -0.5, False,
                      e.lens, 0, e.kv_start)
        if R > B:
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
    are scattered into its pages."""

    keeps_kv = True

    def __init__(self, model: UltravoxModel, slots: int, max_len: int, kv_pages: int):
        lm, tc = model.language_model, model.config.text_config
        dev = model.device
        if int(kv_pages) < 1:
            raise ValueError(f"kv_pages must be >= 1, got {kv_pages}")
        self.kv_pages = int(kv_pages)
        self.table_width = -(-int(max_len) // ops.PAGE)
        L, nkv, hd = tc.num_hidden_layers, tc.num_key_value_heads, lm.head_dim
        self.pool_k = torch.empty(L, self.kv_pages + slots, ops.PAGE, nkv, hd, dtype=torch.bfloat16, device=dev)
        self.pool_v = torch.empty_like(self.pool_k)
        self.table = torch.full((slots, self.table_width), -1, dtype=torch.int32, device=dev)
        R = max(slots, PREFILL_ROWS)        # the rows of a mixed step (slots decode rows + PREFILL_ROWS - slots chunk rows)
        self.page = torch.zeros(R, dtype=torch.int32, device=dev)      # the page map's output: page / offset of every row
        self.off = torch.zeros(R, dtype=torch.int32, device=dev)
        self.cache = model.new_cache(1, max_len)
        self.pages = None                   # the admitted request's pages on the device

    def map_rows(self, e: "_Decoder", R: int) -> None:
        ops.kv_page_map(self.table, e._mrow[:R], e._mpos[:R], self.page[:R], self.off[:R], frozen=e.done)

    def attend(self, e: "_Decoder", li: int, qkv: torch.Tensor) -> torch.Tensor:
        """``_RowKV.attend`` through the page map and the table: every row appends at its (page, offset)."""
        nq, nkv, hd = e.heads
        B, R = e.B, qkv.shape[0]
        kp, vp = self.pool_k[li], self.pool_v[li]
        ops.rope_kv_append_map_(qkv, nq, nkv, hd, e.cos, e.sin, e._mrope[:R], kp, vp, self.page[:R], self.off[:R])
        att = torch.empty(R, nq * hd, dtype=torch.bfloat16, device=qkv.device)
        ops.attention_paged(qkv[:B, :nq * hd], kp, vp, att[:B], nq, hd ** -0.5, self.table, e.lens)
        if R > B:
            ops.attention_indexed_paged(qkv[B:, :nq * hd].unsqueeze(0), kp, vp, att[B:].unsqueeze(0), nq, hd ** -0.5, self.table,
                                        *e._mscal.split(1))
        return att

    def prefill(self, model: UltravoxModel, j: int, input_ids: torch.Tensor, past: int, features: dict) -> torch.Tensor:
        """Gather [0, past) into the scratch row, prefill [past, S) there exactly as ``generate(past_key_values=...)`` does, scatter
        [past, S) into the pages ``install`` gave slot ``j``."""
        S = int(input_ids.shape[1])
        row = self.cache
        if past:
            ops.kv_pages_copy(row.k, row.v, self.pool_k, self.pool_v, self.pages, 0, past, to_pages=False)
            emb = model.prompt_embeds(input_ids, **features)       # embed + splice the whole prompt, prefill only the new suffix
            out = model.forward(input_ids[:, past:], None, emb[:, past:].contiguous(), past_key_values=KVCache(row.k, row.v, past),
                                logits_to_keep=1)
        else:
            out = model.forward(input_ids, past_key_values=KVCache(row.k, row.v), logits_to_keep=1, **features)
        ops.kv_pages_copy(row.k, row.v, self.pool_k, self.pool_v, self.pages, past, S, to_pages=True)
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
    def _forward(self, mixed_in: Optional[torch.Tensor] = None, head_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Embedding -> layers -> final norm -> LM head of a step -> fp32 logits.  A plain step (``mixed_in`` None) feeds the B
        rows of ``token``.  A mixed step feeds ``mixed_in`` [R, D]: the token embedding is written into its first B rows, the
        prompt-chunk rows follow, and the LM head runs over rows ``head_rows`` only."""
        m = self.model
        lm, tc = m.language_model, m.config.text_config
        B = self.B
        # one stream: matrix-vector kernels (fp32 FMAs on the CUDA cores keep up with the weight stream) with RMSNorm / SwiGLU fused
        # into their prologues; more streams: the tensor-core GEMM (at B = 8 the FMA work per weight byte is 8x and the GEMV is
        # instruction-bound)
        one = mixed_in is None and B <= GEMV_MAX_B
        eps = tc.rms_norm_eps
        self.kv.map_rows(self, B if mixed_in is None else mixed_in.shape[0])
        if mixed_in is None:
            h = ops.embed_splice(self.token, lm.model.embed_tokens.weight, None, None).view(B, tc.hidden_size)
        else:
            h = mixed_in
            ops.embed_splice(self.token, lm.model.embed_tokens.weight, None, None, out=h[:B])
        for li, layer in enumerate(lm.model.layers):
            sa, mlp = layer.self_attn, layer.mlp
            if one:     # RMSNorm rides in the matrix-vector kernel's prologue
                qkv = ops.gemv(h, sa.qkv_w, norm=(layer.input_layernorm.weight, eps))
            else:
                qkv = ops.linear(ops.rmsnorm(h, layer.input_layernorm.weight, eps), sa.qkv_w)
            att = self.kv.attend(self, li, qkv)
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
                 repetition_penalty: float = 1.0, generator: Optional[torch.Generator] = None, top_p: Optional[float] = None):
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
        if self.penalty != 1.0:
            ops.repetition_penalty_(logits, self.seq, self.cur_len, self.penalty, self.scratch)
        tok = self.token.view(-1)
        if self.temperature > 0:
            ops.sample(logits, self.temperature, self.top_k, self.u, self.step_idx, out=tok, top_p=self.top_p)
        else:
            ops.argmax(logits, out=tok)
        ops.token_finish(tok, self.done, self.eos, self.pad_id, self.seq, self.cur_len, self.step_idx,
                         (self.pos, self.lens, self.rope_pos), self.all_done)

    def _state(self):
        return [self.pos, self.lens, self.rope_pos, self.token, self.cur_len, self.step_idx, self.done, self.all_done]


class BeamDecodeEngine(DecodeEngine):
    """Beam search over ``batch`` prompts with ``num_beams`` beams each (row b * num_beams + j), as
    hf:generation/utils.py ``_beam_search``: the forward of ``DecodeEngine._step`` runs unchanged over the batch * num_beams
    rows, and the pick becomes log_softmax -> repetition penalty on the log-probs -> top-K continuations per prompt ->
    running beams / finished pool / early-stop heuristic -> KV cache rows gathered by parent beam, all on the device, so a
    step is still one CUDA graph replay.  ``all_done`` is HF's loop condition (negated); ``logprobs`` holds the last step's
    processed log-probs [batch * num_beams, V] and ``logits`` the raw ones.  The cache must have batch * num_beams rows with
    each prompt prefilled into row b * num_beams (``begin`` broadcasts it to the other beams)."""

    def __init__(self, model: UltravoxModel, batch: int, num_beams: int, max_len: int, max_new_tokens: int, use_graph: bool = True,
                 cache=None, eos_token_ids=None, length_penalty: float = 1.0, early_stopping=False, repetition_penalty: float = 1.0):
        nb = int(num_beams)
        if not 1 <= nb <= ops.BEAM_MAX:
            raise ValueError(f"num_beams must be in [1, {ops.BEAM_MAX}], got {num_beams}")
        if early_stopping not in (False, True, "never"):
            raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
        eos_list = [eos_token_ids] if isinstance(eos_token_ids, int) else list(eos_token_ids or [])
        super().__init__(model, batch * nb, max_len, use_graph=use_graph, cache=cache, eos_token_ids=eos_list,
                         repetition_penalty=repetition_penalty)
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
        if self.penalty != 1.0:
            ops.repetition_penalty_(lp, self.seq, self.cur_len, self.penalty, self.scratch)
        s, i = ops.beam_select(lp, self.run_score, self.nb, self.K, scratch=self.row_buf, out=self.cand)
        ops.beam_update(s, i, self.V, self.nb, self.eos, self.max_new, self.len_div, self.es, self.length_penalty > 0.0, self._beam,
                        self._counters, (self.pos, self.lens, self.rope_pos))
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
    all rows followed by three per-row kernels (``uvx_repetition_penalty_slots``, ``uvx_sample_slots``, ``uvx_slot_finish``);
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
    decoding; the decode rows of a mixed step run at 256 rows instead of ``slots`` and are not bit-identical to a plain step."""

    def __init__(self, model: UltravoxModel, slots: int, max_len: int, eos_token_ids=None, pad_token_id: int = 0,
                 use_graph: bool = True, cache=None):
        kv = _RowKV(cache if cache is not None else model.new_cache(slots, max_len))
        self._setup(model, int(slots), kv, eos_token_ids, pad_token_id, use_graph)

    def _setup(self, model: UltravoxModel, slots: int, kv, eos_token_ids, pad_token_id: int, use_graph: bool):
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
        self.kv.release(j)

    def _state(self):
        return [self.pos, self.lens, self.rope_pos, self.token, self.cur_len, self.n_new, self.done, self.n_open]

    def _pick_rows(self, logits: torch.Tensor, r: slice, n_open: torch.Tensor) -> None:
        tok = self.token.view(-1)[r]
        ops.repetition_penalty_slots_(logits, self.seq[r], self.cur_len[r], self.penalties[r], self.active[r], self.scratch[r])
        ops.sample_slots(logits, self.temps[r], self.top_ks[r], self.top_ps[r], self.u[r], self.n_new[r], self.active[r], tok)
        ops.slot_finish(tok, self.done[r], self.eos, self.seq[r], self.cur_len[r], self.n_new[r], self.max_new[r], self.active[r],
                        self.pos[r], self.lens[r], self.rope_pos[r], n_open)

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
            self._seed(j, S)
            self._mrow[j] = j
            self._pick_rows(self._chunk_logits, slice(j, j + 1), self._admit_open)
        return self.token

    def admit(self, slot: int, input_ids: torch.Tensor, max_new_tokens: int, temperature: float = 0.0, top_k: int = 0,
              top_p: float = 1.0, repetition_penalty: float = 1.0, u: Optional[torch.Tensor] = None, past: int = 0,
              pages=None, **features) -> torch.Tensor:
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
        S + max_new_tokens positions, and the first ceil(past / 64) of them hold the conversation's first ``past`` positions."""
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
            self._prefill = dict(slot=j, S=S, done=P, embeds=embeds)
            self._mrow[j] = -1          # the slot's idle decode row must not overwrite position 0 of the prompt
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
        self.penalties[j] = float(repetition_penalty or 1.0)
        if u is not None:
            w = min(u.numel(), self.max_len + 1)
            self.u[j, :w].copy_(u.reshape(-1)[:w])
        self.busy[j] = True
        if not chunked:
            self._pick_rows(logits, slice(j, j + 1), self._admit_open)
        return self.token.view(-1)

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
    (``serving.PagePool``)."""

    def __init__(self, model: UltravoxModel, slots: int, max_len: int, kv_pages: int, eos_token_ids=None, pad_token_id: int = 0,
                 use_graph: bool = True):
        kv = _PagedKV(model, int(slots), max_len, kv_pages)
        self.kv_pages, self.pool_k, self.pool_v = kv.kv_pages, kv.pool_k, kv.pool_v
        self._setup(model, int(slots), kv, eos_token_ids, pad_token_id, use_graph)
