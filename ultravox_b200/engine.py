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
from .model import UltravoxModel

GEMV_MAX_B = int(os.environ.get("UVX_GEMV_MAX_B", "1"))     # decode streams up to which the linears run as matrix-vector kernels


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


class DecodeEngine:
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
        self.model, self.B = model, batch
        dev = model.device
        self.cache = cache if cache is not None else model.new_cache(batch, max_len)
        self.max_len = self.cache.capacity
        self.pos = torch.zeros(batch, dtype=torch.int32, device=dev)        # cache slot of the token being fed
        self.lens = torch.zeros(batch, dtype=torch.int32, device=dev)       # keys visible to it (= pos + 1)
        self.rope_pos = torch.zeros(batch, dtype=torch.int32, device=dev)   # its RoPE position (= pos - left padding)
        self.kv_start: Optional[torch.Tensor] = None
        self.token = torch.zeros(batch, 1, dtype=torch.int64, device=dev)
        self.seq = torch.zeros(batch, self.max_len + 1, dtype=torch.int64, device=dev)
        self.cur_len = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step_idx = torch.zeros(1, dtype=torch.int32, device=dev)
        self.done = torch.zeros(batch, dtype=torch.int32, device=dev)
        self.all_done = torch.zeros(1, dtype=torch.int32, device=dev)
        eos = sorted(set([eos_token_ids] if isinstance(eos_token_ids, int) else (eos_token_ids or [])))
        self.eos = torch.tensor(eos, dtype=torch.int64, device=dev) if eos else None
        self.pad_id = int(pad_token_id)
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
        self.cos, self.sin = model._rope_tables(self.max_len + 1)
        self.graph = None
        self.use_graph = use_graph
        self.launches_per_step = 0
        self.logits = None

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
        pad = kv_start if kv_start is not None else torch.zeros(B, dtype=torch.int32, device=self.pos.device)
        # the pick's token_finish bumps all three by one: the first new token sits at slot S, sees S + 1 keys, RoPE S - pad
        self.pos.fill_(S - 1)
        self.lens.fill_(S)
        self.rope_pos.copy_((S - 1) - pad.to(torch.int32))
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

    # -- one step ------------------------------------------------------------------------------------------
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

    def _step(self):
        m = self.model
        lm, tc = m.language_model, m.config.text_config
        nq, nkv, hd, Dm = tc.num_attention_heads, tc.num_key_value_heads, lm.head_dim, tc.hidden_size
        B = self.B
        # one stream: matrix-vector kernels (fp32 FMAs on the CUDA cores keep up with the weight stream) with RMSNorm / SwiGLU fused
        # into their prologues; more streams: the tensor-core GEMM (at B = 8 the FMA work per weight byte is 8x and the GEMV is
        # instruction-bound)
        one = B <= GEMV_MAX_B
        eps = tc.rms_norm_eps
        h = ops.embed_splice(self.token, lm.model.embed_tokens.weight, None, None).view(B, Dm)
        smax = self.cache.k.shape[2]
        for li, layer in enumerate(lm.model.layers):
            sa, mlp = layer.self_attn, layer.mlp
            kc, vc = self.cache.k[li], self.cache.v[li]
            if one:     # RMSNorm rides in the matrix-vector kernel's prologue
                qkv = ops.gemv(h, sa.qkv_w, norm=(layer.input_layernorm.weight, eps))
            else:
                qkv = ops.linear(ops.rmsnorm(h, layer.input_layernorm.weight, eps), sa.qkv_w)
            ops.rope_kv_append_(qkv, nq, nkv, hd, self.cos, self.sin, self.rope_pos, kc, vc, self.pos)
            att = torch.empty(B, nq * hd, dtype=torch.bfloat16, device=h.device)
            rs = qkv.stride(0)
            ops.attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), att, B, nq, nkv, 1, smax, hd,
                          (rs, rs, nkv * hd, smax * nkv * hd, nkv * hd, smax * nkv * hd, nq * hd, nq * hd), hd ** -0.5, False,
                          self.lens, 0, self.kv_start)
            if one:
                h = ops.gemv(att, sa.o_proj.weight, residual=h)
                gu = ops.gemv(h, mlp.gate_up_w, norm=(layer.post_attention_layernorm.weight, eps))
                h = ops.gemv(gu, mlp.down_proj.weight, residual=h, swiglu=True)         # act_fn(gate) * up in the prologue
            else:
                h = ops.linear(att, sa.o_proj.weight, residual=h)
                x = ops.rmsnorm(h, layer.post_attention_layernorm.weight, eps)
                act = ops.swiglu(ops.linear(x, mlp.gate_up_w), gate_first=True)
                h = ops.linear(act, mlp.down_proj.weight, residual=h)
        hn = ops.rmsnorm(h, lm.model.norm.weight, eps)
        self._pick(ops.lm_head(hn, lm.lm_head.weight))

    def step(self) -> torch.Tensor:
        """Feeds ``self.token`` (the previous output), writes the next token into it; returns the device tensor."""
        if self.use_graph and self.graph is None:
            self._step_warm()
        if self.graph is not None:
            self.graph.replay()
        else:
            self._step()
        return self.token

    def _state(self):
        return [self.pos, self.lens, self.rope_pos, self.token, self.cur_len, self.step_idx, self.done, self.all_done]

    def _step_warm(self):
        # warm-up on a scratch copy of the state, then capture; the state is restored so no token is lost (the cache row and the
        # sequence column the two trial steps write are rewritten with the same values by the first real step)
        saved = [t.clone() for t in self._state()]
        self._step()
        torch.cuda.synchronize()
        for t, s0 in zip(self._state(), saved):
            t.copy_(s0)
        before = _lib.launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            self._step()
        self.launches_per_step = _lib.launch_count() - before
        for t, s0 in zip(self._state(), saved):
            t.copy_(s0)
        torch.cuda.synchronize()
        self.graph = g
