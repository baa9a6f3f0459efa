"""``UltravoxModel`` - drop-in model surface over the hand-written sm_90a kernels.

Mirrors ``ref:ultravox/model/ultravox_model.py``: ``UltravoxModel.forward`` (:277-352), ``_prepare_audio_embeds``
(:354-396), ``generate`` (:398-426), ``ModifiedWhisperEncoder.forward`` (:865-994), ``UltravoxProjector.forward``
(:768-800), ``StackAudioFrames`` (:722-730); parameter names / state-dict keys are the reference's
(``audio_tower.*``, ``multi_modal_projector.*``, ``language_model.*``), so checkpoints load unchanged.

H100-first differences (none observable through the interface):
* every op is a libuvx kernel (``ops``); q/k/v (and gate/up) projections run as ONE wgmma GEMM over a fused
  weight - the per-projection ``nn.Parameter``s are views into that fused storage, so state-dict I/O is unchanged;
* the conv stem runs as implicit GEMMs over a time-major guard-padded activation (no im2col, no permute);
* StackAudioFrames is folded into the ln_pre kernel's addressing; the splice is one sync-free gather kernel driven
  by a device index table (the reference does a host sync per chunk);
* encoder attention masks are generated from ``audio_lens`` inside the attention kernel (no dense mask tensor);
* log-mel can run on device from raw waveforms (``audio_waveforms``), fused with the bf16 time-major re-layout.
There is no CPU fallback: tensors must be CUDA tensors and ``libuvx.so`` must be built.
"""
from __future__ import annotations

import dataclasses
import os
from typing import Optional

import torch
import torch.nn as nn
from transformers.modeling_outputs import CausalLMOutputWithPast

from . import ops
from .config import LossConfig, LossFunction, UltravoxConfig

FUSE_NORM = os.environ.get("UVX_FUSE_NORM", "1") != "0"   # tuning switch: RMSNorm fused into the o_proj / down_proj split-K pass
USE_TILED = os.environ.get("UVX_TILED", "1") != "0"       # LLM prefill GEMMs stream pre-tiled weight images (contiguous DRAM runs)
FUSE_ROPE = os.environ.get("UVX_FUSE_ROPE", "1") != "0"   # RoPE in the q|k|v GEMM epilogue (head_dim 128)
QKV_MODE = os.environ.get("UVX_QKV_MODE", "fused")        # Llama q|k|v GEMM: "fused" RoPE epilogue | "r1" round-1 kernel + uvx_rope | "tma" + uvx_rope
TILED_SET = os.environ.get("UVX_TILED_SET", "gate_up")        # which LLM projections get a pre-tiled image: "all" | "gate_up" | "mlp" (in situ only gate|up gains: r2_ab_bench_v3)
USE_WS = os.environ.get("UVX_GEMM_WS", "0") == "1"         # opt-in: rows <= 256 run the single-pass GEMM form (no split-K) over 128-row images of all four projections
FUSE_SWIGLU = os.environ.get("UVX_FUSE_SWIGLU", "1") != "0"   # act(gate)*up in the gate|up GEMM epilogue (needs the tiled image)
BF16 = torch.bfloat16


# ------------------------------------------------------------------------------------------------ containers
class _P(nn.Module):
    """A leaf holding ``weight`` (and optionally ``bias``) - gives the reference's ``x.weight`` key names."""

    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor] = None):
        super().__init__()
        self.weight = nn.Parameter(weight, requires_grad=False)
        if bias is not None:
            self.bias = nn.Parameter(bias, requires_grad=False)
        else:
            self.bias = None


class _Embed(_P):
    """Token-embedding leaf: ``weight`` plus the two attributes callers read off ``nn.Embedding`` (ref :144-156)."""

    @property
    def num_embeddings(self) -> int:
        return int(self.weight.shape[0])

    @property
    def embedding_dim(self) -> int:
        return int(self.weight.shape[1])


def _empty(*shape, device, dtype=BF16):
    return torch.empty(*shape, device=device, dtype=dtype)


class _WhisperAttn(nn.Module):
    def __init__(self, d, device):
        super().__init__()
        self.qkv_w = _empty(3 * d, d, device=device)   # fused storage (not a parameter; views below are)
        self.qkv_b = torch.zeros(3 * d, device=device, dtype=BF16)
        self.q_proj = _P(self.qkv_w[0:d], self.qkv_b[0:d])
        self.k_proj = _P(self.qkv_w[d:2 * d])           # no bias (hf:modeling_whisper.py:279)
        self.v_proj = _P(self.qkv_w[2 * d:], self.qkv_b[2 * d:])
        self.out_proj = _P(_empty(d, d, device=device), _empty(d, device=device))


class _WhisperLayer(nn.Module):
    def __init__(self, d, ffn, device):
        super().__init__()
        self.self_attn = _WhisperAttn(d, device)
        self.self_attn_layer_norm = _P(_empty(d, device=device), _empty(d, device=device))
        self.fc1 = _P(_empty(ffn, d, device=device), _empty(ffn, device=device))
        self.fc2 = _P(_empty(d, ffn, device=device), _empty(d, device=device))
        self.final_layer_norm = _P(_empty(d, device=device), _empty(d, device=device))


class AudioTower(nn.Module):
    """Whisper encoder weights (``ModifiedWhisperEncoder``, ref :803-994)."""

    def __init__(self, ac, device):
        super().__init__()
        d = ac.d_model
        self.d, self.heads, self.n_mels, self.max_pos = d, ac.encoder_attention_heads, ac.num_mel_bins, ac.max_source_positions
        self.conv1 = _P(_empty(d, ac.num_mel_bins, 3, device=device), _empty(d, device=device))
        self.conv2 = _P(_empty(d, d, 3, device=device), _empty(d, device=device))
        self.embed_positions = _P(_empty(ac.max_source_positions, d, device=device))
        self.layers = nn.ModuleList([_WhisperLayer(d, ac.encoder_ffn_dim, device) for _ in range(ac.encoder_layers)])
        self.layer_norm = _P(_empty(d, device=device), _empty(d, device=device))

    @property
    def max_context_length(self) -> int:   # ref :826-832 (conv strides 1 and 2)
        return self.max_pos * 2


class Projector(nn.Module):
    """``UltravoxProjector`` weights (ref :745-766).  The trainable tensors are views into ONE flat bf16 buffer
    (``flat``) in a fixed order, so the optimizer step and the data-parallel gradient all-reduce are single launches
    over a contiguous 50.3 M-element range; state-dict names are unchanged."""

    def __init__(self, config: UltravoxConfig, device):
        super().__init__()
        dim_in = config.audio_config.d_model * config.stack_factor
        hid = config.hidden_size
        mid = hid // 2 if config.projector_act == "swiglu" else hid
        out = config.text_config.hidden_size
        self.dims = (dim_in, hid, mid, out)
        norm2 = "ln_mid" if config.projector_ln_mid else "ln_post"
        layout = [("ln_pre", (dim_in,)), ("linear_1", (hid, dim_in)), (norm2, (mid if config.projector_ln_mid else out,)),
                  ("linear_2", (out, mid))]
        total = sum(int(torch.Size(shape).numel()) for _, shape in layout)
        self.flat = _empty(total, device=device)
        self.slices = {}
        off = 0
        for name, shape in layout:
            n = int(torch.Size(shape).numel())
            setattr(self, name, _P(self.flat[off:off + n].view(*shape)))
            self.slices[name] = (off, n, shape)
            off += n


class _LlamaAttn(nn.Module):
    def __init__(self, h, nq, nkv, hd, device):
        super().__init__()
        self.qkv_w = _empty((nq + 2 * nkv) * hd, h, device=device)
        self.q_proj = _P(self.qkv_w[: nq * hd])
        self.k_proj = _P(self.qkv_w[nq * hd: (nq + nkv) * hd])
        self.v_proj = _P(self.qkv_w[(nq + nkv) * hd:])
        self.o_proj = _P(_empty(h, nq * hd, device=device))


class _LlamaMLP(nn.Module):
    def __init__(self, h, ffn, device):
        super().__init__()
        self.gate_up_w = _empty(2 * ffn, h, device=device)
        self.gate_proj = _P(self.gate_up_w[:ffn])
        self.up_proj = _P(self.gate_up_w[ffn:])
        self.down_proj = _P(_empty(h, ffn, device=device))


class _LlamaLayer(nn.Module):
    def __init__(self, tc, hd, device):
        super().__init__()
        self.self_attn = _LlamaAttn(tc.hidden_size, tc.num_attention_heads, tc.num_key_value_heads, hd, device)
        self.mlp = _LlamaMLP(tc.hidden_size, tc.intermediate_size, device)
        self.input_layernorm = _P(_empty(tc.hidden_size, device=device))
        self.post_attention_layernorm = _P(_empty(tc.hidden_size, device=device))


class _LlamaInner(nn.Module):
    def __init__(self, tc, hd, device):
        super().__init__()
        self.embed_tokens = _Embed(_empty(tc.vocab_size, tc.hidden_size, device=device))
        self.layers = nn.ModuleList([_LlamaLayer(tc, hd, device) for _ in range(tc.num_hidden_layers)])
        self.norm = _P(_empty(tc.hidden_size, device=device))


class LanguageModel(nn.Module):
    def __init__(self, tc, device):
        super().__init__()
        self.head_dim = getattr(tc, "head_dim", None) or tc.hidden_size // tc.num_attention_heads
        self.model = _LlamaInner(tc, self.head_dim, device)
        self.tied = bool(getattr(tc, "tie_word_embeddings", False))
        if self.tied:
            self.lm_head = _Embed(self.model.embed_tokens.weight.data)
        else:
            self.lm_head = _Embed(_empty(tc.vocab_size, tc.hidden_size, device=device))

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    def tie_weights(self):
        """Tied checkpoints (Llama-3.2-1B): lm_head shares the embedding storage (hf:modeling_utils.py tie_weights)."""
        if self.tied:
            self.lm_head.weight = nn.Parameter(self.model.embed_tokens.weight.data, requires_grad=False)


@dataclasses.dataclass
class KVCache:
    """Static per-layer K (post-RoPE) / V cache, [L, B, S_max, Hkv, D] bf16."""
    k: torch.Tensor
    v: torch.Tensor
    length: int = 0

    def get_seq_length(self) -> int:
        return self.length

    @property
    def capacity(self) -> int:
        return int(self.k.shape[2])

    def grown(self, max_len: int) -> "KVCache":
        """A cache with room for ``max_len`` positions holding the same ``length`` entries (conversation turns grow it)."""
        if max_len <= self.capacity:
            return self
        shape = list(self.k.shape)
        shape[2] = max_len
        k, v = self.k.new_empty(shape), self.v.new_empty(shape)
        k[:, :, :self.length].copy_(self.k[:, :, :self.length])
        v[:, :, :self.length].copy_(self.v[:, :, :self.length])
        return KVCache(k, v, self.length)


@dataclasses.dataclass
class GenerateOutput:
    """``return_dict_in_generate=True`` result: what the reference's conversation mode reads (ref infer.py:131-148), plus the
    final beam scores of a beam search asked for with ``output_scores=True`` (HF's ``sequences_scores``)."""
    sequences: torch.Tensor
    past_key_values: Optional[KVCache]
    sequences_scores: Optional[torch.Tensor] = None


# ------------------------------------------------------------------------------------------------ the model
class UltravoxModel(nn.Module):
    config_class = UltravoxConfig
    _keys_to_ignore_on_load_missing = ["audio_tower.*", "language_model.*"]
    accepts_loss_kwargs = False

    def __init__(self, config: UltravoxConfig, device="cuda"):
        super().__init__()
        self.config = config
        self.vocab_size = config.vocab_size
        self.keep_params: set[str] = set()
        dev = torch.device(device)
        if not config.llm_only_training:
            self.audio_tower = AudioTower(config.audio_config, dev)
            self.multi_modal_projector = Projector(config, dev)
            self.audio_tower_context_length = self.audio_tower.max_context_length
        self.language_model = LanguageModel(config.text_config, dev)
        self.loss_config = LossConfig()
        self._derived: dict = {}
        self._rope: Optional[tuple] = None
        # projector params are the trainable ones in the adapter-only recipe (ref apply_lora r=0 freezes the rest)
        if not config.llm_only_training:
            for p in self.multi_modal_projector.parameters():
                p.requires_grad_(True)

    # -- reference surface ---------------------------------------------------------------------------
    def get_input_embeddings(self):
        return self.language_model.get_input_embeddings()

    def set_input_embeddings(self, value):
        """ref :115-116.  ``value``: anything with a ``weight`` [V, D] (an ``nn.Embedding`` in the reference)."""
        w = value.weight if hasattr(value, "weight") else value
        emb = self.language_model.model.embed_tokens
        emb.weight = nn.Parameter(w.detach().to(self.device, BF16).contiguous(), requires_grad=False)
        self.language_model.tie_weights()

    def get_output_embeddings(self):
        return self.language_model.get_output_embeddings()

    def set_output_embeddings(self, new_embeddings):
        w = new_embeddings.weight if hasattr(new_embeddings, "weight") else new_embeddings
        self.language_model.lm_head.weight = nn.Parameter(w.detach().to(self.device, BF16).contiguous(), requires_grad=False)

    def get_decoder(self):
        return self.language_model.model

    def tie_weights(self, **_):
        return self.language_model.tie_weights()

    def set_loss_config(self, loss_config: LossConfig):
        self.loss_config = loss_config

    @torch.no_grad()
    def resize_token_embeddings(self, new_num_tokens: Optional[int] = None, pad_to_multiple_of: Optional[int] = None):
        """ref :144-156 (-> hf:modeling_utils.py resize_token_embeddings): grows / shrinks ``embed_tokens`` and ``lm_head`` and
        updates the three vocab-size fields.  New rows are set to the mean of the existing rows (HF's ``mean_resizing`` default
        draws them from a Gaussian around that mean)."""
        emb = self.language_model.model.embed_tokens
        old = emb.num_embeddings
        if new_num_tokens is None:
            return emb
        if pad_to_multiple_of:
            new_num_tokens = -(-new_num_tokens // pad_to_multiple_of) * pad_to_multiple_of

        def resized(w):
            out = torch.empty(new_num_tokens, w.shape[1], dtype=w.dtype, device=w.device)
            n = min(old, new_num_tokens)
            out[:n] = w[:n]
            if new_num_tokens > old:
                out[old:] = w.float().mean(0, keepdim=True).to(w.dtype)
            return out

        emb.weight = nn.Parameter(resized(emb.weight.data), requires_grad=False)
        if self.language_model.tied:
            self.language_model.tie_weights()
        else:
            head = self.language_model.lm_head
            head.weight = nn.Parameter(resized(head.weight.data), requires_grad=False)
        self.config.text_config.vocab_size = self.config.vocab_size = self.vocab_size = new_num_tokens
        self._wT = None                     # transposed lm_head of the training path is rebuilt on demand
        return emb

    def merge_and_unload(self):
        """ref :528-559.  LoRA adapters are folded into the fused base weights when a checkpoint is LOADED (``lora.py``), so
        there is nothing left to merge; what remains is the reference's bookkeeping: the merged towers must be saved with the
        adapter checkpoint (``keep_params``), their hub ids no longer apply, and the LoRA configs leave the config."""
        for comp, id_attr, cfg_attr in (("language_model", "text_model_id", "text_model_lora_config"),
                                        ("audio_tower", "audio_model_id", "audio_model_lora_config")):
            lc = getattr(self.config, cfg_attr, None) or {}
            if hasattr(self, comp) and int(lc.get("r", 0) or 0) > 0:
                setattr(self.config, id_attr, None)
                self.keep_params.update(f"{comp}.{n}" for n, _ in getattr(self, comp).named_parameters())
        for cfg_attr in ("text_model_lora_config", "audio_model_lora_config"):
            if hasattr(self.config, cfg_attr):
                delattr(self.config, cfg_attr)

    def print_trainable_parameters(self):
        tr = sum(p.numel() for p in self.parameters() if p.requires_grad)
        tot = sum(p.numel() for p in self.parameters())
        print(f"trainable params: {tr:,d} || all params: {tot:,d} || trainable%: {100 * tr / max(tot, 1):.4f}")

    # -- checkpoints (ref :103-110, :565-594) ---------------------------------------------------------
    def save_pretrained(self, save_directory, state_dict=None, safe_serialization: bool = True, **kwargs):
        """Writes ``config.json`` + the DIFF checkpoint (trainable and explicitly kept parameters only, ref :565-591) as
        ``model.safetensors`` - the layout ``from_pretrained`` (here and in the reference) reads back."""
        import os
        os.makedirs(save_directory, exist_ok=True)
        self.config.save_pretrained(save_directory)
        sd = {k: v.detach().to("cpu").contiguous().clone() for k, v in self.diff_state_dict(state_dict).items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(save_directory, "model.safetensors"), metadata={"format": "pt"})
        else:
            torch.save(sd, os.path.join(save_directory, "pytorch_model.bin"))

    @staticmethod
    def _read_checkpoint_dir(path: str) -> dict:
        """All tensors of a HF-style checkpoint directory: single / sharded safetensors or ``pytorch_model.bin``."""
        import glob
        import json
        import os
        from safetensors.torch import load_file
        idx = os.path.join(path, "model.safetensors.index.json")
        files = []
        if os.path.exists(idx):
            files = sorted({os.path.join(path, f) for f in json.load(open(idx))["weight_map"].values()})
        elif os.path.exists(os.path.join(path, "model.safetensors")):
            files = [os.path.join(path, "model.safetensors")]
        else:
            files = sorted(glob.glob(os.path.join(path, "*.safetensors")))
        out = {}
        for f in files:
            out.update(load_file(f))
        if not files and os.path.exists(os.path.join(path, "pytorch_model.bin")):
            out = torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu", weights_only=True)
        return out

    @staticmethod
    def _resolve_dir(model_id: str) -> str:
        import os
        if os.path.isdir(model_id):
            return model_id
        from huggingface_hub import snapshot_download
        return snapshot_download(model_id, allow_patterns=["*.safetensors", "*.json", "*.bin"])

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, *model_args, config: Optional[UltravoxConfig] = None, device="cuda",
                        **kwargs):
        """ref :103-110 -> ``PreTrainedModel.from_pretrained``: (1) the config, (2) the base towers named by ``text_model_id`` /
        ``audio_model_id`` (their own checkpoints, ref :440-526), (3) the diff checkpoint saved by ``save_pretrained`` (projector,
        merged / LoRA tower weights) on top, missing tower keys allowed (``_keys_to_ignore_on_load_missing``), (4) derived
        device buffers.  ``torch_dtype`` / ``device_map`` style kwargs of the HF API are accepted and ignored (bf16, one GPU)."""
        path = cls._resolve_dir(str(pretrained_model_name_or_path))
        cfg = config or UltravoxConfig.from_pretrained(path)
        model = cls(cfg, device=device)
        if cfg.text_model_id:
            base = cls._read_checkpoint_dir(cls._resolve_dir(cfg.text_model_id))
            model.load_state_dict({"language_model." + k: v for k, v in base.items()}, strict=False, _track=False)
        if cfg.audio_model_id and hasattr(model, "audio_tower"):
            base = cls._read_checkpoint_dir(cls._resolve_dir(cfg.audio_model_id))
            enc = {}
            for k, v in base.items():                      # WhisperModel / WhisperForConditionalGeneration -> encoder only
                for pre in ("model.encoder.", "encoder."):
                    if k.startswith(pre):
                        enc["audio_tower." + k[len(pre):]] = v
            model.load_state_dict(enc, strict=False, _track=False)
        model.load_state_dict(cls._read_checkpoint_dir(path), strict=True)
        model.prepare()
        return model.eval()

    @property
    def device(self):
        return self.language_model.model.norm.weight.device

    @property
    def dtype(self):
        return BF16

    def diff_state_dict(self, state_dict=None):
        """ref :565-584 - only trainable (+ explicitly kept) parameters."""
        sd = state_dict if state_dict is not None else self.state_dict()
        trainable = {k for k, v in self.named_parameters() if v.requires_grad}
        return {k: v for k, v in sd.items() if k in self.keep_params or k in trainable}

    # -- weights -------------------------------------------------------------------------------------
    @torch.no_grad()
    def init_random_(self, seed: int = 42):
        """Seeded synthetic weights (SURVEY.md 8d): Linear/Conv/Embedding ~ N(0, initializer_range), biases 0,
        Layer/RMS-norm weight 1, projector RMSNorm weights = norm_init, sinusoidal ``embed_positions``."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        std = self.config.initializer_range
        for name, p in self.named_parameters():
            if name.endswith("embed_positions.weight"):
                p.copy_(_sinusoids(p.shape[0], p.shape[1]).to(p.device, p.dtype))
            elif "multi_modal_projector.ln_" in name:
                p.fill_(self.config.norm_init)
            elif "layer_norm" in name or "layernorm" in name or name.endswith("model.norm.weight"):
                p.fill_(1.0) if name.endswith("weight") else p.zero_()
            elif name.endswith("bias"):
                p.zero_()
            else:
                # chunked fill keeps the fp32 staging buffer small for 8B / 70B
                flat = p.view(-1)
                step = 1 << 26
                for i in range(0, flat.numel(), step):
                    n = min(step, flat.numel() - i)
                    flat[i:i + n] = (torch.randn(n, generator=g, device=p.device, dtype=torch.float32) * std).to(p.dtype)
        self.prepare()
        return self

    @torch.no_grad()
    def prepare(self):
        """(Re)build derived device buffers: conv weights re-laid for the implicit GEMM, rope tables.  Call after
        loading / changing encoder conv weights."""
        if hasattr(self, "audio_tower"):
            at = self.audio_tower
            self._derived["conv1_w"] = at.conv1.weight.permute(0, 2, 1).reshape(at.d, -1).contiguous()
            self._derived["conv2_w"] = at.conv2.weight.permute(0, 2, 1).reshape(at.d, -1).contiguous()
        tc = self.config.text_config
        rp = getattr(tc, "rope_parameters", None) or {}
        scaling = getattr(tc, "rope_scaling", None) or (rp if rp.get("rope_type", "default") != "default" else None)
        theta = rp.get("rope_theta", None) or getattr(tc, "rope_theta", 10000.0)
        inv = ops.llama3_inv_freq(self.language_model.head_dim, float(theta), scaling)
        self._inv_freq = inv
        self._rope = None
        self._tiled = None          # pre-tiled LLM weight images are rebuilt lazily from the (possibly new) weights
        self._wT = None
        return self

    @torch.no_grad()
    def _tiled_weights(self):
        """Per-layer pre-tiled images of the frozen LLM projections for the prefill GEMMs (``ops.TiledWeight``): q|k|v, o and
        down as 128-row tiles, gate|up as 128-row tiles with 16 gate / 16 up rows interleaved (fused SwiGLU): 128-wide tiles let
        one CTA cover all rows of a prefill (two 128-row sub-tiles), so every weight byte is read once.  A derived copy like
        the conv weights (the named parameters keep the reference layout for state-dict I/O, decode GEMVs and training); built
        once, on first use, if the GPU has room for the second copy (8B: +15 GB; a 70B replica has not - it streams the
        row-major weights)."""
        if getattr(self, "_tiled", None) is None:
            self._tiled = False
            layers = self.language_model.model.layers
            if USE_TILED and len(layers) > 0 and layers[0].self_attn.qkv_w.is_cuda:
                tc = self.config.text_config
                hs, ffn = tc.hidden_size, tc.intermediate_size
                per_layer = 2 * (layers[0].self_attn.qkv_w.numel() + hs * layers[0].self_attn.o_proj.weight.shape[1] + 3 * hs * ffn)
                free, _ = torch.cuda.mem_get_info(self.device)
                if hs % 64 == 0 and ffn % 64 == 0 and ffn % 8 == 0 and free > 1.15 * per_layer * len(layers) + (8 << 30):
                    out = []
                    for layer in layers:
                        sa, mlp = layer.self_attn, layer.mlp
                        attn_t = USE_WS or TILED_SET == "all"
                        down_t = USE_WS or TILED_SET in ("all", "mlp")
                        gu_rows = 128
                        lm_hd = self.language_model.head_dim
                        out.append(dict(qkv=ops.TiledWeight(sa.qkv_w, 128, rope_pairs=USE_WS and lm_hd == 128) if attn_t else None,
                                        o=ops.TiledWeight(sa.o_proj.weight, 128) if attn_t else None,
                                        gate_up=ops.TiledWeight(mlp.gate_up_w, gu_rows, swiglu=True) if FUSE_SWIGLU
                                        else ops.TiledWeight(mlp.gate_up_w, gu_rows),
                                        down=ops.TiledWeight(mlp.down_proj.weight, 128) if down_t else None))
                    # the prefill GEMMs read these images with ops.GEMM_W_STATIC (their weight stream starts before the previous
                    # kernel ends): every image is complete before the first such call
                    if not torch.cuda.is_current_stream_capturing():
                        torch.cuda.current_stream(self.device).synchronize()
                    self._tiled = out
        return self._tiled or None

    def _rope_tables(self, need: int):
        """cos/sin [n, D/2] fp32; grown geometrically (long conversations with KV reuse decode one position at a time - growing
        to exactly ``need`` would rebuild the table on every step past the initial size)."""
        have = 0 if self._rope is None else self._rope[0].shape[0]
        if have < need:
            cap = int(getattr(self.config.text_config, "max_position_embeddings", 0) or 0)
            n = max(need, 4096, 2 * have)
            if cap >= need:
                n = min(n, cap)
            self._rope = ops.rope_tables(self._inv_freq, n, self.device)
        return self._rope

    # -- audio tower ---------------------------------------------------------------------------------
    def encode_audio(self, x_tm: torch.Tensor, audio_lens: Optional[torch.Tensor],
                     kv_len: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x_tm [N, T+2, n_mels] bf16 guard-padded time-major mel -> encoder output [N, ceil(T/2), d]
        (``ModifiedWhisperEncoder.forward``, ref :865-994)."""
        at = self.audio_tower
        N, Tp, _ = x_tm.shape
        T = Tp - 2
        if T > at.max_context_length:
            raise ValueError(f"Whisper expects the mel input features to be of length {at.max_context_length} or less, "
                             f"but found {T}. Make sure to pad the input mel features to {at.max_context_length}.")
        d, H = at.d, at.heads
        T2 = (T + 1) // 2
        dev = x_tm.device
        h1 = torch.zeros(N, T + 2, d, dtype=BF16, device=dev)
        ops.conv1d_k3(x_tm, self._derived["conv1_w"], at.conv1.bias, 1, h1, out_guard=True)
        h = torch.empty(N, T2, d, dtype=BF16, device=dev)
        ops.conv1d_k3(h1, self._derived["conv2_w"], at.conv2.bias, 2, h, out_guard=False,
                      pos=at.embed_positions.weight[:T2])
        if kv_len is None and audio_lens is not None:
            # hf _get_feat_extract_output_lengths (ref :915-917); computed where the tensor lives, then moved
            kv_len = ((audio_lens.to(torch.int64) - 1) // 2 + 1).to(torch.int32).to(dev)
        block = int(self.config.audio_latency_block_size or 0)
        hd = d // H
        x = torch.empty_like(h)
        qkv = torch.empty(N * T2, 3 * d, dtype=BF16, device=dev)
        att = torch.empty(N * T2, d, dtype=BF16, device=dev)
        ff = torch.empty(N * T2, at.layers[0].fc1.weight.shape[0], dtype=BF16, device=dev)
        for layer in at.layers:
            sa = layer.self_attn
            ops.layernorm(h, layer.self_attn_layer_norm.weight, layer.self_attn_layer_norm.bias, 1e-5, out=x)
            ops.linear(x, sa.qkv_w, sa.qkv_b, out=qkv)
            if hd == 64:
                ops.attention_encoder_tc(qkv, N, T2, H, hd ** -0.5, kv_len, block, out=att)
            else:
                ops.attention_fused_qkv(qkv, N, T2, H, H, hd, hd ** -0.5, False, kv_len, block, out=att)
            ops.linear(att, sa.out_proj.weight, sa.out_proj.bias, residual=h, out=h)
            ops.layernorm(h, layer.final_layer_norm.weight, layer.final_layer_norm.bias, 1e-5, out=x)
            ops.linear(x, layer.fc1.weight, layer.fc1.bias, act=ops.ACT_GELU, out=ff)
            ops.linear(ff, layer.fc2.weight, layer.fc2.bias, residual=h, out=h)
        return ops.layernorm(h, at.layer_norm.weight, at.layer_norm.bias, 1e-5, out=x)

    def project_audio(self, enc: torch.Tensor) -> torch.Tensor:
        """``UltravoxProjector.forward`` (ref :768-800): [N, T2, d] -> [N, ceil(T2/stack), D_text]."""
        pj, cfg = self.multi_modal_projector, self.config
        x = ops.stack_rmsnorm(enc, pj.ln_pre.weight, cfg.stack_factor, 1e-6)
        y = ops.linear(x, pj.linear_1.weight)
        if cfg.projector_act != "swiglu":
            raise NotImplementedError(f"projector_act={cfg.projector_act!r}: only 'swiglu' (all released configs) is built")
        z = ops.swiglu(y, gate_first=False)
        if cfg.projector_ln_mid:
            z = ops.rmsnorm(z, pj.ln_mid.weight, 1e-6)
        a = ops.linear(z, pj.linear_2.weight)
        if not cfg.projector_ln_mid:
            a = ops.rmsnorm(a, pj.ln_post.weight, 1e-6)
        return a

    def mel_chunks_from_waveforms(self, audio_waveforms: torch.Tensor, audio_num_frames: torch.Tensor,
                                  context: int = 3000, audio_pad_frames: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Zero-padded waveforms [B, L] (what ``UltravoxProcessor(defer_mel=True)`` hands over) -> time-major mel chunks
        [N, T+2, n_mels] bf16 with guard rows, chunked exactly like ``_chunk_and_pad_audio`` (ref processing :153-215):
        the log-mel (with its per-CLIP max) is computed once per clip on the GPU, then cut into <= ``context``-frame pieces;
        continuation chunks are zero-padded to ``context``, first chunks keep the batch width."""
        from .processing import frame_chunks
        dev = self.device
        waves = audio_waveforms.to(dev, torch.float32, non_blocking=True)
        n_mels = self.audio_tower.n_mels
        tm = ops.logmel(waves, n_mels, want_f32=False, want_tm=True)            # [B, Tfull+2, n_mels]
        t_full = tm.shape[1] - 2
        if audio_pad_frames is not None:
            # collated batches (``DataCollatorForSeq2SeqWithAudio`` over deferred-mel samples): inside its own sample a clip was
            # zero-padded as a WAVEFORM to ``audio_pad_frames`` frames (those frames hold the log-mel of silence, hf
            # feature_extraction_whisper.py:296-303); beyond that the reference collator pads the MEL with literal 0.0
            # (ref ultravox_processing.py:49-52).  Padding content is observable through the conv stem (SURVEY 7).
            lim = audio_pad_frames.to(dev).view(-1, 1) + 1                      # +1: guard row
            keep = torch.arange(t_full + 2, device=dev).view(1, -1) < lim
            tm = tm * keep.unsqueeze(-1).to(tm.dtype)
        plan, _ = frame_chunks(audio_num_frames.tolist(), context)
        if len(plan) == tm.shape[0] and t_full <= context:
            return tm                                                             # one chunk per clip: nothing to cut
        width = context if any(p[3] for p in plan) else min(t_full, context)
        out = torch.zeros(len(plan), width + 2, n_mels, dtype=BF16, device=dev)
        for i, (clip, off, _, cont) in enumerate(plan):
            n = min(width, t_full - off)
            out[i, 1:1 + n] = tm[clip, 1 + off:1 + off + n]
        return out

    def _prepare_audio_embeds(self, input_ids, audio_values=None, audio_token_start_idx=None, audio_lens=None,
                              audio_token_len=None, audio_batch_size=None, audio_tm=None) -> torch.Tensor:
        """Embedding gather + audio splice (ref :354-396).  Returns the spliced ``inputs_embeds`` [B, S, D]."""
        assert (audio_token_start_idx is not None and audio_token_len is not None and audio_lens is not None
                and audio_batch_size is not None), \
            "inputs_embeds/audio_values/audio_token_start_idx/audio_token_len/audio_lens/audio_batch_size must be provided."
        n = audio_values.shape[0] if audio_values is not None else audio_tm.shape[0]
        assert len(audio_token_start_idx) == len(audio_token_len) == len(audio_lens) == n, \
            "audio_token_start_idx/audio_token_len/audio_lens/audio_values must have the same batch size."
        assert len(audio_batch_size) == len(input_ids), "audio_batch_size and inputs_embeds must have the same batch size."
        dev = self.device
        if audio_tm is None:
            audio_tm = ops.mel_to_timemajor(audio_values.to(dev, torch.float32))
        enc = self.encode_audio(audio_tm, audio_lens)
        aud = self.project_audio(enc)
        B, S = input_ids.shape
        src = ops.splice_plan(audio_token_start_idx.to(dev, torch.int64).contiguous(),
                              audio_token_len.to(dev, torch.int32).contiguous(),
                              audio_batch_size.to(dev, torch.int64).reshape(-1).contiguous(), B, S, aud.shape[1])
        return ops.embed_splice(input_ids, self.language_model.model.embed_tokens.weight, aud, src)

    # -- llama ---------------------------------------------------------------------------------------
    def llama_hidden(self, inputs_embeds: torch.Tensor, cache: Optional[KVCache] = None,
                     kv_len: Optional[torch.Tensor] = None, kv_start: Optional[torch.Tensor] = None,
                     positions: Optional[torch.Tensor] = None) -> torch.Tensor:
        """All decoder layers + final RMSNorm (hf:models/llama/modeling_llama.py:355-426).  ``inputs_embeds`` [B,S,D]
        is consumed in place (it becomes the residual stream).  ``kv_len`` / ``kv_start`` [B] int32 bound each sequence's visible
        keys to [kv_start, kv_len) (right / left padding, hf:masking_utils padding mask); ``positions`` [B*S] int32 overrides
        the RoPE position of every row (mask-derived ``position_ids`` of left-padded generation, hf:generation/utils.py:707-729)."""
        lm, tc = self.language_model, self.config.text_config
        B, S, Dm = inputs_embeds.shape
        nq, nkv, hd = tc.num_attention_heads, tc.num_key_value_heads, lm.head_dim
        eps = tc.rms_norm_eps
        dev = inputs_embeds.device
        past = cache.length if cache is not None else 0
        cos, sin = self._rope_tables(past + S)
        h = inputs_embeds.view(B * S, Dm)
        x = torch.empty_like(h)
        qkv = torch.empty(B * S, (nq + 2 * nkv) * hd, dtype=BF16, device=dev)
        att = torch.empty(B * S, nq * hd, dtype=BF16, device=dev)
        ffn = tc.intermediate_size
        tiled = self._tiled_weights()
        if USE_WS and B * S > 256:
            tiled = None            # the 128-row images belong to the single-pass GEMM form (rows <= 256); larger batches read the row-major weights
        fuse_act = tiled is not None and tiled[0]["gate_up"].swiglu
        gu = None if fuse_act else torch.empty(B * S, 2 * ffn, dtype=BF16, device=dev)
        act = torch.empty(B * S, ffn, dtype=BF16, device=dev)
        rs = qkv.stride(0)
        layers = lm.model.layers
        # RoPE rides in the q|k|v GEMM epilogue when a head is one 128-wide tile; same positions rule as uvx_rope
        rope = (cos, sin, positions, S, past, (nq + nkv) * hd) if (FUSE_ROPE and QKV_MODE == "fused" and hd == 128) else None
        qkv_flags = 1 if QKV_MODE == "r1" else 0
        ops.rmsnorm(h, layers[0].input_layernorm.weight, eps, out=x)
        for li, layer in enumerate(layers):
            sa, mlp = layer.self_attn, layer.mlp
            tw = tiled[li] if tiled is not None else None
            if tw is not None and tw["qkv"] is not None:
                ops.linear_tiled(x, tw["qkv"], out=qkv, rope=rope, flags=ops.GEMM_W_STATIC)
            else:
                ops.linear(x, sa.qkv_w, out=qkv, rope=rope, flags=qkv_flags)
            if rope is None:
                ops.rope_(qkv, nq, nkv, hd, cos, sin, rows_per_seq=S, pos_offset=past, positions=positions)
            if cache is None:
                ops.attention_fused_qkv(qkv, B, S, nq, nkv, hd, hd ** -0.5, True, kv_len, 0, out=att, kv_start=kv_start)
            else:
                kc, vc = cache.k[li], cache.v[li]            # [B, S_max, Hkv, D]
                ops.kv_write(qkv, kc, vc, B, S, past, nq, nkv, hd)
                smax = kc.shape[1]
                ops.attention(qkv.data_ptr(), kc.data_ptr(), vc.data_ptr(), att, B, nq, nkv, S, past + S, hd,
                              (rs, S * rs, nkv * hd, smax * nkv * hd, nkv * hd, smax * nkv * hd, nq * hd, S * nq * hd),
                              hd ** -0.5, True, kv_len, 0, kv_start)
            # o_proj / down_proj write the residual stream AND the RMSNorm the next block reads (fused into split-K's pass 2)
            n1 = (layer.post_attention_layernorm.weight, eps, x) if FUSE_NORM else None
            if tw is not None and tw["o"] is not None:
                ops.linear_tiled(att, tw["o"], residual=h, out=h, norm=n1, flags=ops.GEMM_W_STATIC)
            else:
                ops.linear(att, sa.o_proj.weight, residual=h, out=h, norm=n1)
            if not FUSE_NORM:
                ops.rmsnorm(h, layer.post_attention_layernorm.weight, eps, out=x)
            if fuse_act:
                ops.linear_tiled(x, tw["gate_up"], out=act, act=ops.ACT_SWIGLU, flags=ops.GEMM_W_STATIC)   # silu(gate) * up from the accumulators
            else:
                if tw is not None:
                    ops.linear_tiled(x, tw["gate_up"], out=gu, flags=ops.GEMM_W_STATIC)
                else:
                    ops.linear(x, mlp.gate_up_w, out=gu)
                ops.swiglu(gu, gate_first=True, out=act)
            nxt = layers[li + 1].input_layernorm.weight if li + 1 < len(layers) else lm.model.norm.weight
            n2 = (nxt, eps, x) if FUSE_NORM else None
            if tw is not None and tw["down"] is not None:
                ops.linear_tiled(act, tw["down"], residual=h, out=h, norm=n2, flags=ops.GEMM_W_STATIC)
            else:
                ops.linear(act, mlp.down_proj.weight, residual=h, out=h, norm=n2)
            if not FUSE_NORM:
                ops.rmsnorm(h, nxt, eps, out=x)
        if cache is not None:
            cache.length = past + S
        return x.view(B, S, Dm)

    def load_state_dict(self, state_dict, strict: bool = True, _track: bool = True, **kwargs):
        """Accepts the reference's checkpoints as they are saved: the diff checkpoint of ``save_pretrained`` (projector + kept
        keys only - the towers' keys may be missing, ``_keys_to_ignore_on_load_missing``), plain full state dicts, or
        PEFT-wrapped names with LoRA adapters on the encoder / LLM projections (ref training/model_types.py:300-333) - the
        adapters are folded into the base weights.  Loaded keys are remembered in ``keep_params`` like the reference's pre-load
        hook does (ref :593-594), so ``diff_state_dict`` / ``save_pretrained`` write them back out."""
        import re
        from . import lora
        if lora.has_lora_keys(state_dict):
            scaling = {"audio_tower": lora.lora_scaling(getattr(self.config, "audio_model_lora_config", None)),
                       "language_model": lora.lora_scaling(getattr(self.config, "text_model_lora_config", None))}
            state_dict = lora.merge_lora_state_dict(state_dict, scaling)
        if self.language_model.tied and "language_model.lm_head.weight" not in state_dict \
                and "language_model.model.embed_tokens.weight" in state_dict:
            state_dict = dict(state_dict)
            state_dict["language_model.lm_head.weight"] = state_dict["language_model.model.embed_tokens.weight"]
        if _track:
            self.keep_params.update(state_dict.keys())
        res = super().load_state_dict(state_dict, strict=False, **kwargs)
        ignorable = [re.compile(p.replace(".", r"\.").replace("*", ".*")) for p in self._keys_to_ignore_on_load_missing]
        missing = [k for k in res.missing_keys if not any(r.match(k) for r in ignorable)]
        if strict and (missing or res.unexpected_keys):
            raise RuntimeError(f"Error(s) in loading state_dict for UltravoxModel: missing keys {missing}, "
                               f"unexpected keys {list(res.unexpected_keys)}")
        res.missing_keys[:] = missing
        self._wT = None
        self._tiled = None
        return res

    def new_cache(self, batch: int, max_len: int) -> KVCache:
        tc, lm = self.config.text_config, self.language_model
        shape = (tc.num_hidden_layers, batch, max_len, tc.num_key_value_heads, lm.head_dim)
        return KVCache(torch.empty(shape, dtype=BF16, device=self.device), torch.empty(shape, dtype=BF16, device=self.device))

    @staticmethod
    def _pad_bounds(attention_mask: Optional[torch.Tensor]):
        """attention_mask [B,S] with one contiguous run of ones per row -> (kv_start, kv_len) int32 [B] (None where the
        bound is trivial).  Right padding (training collator, ref ultravox_processing.py:43-51) gives kv_len, left padding
        (inference collator / ``tokenizer.padding_side = "left"``, ref :53-63, infer.py:155-180) gives kv_start."""
        if attention_mask is None:
            return None, None
        m = attention_mask.to(torch.bool)
        if bool(m.all()):
            return None, None
        S = m.shape[1]
        ar = torch.arange(S, device=m.device)[None, :]
        n = m.sum(-1)
        start = torch.where(n > 0, m.to(torch.int64).argmax(-1), torch.zeros_like(n))
        end = start + n
        if not torch.equal(m, (ar >= start[:, None]) & (ar < end[:, None])):
            raise NotImplementedError("attention_mask rows must be one contiguous run of ones (left and/or right padding)")
        kv_start = start.to(torch.int32) if bool((start > 0).any()) else None
        kv_len = end.to(torch.int32) if bool((end < S).any()) else None
        return kv_start, kv_len

    def attach_encoder_lora(self, r: int = 8, alpha: float = 8.0, seed: int = 0):
        """``apply_lora(audio_tower, audio_model_lora_config)`` (ref :496, :690-709) for the released recipes' ``r: 8`` on q_proj /
        k_proj: registers ``autograd.EncoderLora`` as ``self.encoder_lora`` with trainable parameters; ``forward`` with gradients
        enabled then routes the encoder through ``EncoderLoraFn`` so ``loss.backward()`` fills their ``.grad``."""
        from .autograd import EncoderLora
        self.encoder_lora = EncoderLora(self, r=r, alpha=alpha, seed=seed)
        for p in self.encoder_lora.parameters():
            p.requires_grad_(True)
        return self.encoder_lora

    # -- forward / generate --------------------------------------------------------------------------
    def forward(self, input_ids: torch.Tensor, audio_values: Optional[torch.Tensor] = None,
                inputs_embeds: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None,
                attention_mask: Optional[torch.Tensor] = None, audio_token_start_idx: Optional[torch.Tensor] = None,
                audio_lens: Optional[torch.Tensor] = None, audio_token_len: Optional[torch.Tensor] = None,
                audio_batch_size: Optional[torch.Tensor] = None, past_key_values: Optional[KVCache] = None,
                alt_input_ids=None, alt_attention_mask=None, alt_labels=None, logits_to_keep: int = 0,
                audio_waveforms: Optional[torch.Tensor] = None, audio_num_frames: Optional[torch.Tensor] = None,
                audio_pad_frames: Optional[torch.Tensor] = None, **kwargs) -> CausalLMOutputWithPast:
        """Same signature and semantics as the reference ``forward`` (ref :277-352).  ``logits_to_keep=1`` computes
        only the last position's logits (the TTFT path, hf:modeling_llama.py:485-491)."""
        dev = self.device
        input_ids = input_ids.to(dev)
        has_audio = (audio_waveforms is not None and len(audio_waveforms) > 0) or (audio_values is not None and len(audio_values) > 0)
        # the training door (HF Trainer: model(**batch) -> loss.backward(), ref train.py:250-330): gradients are enabled, a
        # projector parameter wants one and the loss depends on it -> the forward is built from autograd.Functions
        grad_path = (torch.is_grad_enabled() and labels is not None and inputs_embeds is None and has_audio
                     and past_key_values is None and hasattr(self, "multi_modal_projector")
                     and any(p.requires_grad for p in self.multi_modal_projector.parameters()))
        if grad_path:
            with torch.no_grad():
                if audio_waveforms is not None and len(audio_waveforms) > 0:
                    tm = self.mel_chunks_from_waveforms(audio_waveforms, audio_num_frames, audio_pad_frames=audio_pad_frames)
                else:
                    tm = ops.mel_to_timemajor(audio_values.to(dev, torch.float32))
                lora = getattr(self, "encoder_lora", None)
                if lora is None or not lora.A.requires_grad:
                    inputs_embeds = self.encode_audio(tm, audio_lens).clone()   # encoder output; the towers are frozen
            if lora is not None and lora.A.requires_grad:
                # encoder LoRA training through the autograd door: the adapters are autograd inputs of the encoder node
                from .autograd import EncoderLoraFn
                inputs_embeds = EncoderLoraFn.apply(self, tm, audio_lens, lora.A, lora.Bq, lora.Bk)
        elif inputs_embeds is None:
            inputs_embeds = self.prompt_embeds(input_ids, audio_values, audio_token_start_idx, audio_lens, audio_token_len,
                                               audio_batch_size, audio_waveforms, audio_num_frames, audio_pad_frames)
        else:
            inputs_embeds = inputs_embeds.clone()
        if self.training and self.loss_config.loss_function not in (LossFunction.CrossEntropy, LossFunction.KL_Divergence):
            raise ValueError(f"Unsupported loss function: {self.loss_config.loss_function}")
        if grad_path:
            return self._forward_with_grad(input_ids, inputs_embeds, labels, attention_mask, audio_token_start_idx,
                                           audio_token_len, audio_batch_size, alt_input_ids, alt_labels, logits_to_keep)
        kv_start, kv_len = self._pad_bounds(attention_mask.to(dev) if attention_mask is not None else None)
        position_ids = kwargs.get("position_ids")
        positions = position_ids.to(dev, torch.int32).reshape(-1).contiguous() if position_ids is not None else None
        hidden = self.llama_hidden(inputs_embeds, past_key_values, kv_len, kv_start, positions)
        B, S, Dm = hidden.shape
        lm_w = self.language_model.lm_head.weight
        if logits_to_keep == 1:
            logits = ops.lm_head(hidden[:, -1, :], lm_w).view(B, 1, -1)
        else:
            logits = ops.linear(hidden.view(B * S, Dm), lm_w, out_dtype=torch.float32).view(B, S, -1)
        loss = None
        if labels is not None:
            from .losses import causal_lm_loss
            loss = causal_lm_loss(logits, labels.to(dev), self.config.ignore_index)
        if self.training and self.loss_config.loss_function == LossFunction.KL_Divergence:
            loss = self._compute_kl_loss(logits, labels, alt_input_ids, alt_labels)
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=past_key_values)

    def prompt_embeds(self, input_ids: torch.Tensor, audio_values: Optional[torch.Tensor] = None,
                      audio_token_start_idx: Optional[torch.Tensor] = None, audio_lens: Optional[torch.Tensor] = None,
                      audio_token_len: Optional[torch.Tensor] = None, audio_batch_size: Optional[torch.Tensor] = None,
                      audio_waveforms: Optional[torch.Tensor] = None, audio_num_frames: Optional[torch.Tensor] = None,
                      audio_pad_frames: Optional[torch.Tensor] = None, **kwargs) -> torch.Tensor:
        """The spliced ``inputs_embeds`` [B, S, D] that ``forward`` feeds the LLM: log-mel (for waveforms), encoder, projector,
        token embeddings and the audio splice; token embeddings alone without audio."""
        input_ids = input_ids.to(self.device)
        if audio_waveforms is not None and len(audio_waveforms) > 0:
            tm = self.mel_chunks_from_waveforms(audio_waveforms, audio_num_frames, audio_pad_frames=audio_pad_frames)
            return self._prepare_audio_embeds(input_ids, None, audio_token_start_idx, audio_lens, audio_token_len, audio_batch_size,
                                              audio_tm=tm)
        if audio_values is not None and len(audio_values) > 0:
            return self._prepare_audio_embeds(input_ids, audio_values, audio_token_start_idx, audio_lens, audio_token_len,
                                              audio_batch_size)
        return ops.embed_splice(input_ids, self.language_model.model.embed_tokens.weight, None, None)

    def _forward_with_grad(self, input_ids, enc, labels, attention_mask, audio_token_start_idx, audio_token_len,
                           audio_batch_size, alt_input_ids, alt_labels, logits_to_keep) -> CausalLMOutputWithPast:
        """``forward`` for training: loss carries a grad_fn through ProjectorFn / SpliceFn / LlamaStackFn / HeadLossFn
        (``autograd.py``), so ``out.loss.backward()`` fills ``multi_modal_projector.*.grad``; logits are returned like the
        reference does (all rows, fp32, detached - computed outside the graph)."""
        from . import autograd as ag
        dev = self.device
        assert audio_token_start_idx is not None and audio_token_len is not None and audio_batch_size is not None, \
            "inputs_embeds/audio_values/audio_token_start_idx/audio_token_len/audio_lens/audio_batch_size must be provided."
        kv_start, kv_len = self._pad_bounds(attention_mask.to(dev) if attention_mask is not None else None)
        if kv_start is not None:
            raise NotImplementedError("training batches are right-padded (ref ultravox_processing.py:43-51); left padding is for generation")
        if self.training and self.loss_config.loss_function == LossFunction.KL_Divergence and (alt_input_ids is None or alt_labels is None):
            raise ValueError("labels must be provided")
        kl = self.training and self.loss_config.loss_function == LossFunction.KL_Divergence
        prev = self.loss_config
        if not kl and prev.loss_function != LossFunction.CrossEntropy:
            self.loss_config = LossConfig()               # eval-mode forward with grad enabled: CE, like the reference (:335-338)
        try:
            loss, hidden = ag.adapter_loss(self, input_ids, enc, (audio_token_start_idx, audio_token_len, audio_batch_size),
                                           labels.to(dev), alt_input_ids if kl else None, alt_labels if kl else None, kv_len)
        finally:
            self.loss_config = prev
        B, S, Dm = hidden.shape
        with torch.no_grad():
            lm_w = self.language_model.lm_head.weight
            if logits_to_keep == 1:
                logits = ops.lm_head(hidden[:, -1, :], lm_w).view(B, 1, -1)
            else:
                logits = ops.linear(hidden.reshape(B * S, Dm), lm_w, out_dtype=torch.float32).view(B, S, -1)
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=None)

    def _compute_kl_loss(self, logits: torch.Tensor, labels, alt_input_ids, alt_labels) -> torch.Tensor:
        """ref :202-257: teacher = this LLM on the text-only ``alt_*`` twin (no grad), KL at ``kl_temperature`` on the
        prediction rows + ``eot_loss_weight`` x KL on the EOT rows."""
        from .losses import kl_distill_loss, prediction_rows
        if labels is None or alt_labels is None or alt_input_ids is None:
            raise ValueError("labels must be provided")
        dev = self.device
        rows, is_eot = prediction_rows(labels, self.config.ignore_index)
        t_rows, _ = prediction_rows(alt_labels, self.config.ignore_index)
        V = logits.shape[-1]
        student = logits.reshape(-1, V).index_select(0, rows.to(dev)).contiguous()
        with torch.no_grad():
            emb = ops.embed_splice(alt_input_ids.to(dev), self.language_model.model.embed_tokens.weight, None, None)
            hid = self.llama_hidden(emb).view(-1, emb.shape[-1])
            teacher = ops.linear(ops.gather_rows(hid, t_rows.to(dev, torch.int32)), self.language_model.lm_head.weight,
                                 out_dtype=torch.float32)
        return kl_distill_loss(student, teacher, is_eot, self.loss_config.kl_temperature, self.loss_config.eot_loss_weight)

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, audio_values: Optional[torch.Tensor] = None,
                 inputs_embeds: Optional[torch.Tensor] = None, audio_token_start_idx=None, audio_lens=None,
                 audio_token_len=None, audio_batch_size=None, max_new_tokens: int = 20, eos_token_id=None,
                 attention_mask: Optional[torch.Tensor] = None, past_key_values: Optional[KVCache] = None,
                 return_dict_in_generate: bool = False, streamer=None, pad_token_id: Optional[int] = None,
                 repetition_penalty: float = 1.0, temperature: Optional[float] = None, do_sample: bool = False,
                 top_k: Optional[int] = None, top_p: Optional[float] = None, generator: Optional[torch.Generator] = None,
                 audio_waveforms: Optional[torch.Tensor] = None, audio_num_frames: Optional[torch.Tensor] = None,
                 audio_pad_frames: Optional[torch.Tensor] = None, use_graph: bool = True, num_beams: int = 1,
                 length_penalty: float = 1.0, early_stopping=False, num_return_sequences: int = 1, output_scores: bool = False,
                 **kwargs):
        """``GenerationMixin.generate`` for this model (ref :398-426; arguments as ``LocalInference._generate`` passes them, ref
        infer.py:309-342).  Returns prompt ids followed by the new tokens.

        Greedy when ``do_sample`` is false (the reference's default: temperature None / 0, ref infer.py:319-328); with
        ``do_sample=True`` tokens are drawn from softmax(logits / temperature) over the ``top_k`` largest logits (HF
        ``GenerationConfig`` defaults: temperature 1.0, top_k 50), reproducibly for a seeded ``generator``.  ``top_p < 1``
        then keeps the nucleus of that distribution, as HF's ``TopPLogitsWarper`` after ``TopKLogitsWarper``: the smallest
        set of largest logits whose probability exceeds ``top_p`` (always the largest one, so ``top_p=0`` is greedy; a tie
        group at the cut is kept whole).  ``top_p`` must lie in [0, 1] (``ValueError`` otherwise); it is ignored when not
        sampling, and ``None`` or 1.0 means no nucleus filter.
        ``past_key_values``: conversation KV reuse (ref infer.py:126-148): the cache already holds the first
        ``past_key_values.length`` positions of ``input_ids`` (earlier turns incl. the reply), so only the new suffix is
        embedded, spliced and prefilled; ``return_dict_in_generate=True`` hands the cache back for the next turn.
        ``streamer``: object with ``put(tensor)`` / ``end()`` (transformers' streamer protocol: the prompt first, then one
        call per new token).  Rows that have produced an EOS keep emitting ``pad_token_id`` (default: the first EOS id).

        The prompt is prefilled by the tensor-core path; every later token is one replay of a CUDA graph holding the whole
        decode step (``engine.DecodeEngine``: GEMV linears, device-side positions / EOS / sequence bookkeeping), so the loop
        has no per-token host synchronisation unless a streamer asks for the token.

        ``num_beams > 1`` runs beam search as hf:generation/utils.py ``_beam_search`` does (the reference passes the argument
        through to ``language_model.generate``, ref :398-426): log-probs, ``repetition_penalty`` applied to them, the top
        ``max(2, 1 + #EOS) * num_beams`` continuations per prompt, hypotheses scored ``sum log-prob / generated_len **
        length_penalty``, ``early_stopping`` in {False, True, "never"}.  Each prompt is prefilled once and its cache rows are
        broadcast to its beams; every later step is one graph replay (``engine.BeamDecodeEngine``).  Returns the best
        ``num_return_sequences`` hypotheses per prompt, [B * num_return_sequences, S + longest], filled past each one's end with
        ``pad_token_id`` (or the first EOS id when that is unset or 0).  With ``return_dict_in_generate=True`` and
        ``output_scores=True`` their scores are in ``sequences_scores``; ``past_key_values`` is None, because the cache rows
        belong to the running beams, not to the returned hypotheses.  Not built: beam sampling (``do_sample=True``), a
        streamer, conversation KV reuse and per-step ``scores`` / ``beam_indices``."""
        from .engine import DecodeEngine
        unknown = [k for k, v in kwargs.items() if isinstance(v, torch.Tensor)]
        if unknown:
            raise TypeError(f"generate() got unexpected tensor arguments {unknown}")
        if not isinstance(num_beams, int) or not 1 <= num_beams <= ops.BEAM_MAX:
            raise ValueError(f"num_beams must be an integer in [1, {ops.BEAM_MAX}], got {num_beams!r}")
        if not isinstance(num_return_sequences, int) or not 1 <= num_return_sequences <= num_beams:
            raise ValueError(f"num_return_sequences ({num_return_sequences!r}) must be in [1, num_beams = {num_beams}]")
        if num_beams > 1:
            if do_sample:
                raise NotImplementedError("beam sampling (num_beams > 1 with do_sample=True) is not built")
            if streamer is not None:
                raise ValueError("`streamer` cannot be used with beam search (yet!). Make sure that `num_beams` is set to 1.")
            if past_key_values is not None:
                raise NotImplementedError("conversation KV reuse with beam search is not built")
            if early_stopping not in (False, True, "never"):
                raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")
        if top_p is not None and not 0.0 <= float(top_p) <= 1.0:       # NaN fails too
            raise ValueError(f"`top_p` has to be a float in [0, 1], but is {top_p}")
        sampling = bool(do_sample) and (temperature is None or float(temperature) > 0)
        temp = (1.0 if temperature is None else float(temperature)) if sampling else 0.0
        k_top = (50 if top_k is None else int(top_k)) if sampling else 0
        p_top = float(top_p) if sampling and top_p is not None else 1.0
        dev = self.device
        input_ids = input_ids.to(dev)
        B, S = input_ids.shape
        # left-padded batches (ref infer.py:155-180 batches prompts with padding_side="left"): keys in the padding are masked
        # for the whole generation and RoPE positions count real tokens only (hf:generation/utils.py:707-729)
        kv_start = None
        position_ids = None
        if attention_mask is not None and not bool(attention_mask.to(torch.bool).all()):
            am = attention_mask.to(dev)
            kv_start, kv_len = self._pad_bounds(am)
            if kv_len is not None:
                raise NotImplementedError("generate() needs left padding (or none); right-padded prompts cannot be continued")
            if past_key_values is not None:
                raise NotImplementedError("conversation KV reuse with padded batches (the reference has none either, infer.py:155)")
            position_ids = (am.to(torch.int64).cumsum(-1) - 1).clamp_min(0)
        if num_beams > 1:
            seqs, scores = self._beam_search(
                input_ids, dict(audio_values=audio_values, inputs_embeds=inputs_embeds, attention_mask=attention_mask,
                                audio_token_start_idx=audio_token_start_idx, audio_lens=audio_lens, audio_token_len=audio_token_len,
                                audio_batch_size=audio_batch_size, position_ids=position_ids, audio_waveforms=audio_waveforms,
                                audio_num_frames=audio_num_frames, audio_pad_frames=audio_pad_frames),
                kv_start, max_new_tokens, eos_token_id, pad_token_id, num_beams, length_penalty, early_stopping,
                num_return_sequences, repetition_penalty or 1.0, use_graph)
            if return_dict_in_generate:
                return GenerateOutput(seqs, None, scores if output_scores else None)
            return seqs
        has_wave = audio_waveforms is not None and len(audio_waveforms) > 0
        has_mel = audio_values is not None and len(audio_values) > 0
        if past_key_values is None:
            cache = self.new_cache(B, S + max_new_tokens)
            out = self.forward(input_ids, audio_values, inputs_embeds, None, attention_mask, audio_token_start_idx, audio_lens,
                               audio_token_len, audio_batch_size, cache, logits_to_keep=1, position_ids=position_ids,
                               audio_waveforms=audio_waveforms, audio_num_frames=audio_num_frames, audio_pad_frames=audio_pad_frames)
        else:
            P = past_key_values.length
            if not (0 <= P < S) or past_key_values.k.shape[1] != B:
                raise ValueError(f"past_key_values holds {P} positions for batch {past_key_values.k.shape[1]}; the prompt has "
                                 f"{S} tokens for batch {B} - it must extend the cached prefix")
            cache = past_key_values.grown(S + max_new_tokens)
            if inputs_embeds is None:                       # embed + splice the whole prompt, prefill only the new suffix
                if has_wave:
                    tm = self.mel_chunks_from_waveforms(audio_waveforms, audio_num_frames, audio_pad_frames=audio_pad_frames)
                    inputs_embeds = self._prepare_audio_embeds(input_ids, None, audio_token_start_idx, audio_lens,
                                                               audio_token_len, audio_batch_size, audio_tm=tm)
                elif has_mel:
                    inputs_embeds = self._prepare_audio_embeds(input_ids, audio_values, audio_token_start_idx, audio_lens,
                                                               audio_token_len, audio_batch_size)
                else:
                    inputs_embeds = ops.embed_splice(input_ids, self.language_model.model.embed_tokens.weight, None, None)
            out = self.forward(input_ids[:, P:], None, inputs_embeds[:, P:].contiguous(), past_key_values=cache, logits_to_keep=1)
        eos = sorted(set([eos_token_id] if isinstance(eos_token_id, int) else (eos_token_id or [])))
        pad_id = pad_token_id if pad_token_id is not None else (min(eos) if eos else 0)
        eng = DecodeEngine(self, B, cache.capacity, use_graph=use_graph, cache=cache, eos_token_ids=eos, pad_token_id=pad_id,
                           temperature=temp, top_k=k_top, top_p=p_top, repetition_penalty=repetition_penalty or 1.0,
                           generator=generator)
        if streamer is not None:
            streamer.put(input_ids)
        tok = eng.begin(input_ids, out.logits.view(B, -1), kv_start)
        n_new = 1
        sync_every = 8          # without a streamer the host looks at the all-done flag every few tokens only
        while True:
            if streamer is not None:
                streamer.put(tok.clone())
            stop = n_new >= max_new_tokens
            if not stop and eos and (streamer is not None or n_new % sync_every == 0):
                stop = bool(int(eng.all_done))
            if stop:
                break
            eng.step()
            n_new += 1
        if streamer is not None:
            streamer.end()
        new = eng.seq[:, S:S + n_new]
        if eos and streamer is None and n_new > 1:
            # the loop may have run a few tokens past the step at which every row had finished: HF stops right there
            hit = torch.isin(new, eng.eos)
            first = torch.where(hit.any(-1), hit.to(torch.int32).argmax(-1), torch.full((B,), n_new, device=dev))
            n_new = min(n_new, int(first.max()) + 1)
            new = new[:, :n_new]
        cache.length = S + n_new - 1                        # the last new token has not been fed yet
        sequences = torch.cat([input_ids, new], dim=1)
        return GenerateOutput(sequences, cache) if return_dict_in_generate else sequences

    def _beam_search(self, input_ids: torch.Tensor, forward_kw: dict, kv_start: Optional[torch.Tensor], max_new_tokens: int,
                     eos_token_id, pad_token_id: Optional[int], num_beams: int, length_penalty: float, early_stopping,
                     num_return_sequences: int, repetition_penalty: float, use_graph: bool, step_hook=None):
        """``generate``'s beam branch -> (sequences [B * num_return_sequences, S + longest], their scores).  The B prompts are
        prefilled once into cache rows b * num_beams (a view of the [L, B * num_beams, S_max, ...] cache as B rows of
        num_beams * S_max positions).  ``step_hook(engine)``, if given, runs after every beam step (the host then checks
        the done flag every step)."""
        from .engine import BeamDecodeEngine
        B, S = input_ids.shape
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        eos_list = [eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id or [])
        cache = self.new_cache(B * num_beams, S + max_new_tokens)
        L, _, smax, hkv, hd = cache.k.shape
        prompt_rows = KVCache(cache.k.view(L, B, num_beams * smax, hkv, hd), cache.v.view(L, B, num_beams * smax, hkv, hd))
        fk = dict(forward_kw)
        out = self.forward(input_ids, fk.pop("audio_values"), fk.pop("inputs_embeds"), None, fk.pop("attention_mask"),
                           fk.pop("audio_token_start_idx"), fk.pop("audio_lens"), fk.pop("audio_token_len"),
                           fk.pop("audio_batch_size"), prompt_rows, logits_to_keep=1, **fk)
        eng = BeamDecodeEngine(self, B, num_beams, cache.capacity, max_new_tokens, use_graph=use_graph, cache=cache,
                               eos_token_ids=eos_list, length_penalty=length_penalty, early_stopping=early_stopping,
                               repetition_penalty=repetition_penalty)
        eng.begin(input_ids, out.logits.view(B, -1), kv_start)
        n_new = 1
        sync_every = 8          # the host looks at the device's done flag every few steps only
        while True:
            if step_hook is not None:
                step_hook(eng)
            stop = n_new >= max_new_tokens
            if not stop and (step_hook is not None or n_new % sync_every == 0):
                stop = bool(int(eng.all_done))
            if stop:
                break
            eng.step()
            n_new += 1
        # hf:generation/utils.py _beam_search: `pad_token_id or eos_token_id[0] if eos_token_id is not None else -1`, with the
        # pad id defaulting to the first EOS id
        fill = (pad_token_id if pad_token_id else eos_list[0]) if eos_list else -1
        return eng.result(S, num_return_sequences, fill)


class SwiGLU(nn.Module):
    """``silu(gate) * x`` with ``x, gate = chunk(2, -1)`` (ref ultravox_model.py:739-742), as the module the reference registers
    under ``ACT2FN["swiglu"]``; runs ``uvx_swiglu`` (CUDA bf16 only - there is no CPU fallback)."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return ops.swiglu(x, gate_first=False)


def apply_repetition_penalty(logits: torch.Tensor, sequences: torch.Tensor, penalty: float) -> torch.Tensor:
    """CTRL-style penalty on every token already in ``sequences`` ([B, T] ids): positive scores are divided by ``penalty``,
    negative ones multiplied (hf:generation/logits_process.py ``RepetitionPenaltyLogitsProcessor``, which the reference's
    pipeline enables with 1.1, ref ultravox_pipeline.py:95-113).  Plain tensor ops on the [B, V] logits of one step."""
    if penalty == 1.0:
        return logits
    seen = torch.gather(logits, 1, sequences)
    seen = torch.where(seen < 0, seen * penalty, seen / penalty)
    return logits.scatter(1, sequences, seen)


def _sinusoids(length: int, channels: int, max_timescale: float = 10000.0) -> torch.Tensor:
    """Whisper's fixed positional table (hf:models/whisper/modeling_whisper.py:55-65)."""
    import math
    inc = math.log(max_timescale) / (channels // 2 - 1)
    inv = torch.exp(-inc * torch.arange(channels // 2))
    t = torch.arange(length).view(-1, 1) * inv.view(1, -1)
    return torch.cat([t.sin(), t.cos()], dim=1)


# -- registration with the transformers Auto* machinery, as the reference does at import time (ref ultravox_model.py:997-1003)
def _register_with_transformers() -> None:
    import transformers
    from transformers.activations import ACT2FN
    transformers.AutoConfig.register("ultravox", UltravoxConfig, exist_ok=True)
    transformers.AutoModel.register(UltravoxConfig, UltravoxModel, exist_ok=True)
    try:
        ACT2FN["swiglu"] = SwiGLU
    except TypeError:                        # ClassInstantier of older transformers takes (class, kwargs) tuples as well
        ACT2FN["swiglu"] = (SwiGLU, {})


_register_with_transformers()
