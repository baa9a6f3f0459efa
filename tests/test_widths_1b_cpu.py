"""CPU checks behind the config-1 (Llama-3.2-1B, head_dim 64) per-op suite ``test_widths_1b_gpu.py``."""
import torch


def test_llama3_inv_freq_head_dim_64_matches_transformers():
    """``ops.llama3_inv_freq(64, ...)`` with the tiny_1b preset's theta and llama3 scaling equals transformers' llama3 RoPE
    init for a head_dim-64 Llama config, bit for bit (the tables the D = 64 RoPE, decode and prefill tests build on)."""
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS

    from ultravox_b200 import ops
    from ultravox_b200.config import PRESETS
    tc = PRESETS["tiny_1b"]["text_config"]
    assert tc["head_dim"] == 64
    cfg = LlamaConfig(hidden_size=tc["hidden_size"], num_attention_heads=tc["num_attention_heads"],
                      num_key_value_heads=tc["num_key_value_heads"], head_dim=tc["head_dim"],
                      max_position_embeddings=tc["max_position_embeddings"], rope_theta=tc["rope_theta"],
                      rope_scaling=tc["rope_scaling"])
    want, attention_scaling = ROPE_INIT_FUNCTIONS["llama3"](cfg, "cpu")
    got = ops.llama3_inv_freq(64, tc["rope_theta"], tc["rope_scaling"])
    assert attention_scaling == 1.0
    assert got.dtype == torch.float32 and got.shape == (32,)
    assert torch.equal(got, want.to(torch.float32))
