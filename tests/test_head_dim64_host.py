# -*- coding: utf-8 -*-
"""Head-dim-64 models on the host: Llama-3 RoPE scaling against transformers, geometry() of the Llama-3.2-1B,
TinyLlama and Qwen2.5-0.5B configs, the Llama-3.2-1B module tree, and the refusal of a config whose head_dim differs
from hidden_size // num_attention_heads.  No GPU needed."""
import pytest
import torch


def llama32_1b_config(**over):
    from transformers import LlamaConfig
    kw = dict(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16,
              num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=131072, rms_norm_eps=1e-5,
              rope_theta=500000.0, tie_word_embeddings=True, bos_token_id=128000, eos_token_id=128001,
              rope_scaling={'rope_type': 'llama3', 'factor': 32.0, 'low_freq_factor': 1.0, 'high_freq_factor': 4.0,
                            'original_max_position_embeddings': 8192})
    kw.update(over)
    return LlamaConfig(**kw)


# the rope tables depend on the head geometry and the RoPE parameters only: one small layer on the CPU
SMALL = dict(num_hidden_layers=1, vocab_size=64, intermediate_size=128)


def tinyllama_config():
    from transformers import LlamaConfig
    return LlamaConfig(vocab_size=32000, hidden_size=2048, intermediate_size=5632, num_hidden_layers=22,
                       num_attention_heads=32, num_key_value_heads=4, max_position_embeddings=2048, rms_norm_eps=1e-5,
                       rope_theta=10000.0, tie_word_embeddings=False)


def qwen25_05b_config():
    from transformers import Qwen2Config
    return Qwen2Config(vocab_size=151936, hidden_size=896, intermediate_size=4864, num_hidden_layers=24,
                       num_attention_heads=14, num_key_value_heads=2, max_position_embeddings=32768, rms_norm_eps=1e-6,
                       rope_theta=1000000.0, use_sliding_window=False, tie_word_embeddings=True)


def test_rope_tables_follow_transformers_llama3():
    """rope_type llama3 (Llama-3.2-1B: factor 32, low 1, high 4, original 8192, theta 5e5): cos / sin equal
    LlamaRotaryEmbedding's bf16 output bit for bit for positions 0..4095"""
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = llama32_1b_config(**SMALL)
    cos, sin = LlamaForCausalLM(cfg, device='cpu').rope_tables(4096)
    x = torch.zeros((1, 4096, 64), dtype=torch.bfloat16)
    hc, hs = LlamaRotaryEmbedding(cfg)(x, torch.arange(4096)[None])
    assert cos.shape == (4096, 32) and hc.dtype == torch.bfloat16
    assert torch.equal(hc[0, :, :32], hc[0, :, 32:])
    assert torch.equal(cos, hc[0, :, :32]) and torch.equal(sin, hs[0, :, :32])
    # the scaling really acts: the lowest frequencies are divided by 32, the highest are left alone
    plain = LlamaForCausalLM(llama32_1b_config(rope_scaling=None, **SMALL), device='cpu').rope_tables(4096)
    assert torch.equal(sin[:, 0], plain[1][:, 0])
    assert torch.allclose(sin[1:, -1].float() * 32, plain[1][1:, -1].float(), rtol=2 ** -6, atol=0)


def test_rope_parameters_of_transformers_5_are_read():
    """the same tables whether the llama3 parameters arrive as `rope_scaling` or as transformers-5 `rope_parameters`"""
    from transformers import LlamaConfig
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    a = llama32_1b_config(**SMALL)
    rp = dict(a.rope_parameters)
    b = LlamaConfig(**{k: v for k, v in a.to_dict().items() if k not in ('rope_scaling', 'rope_parameters')},
                    rope_parameters=rp)
    ta = LlamaForCausalLM(a, device='cpu').rope_tables(512)
    tb = LlamaForCausalLM(b, device='cpu').rope_tables(512)
    assert torch.equal(ta[0], tb[0]) and torch.equal(ta[1], tb[1])


@pytest.mark.parametrize('name,cfg,geo', [
    ('llama3.2-1b', llama32_1b_config, dict(n_layers=16, hidden=2048, n_q_heads=32, n_kv_heads=8, head_dim=64,
                                            inter=8192, vocab=128256)),
    ('tinyllama', tinyllama_config, dict(n_layers=22, hidden=2048, n_q_heads=32, n_kv_heads=4, head_dim=64,
                                         inter=5632, vocab=32000)),
    ('qwen2.5-0.5b', qwen25_05b_config, dict(n_layers=24, hidden=896, n_q_heads=14, n_kv_heads=2, head_dim=64,
                                             inter=4864, vocab=151936))])
def test_geometry_of_head_dim64_configs(name, cfg, geo):
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cls = Qwen2ForCausalLM if name.startswith('qwen') else LlamaForCausalLM
    assert cls(cfg(), device='meta').geometry() == geo


def test_module_tree_matches_transformers_llama32_1b():
    """the Llama-3.2-1B tree on the meta device: every HF parameter name and shape (the tied head included)"""
    from transformers import LlamaForCausalLM as HF
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = llama32_1b_config()
    with torch.device('meta'):
        hf = HF(cfg)
    ours = LlamaForCausalLM(cfg, device='meta')
    want = {k: tuple(v.shape) for k, v in hf.named_parameters(remove_duplicate=False)}
    got = {k: tuple(v.shape) for k, v in ours.named_parameters()}
    assert got == want
    assert got['model.layers.0.self_attn.k_proj.weight'] == (512, 2048)
    assert got['model.layers.0.self_attn.o_proj.weight'] == (2048, 2048)


def test_head_dim_other_than_hidden_over_heads_raises():
    """the fused projections are hidden_size // num_attention_heads wide per head: a config that sets another
    head_dim (e.g. 128 for 2048 / 32) is refused, naming both values"""
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = llama32_1b_config(num_hidden_layers=1, vocab_size=64, head_dim=128)
    with pytest.raises(ValueError, match=r'head_dim 128.*= 64'):
        LlamaForCausalLM(cfg, device='meta').geometry()


def test_yarn_still_raises_for_llama():
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = llama32_1b_config(rope_scaling={'rope_type': 'yarn', 'factor': 4.0, 'original_max_position_embeddings': 8192},
                            **SMALL)
    with pytest.raises(ValueError, match='yarn'):
        LlamaForCausalLM(cfg, device='cpu').rope_tables(64)
