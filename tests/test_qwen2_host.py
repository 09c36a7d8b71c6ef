# -*- coding: utf-8 -*-
"""Qwen2 (HF model_type `qwen2`) on the host: module tree against transformers' Qwen2ForCausalLM, geometry, the fused
QKV bias, RoPE tables and the refusal of a GEMM set that would drop the bias.  No GPU needed."""
import pytest
import torch


def _qwen2_7b_config(**over):
    from transformers import Qwen2Config
    kw = dict(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
              num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=32768, rms_norm_eps=1e-6,
              rope_theta=1000000.0, sliding_window=131072, use_sliding_window=False, max_window_layers=28,
              tie_word_embeddings=False)
    kw.update(over)
    return Qwen2Config(**kw)


def test_module_tree_matches_transformers_qwen2():
    """the Qwen2-7B tree on the meta device: every HF parameter name and shape, q/k/v biases, no o / MLP / head bias"""
    from transformers import Qwen2ForCausalLM as HF
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cfg = _qwen2_7b_config()
    with torch.device('meta'):
        hf = HF(cfg)
    ours = Qwen2ForCausalLM(cfg, device='meta')
    want = {k: tuple(v.shape) for k, v in hf.named_parameters()}
    got = {k: tuple(v.shape) for k, v in ours.named_parameters()}
    assert got == want
    assert got['model.layers.0.self_attn.q_proj.bias'] == (3584,)
    assert got['model.layers.0.self_attn.k_proj.bias'] == (512,) and got['model.layers.0.self_attn.v_proj.bias'] == (512,)
    assert not any(k.endswith('o_proj.bias') or '.mlp.' in k and k.endswith('bias') for k in got)
    assert ours.geometry() == dict(n_layers=28, hidden=3584, n_q_heads=28, n_kv_heads=4, head_dim=128, inter=18944,
                                   vocab=152064)


def test_llama_tree_has_no_biases():
    from transformers import LlamaConfig
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=64, hidden_size=256, intermediate_size=256, num_hidden_layers=1,
                      num_attention_heads=2, num_key_value_heads=2)
    m = LlamaForCausalLM(cfg, device='cpu')
    assert not any(k.endswith('bias') for k, _ in m.named_parameters())
    m.fuse()
    assert m.model.layers[0].self_attn.qkv_bias is None


def test_fuse_stacks_the_qkv_biases():
    """fuse(): one qkv_bias [q; k; v], the HF-named biases become views of it (as the weights do)"""
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cfg = _qwen2_7b_config(vocab_size=64, hidden_size=896, intermediate_size=256, num_hidden_layers=2,
                           num_attention_heads=7, num_key_value_heads=1)
    m = Qwen2ForCausalLM(cfg, device='cpu').init_weights(seed=3, std=0.5)
    a = m.model.layers[1].self_attn
    q, k, v = a.q_proj.bias.clone(), a.k_proj.bias.clone(), a.v_proj.bias.clone()
    m.fuse()
    assert a.qkv_bias.shape == (896 + 2 * 128,) and a.qkv_bias.is_contiguous()
    assert torch.equal(a.qkv_bias, torch.cat([q, k, v]))
    assert a.q_proj.bias.data_ptr() == a.qkv_bias.data_ptr()
    assert a.k_proj.bias.data_ptr() == a.qkv_bias[896:].data_ptr()
    assert a.v_proj.bias.data_ptr() == a.qkv_bias[1024:].data_ptr()
    # a checkpoint loaded after fuse() lands in the fused operand
    sd = {k_: t.clone() for k_, t in m.state_dict().items()}
    sd['model.layers.1.self_attn.k_proj.bias'].fill_(0.25)
    m.load_state_dict(sd)
    assert torch.all(a.qkv_bias[896:1024] == 0.25)


@pytest.mark.parametrize('gemm_set', ['qkv', 'gate_up,qkv2'])
def test_gemm_set_naming_qkv_is_refused_for_biased_qkv(monkeypatch, gemm_set):
    """k_gemm_ws has no bias epilogue: a GEMM set that would route the biased QKV projection through it raises instead
    of dropping the bias"""
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cfg = _qwen2_7b_config(vocab_size=64, hidden_size=256, intermediate_size=256, num_hidden_layers=1,
                           num_attention_heads=2, num_key_value_heads=1)
    m = Qwen2ForCausalLM(cfg, device='cpu')
    m.fuse()
    monkeypatch.setenv('PIA_GEMM_SET', gemm_set)
    with pytest.raises(ValueError, match='bias'):
        m._layer_gemm_plans(m.model.layers[0], None)


def test_rope_tables_follow_transformers_qwen2():
    """rope_theta 1e6 (stored in rope_parameters by transformers 5): cos / sin equal Qwen2RotaryEmbedding's; an unknown
    scaling type (Qwen2.5's optional YaRN) raises"""
    from transformers.models.qwen2.modeling_qwen2 import Qwen2RotaryEmbedding
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cfg = _qwen2_7b_config(vocab_size=64, hidden_size=256, intermediate_size=256, num_hidden_layers=1,
                           num_attention_heads=2, num_key_value_heads=1)
    m = Qwen2ForCausalLM(cfg, device='cpu')
    cos, sin = m.rope_tables(4096)
    x = torch.zeros((1, 4096, 128), dtype=torch.bfloat16)
    hc, hs = Qwen2RotaryEmbedding(cfg)(x, torch.arange(4096)[None])
    assert torch.allclose(cos.float(), hc[0, :, :64].float(), atol=0, rtol=2 ** -8)
    assert torch.allclose(sin.float(), hs[0, :, :64].float(), atol=0, rtol=2 ** -8)
    yarn = _qwen2_7b_config(vocab_size=64, hidden_size=256, intermediate_size=256, num_hidden_layers=1,
                            num_attention_heads=2, num_key_value_heads=1,
                            rope_scaling={'rope_type': 'yarn', 'factor': 4.0, 'original_max_position_embeddings': 32768})
    with pytest.raises(ValueError, match='yarn'):
        Qwen2ForCausalLM(yarn, device='cpu').rope_tables(64)
