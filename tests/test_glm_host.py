# -*- coding: utf-8 -*-
"""GLM-family models on the host: module trees against transformers' GlmForCausalLM / Glm4ForCausalLM at the
GLM-4-9B shape, geometry(), the RoPE tables against GlmRotaryEmbedding, ChatGLM config.json translation and tensor
names, and every refusal.  No GPU needed."""
import json

import pytest
import torch

from tests.tiny_glm import glm_config, glm_hf_model, thudm_config, thudm_state_dict


def _glm4_9b(kind='glm', **over):
    from transformers import Glm4Config, GlmConfig
    kw = dict(vocab_size=151552, hidden_size=4096, intermediate_size=13696, num_hidden_layers=40,
              num_attention_heads=32, num_key_value_heads=2, head_dim=128, max_position_embeddings=131072,
              rms_norm_eps=1.5625e-07, attention_bias=True, tie_word_embeddings=False)
    kw.update(over)
    return (GlmConfig if kind == 'glm' else Glm4Config)(**kw)


@pytest.mark.parametrize('kind', ['glm', 'glm4'])
def test_module_tree_matches_transformers(kind):
    """GLM-4-9B on the meta device: every HF parameter name and shape (fused gate_up_proj, q/k/v biases, the sandwich
    norms of glm4), and geometry()"""
    import transformers
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import Glm4ForCausalLM, GlmForCausalLM
    HF = transformers.GlmForCausalLM if kind == 'glm' else transformers.Glm4ForCausalLM
    ours_cls = GlmForCausalLM if kind == 'glm' else Glm4ForCausalLM
    cfg = _glm4_9b(kind)
    with torch.device('meta'):
        hf = HF(cfg)
    ours = ours_cls(cfg, device='meta')
    want = {k: tuple(v.shape) for k, v in hf.named_parameters()}
    got = {k: tuple(v.shape) for k, v in ours.named_parameters()}
    assert got == want
    assert got['model.layers.0.mlp.gate_up_proj.weight'] == (2 * 13696, 4096)
    assert got['model.layers.0.self_attn.k_proj.bias'] == (256,)
    assert ('model.layers.0.post_mlp_layernorm.weight' in got) == (kind == 'glm4')
    assert ours.geometry() == dict(n_layers=40, hidden=4096, n_q_heads=32, n_kv_heads=2, head_dim=128, inter=13696,
                                   vocab=151552, rotary_dim=64)


def test_geometry_of_the_tiny_shapes():
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    g = GlmForCausalLM(glm_config('glm', 64), device='meta').geometry()
    assert (g['n_q_heads'], g['n_kv_heads'], g['head_dim'], g['rotary_dim']) == (6, 2, 64, 32)
    g = GlmForCausalLM(glm_config('glm', 128), device='meta').geometry()
    assert (g['n_q_heads'], g['n_kv_heads'], g['head_dim'], g['rotary_dim']) == (16, 2, 128, 64)


@pytest.mark.parametrize('theta', [10000.0, 10000.0 * 500])   # ChatGLM3-6B-32k: rope_ratio 50; GLM-4 long: 500
@pytest.mark.parametrize('hd', [128, 64])
def test_rope_tables_bit_equal_to_transformers(theta, hd):
    from transformers.models.glm.modeling_glm import GlmRotaryEmbedding
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    cfg = glm_config('glm', hd)
    cfg.rope_parameters = {'rope_type': 'default', 'rope_theta': theta, 'partial_rotary_factor': 0.5}
    cos, sin = GlmForCausalLM(cfg, device='cpu').rope_tables(4096)
    assert cos.shape == (4096, hd // 4)
    hc, hs = GlmRotaryEmbedding(cfg)(torch.zeros((1, 4096, hd), dtype=torch.bfloat16), torch.arange(4096)[None])
    assert hc.shape[-1] == hd // 2
    assert torch.equal(cos, hc[0, :, :hd // 4]) and torch.equal(sin, hs[0, :, :hd // 4])


def test_rope_type_other_than_default_raises():
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    cfg = glm_config('glm', 128)
    cfg.rope_parameters = {'rope_type': 'yarn', 'rope_theta': 10000.0, 'factor': 4.0, 'partial_rotary_factor': 0.5}
    with pytest.raises(ValueError, match='yarn'):
        GlmForCausalLM(cfg, device='cpu').rope_tables(64)


def test_fused_mlp_operand_is_the_checkpoint_weight():
    """fuse(): the gate/up GEMM operand is gate_up_proj.weight itself (no copy); the QKV bias is stacked [q; k; v]"""
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    m = GlmForCausalLM(glm_config('glm', 64), device='cpu').init_weights(seed=1, std=0.5)
    m.fuse()
    layer = m.model.layers[1]
    assert layer.mlp.gate_up_weight.data_ptr() == layer.mlp.gate_up_proj.weight.data_ptr()
    a = layer.self_attn
    assert torch.equal(a.qkv_bias, torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias]))


# -------------------------------------------------------------------------------------------------- ChatGLM format
def _chatglm3_6b_json(**over):
    cfg = dict(model_type='chatglm', add_bias_linear=False, add_qkv_bias=True, apply_query_key_layer_scaling=True,
               apply_residual_connection_post_layernorm=False, attention_softmax_in_fp32=True, ffn_hidden_size=13696,
               hidden_size=4096, kv_channels=128, layernorm_epsilon=1e-05, multi_query_attention=True,
               multi_query_group_num=2, num_attention_heads=32, num_layers=28, original_rope=True,
               padded_vocab_size=65024, post_layer_norm=True, rmsnorm=True, seq_length=8192, eos_token_id=2,
               pad_token_id=0, torch_dtype='float16', quantization_bit=0, pre_seq_len=None)
    cfg.update(over)
    return cfg


def test_chatglm_config_translation(tmp_path):
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    from painlessinferenceacceleration_b200.models.chatglm3.modeling_chatglm import \
        ChatGLMForConditionalGeneration as Chatglm3
    assert Chatglm3 is ChatGLMForConditionalGeneration
    (tmp_path / 'config.json').write_text(json.dumps(_chatglm3_6b_json(rope_ratio=50)))
    cfg = ChatGLMForConditionalGeneration._pretrained_config(str(tmp_path))
    assert cfg.model_type == 'glm'
    assert (cfg.num_hidden_layers, cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size) == (28, 4096, 13696, 65024)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim) == (32, 2, 128)
    assert cfg.rms_norm_eps == 1e-5 and cfg.attention_bias and cfg.max_position_embeddings == 8192
    m = ChatGLMForConditionalGeneration(cfg, device='meta')
    assert m.geometry() == dict(n_layers=28, hidden=4096, n_q_heads=32, n_kv_heads=2, head_dim=128, inter=13696,
                                vocab=65024, rotary_dim=64)
    assert m._rope_parameters() == ('default', 500000.0, 0.5)
    # multi_query_attention=False: every head has its own K / V
    full = ChatGLMForConditionalGeneration.chatglm_config(_chatglm3_6b_json(multi_query_attention=False))
    assert full.num_key_value_heads == 32 and full.chatglm_qkv_per_head
    assert not cfg.chatglm_qkv_per_head
    # fields THUDM's ChatGLMConfig defaults: kv_channels 128, multi_query_group_num 1
    short = _chatglm3_6b_json()
    del short['kv_channels'], short['multi_query_group_num']
    short = ChatGLMForConditionalGeneration.chatglm_config(short)
    assert (short.head_dim, short.num_key_value_heads) == (128, 1)
    # a transformers-format directory is not a chatglm checkpoint
    (tmp_path / 'config.json').write_text(json.dumps(dict(_chatglm3_6b_json(), model_type='glm')))
    with pytest.raises(ValueError, match='chatglm'):
        ChatGLMForConditionalGeneration._pretrained_config(str(tmp_path))


def test_chatglm_tensor_names_map_onto_the_glm_tree():
    """a synthesised THUDM state dict of a tiny GLM: every tensor lands on the transformers name it came from, the
    inv_freq buffer is dropped"""
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    hf = glm_hf_model('glm', 64, seed=4)
    hf_sd = hf.state_dict()
    sd = thudm_state_dict(hf_sd)
    assert 'transformer.rotary_pos_emb.inv_freq' in sd
    cfg = ChatGLMForConditionalGeneration.chatglm_config(thudm_config(hf.config))
    m = ChatGLMForConditionalGeneration(cfg, device='cpu')
    conv = m._convert_checkpoint_keys(sd)
    own = dict(m.named_parameters())
    assert sorted(conv) == sorted(own) == sorted(k for k in hf_sd if k in own)
    for k, v in conv.items():
        assert torch.equal(v, hf_sd[k]), k
    with pytest.raises(ValueError, match='unexpected'):
        m._convert_checkpoint_keys({'transformer.prefix_encoder.embedding.weight': torch.zeros(1)})


@pytest.mark.parametrize('field,value,match', [
    ('rmsnorm', False, 'rmsnorm'),
    ('add_bias_linear', True, 'add_bias_linear'),
    ('apply_residual_connection_post_layernorm', True, 'apply_residual_connection_post_layernorm'),
    ('post_layer_norm', False, 'post_layer_norm'),
    ('original_rope', False, 'original_rope'),
    ('quantization_bit', 4, 'quantization_bit'),
    ('quantization_bit', 8, 'quantization_bit'),
    ('pre_seq_len', 128, 'pre_seq_len'),
    ('position_encoding_2d', True, 'position_encoding_2d'),
    ('kv_channels', 64, 'kv_channels')])
def test_chatglm_refuses_other_networks(field, value, match):
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    with pytest.raises((NotImplementedError, ValueError), match=match):
        ChatGLMForConditionalGeneration.chatglm_config(_chatglm3_6b_json(**{field: value}))


def test_chatglm_v1_without_multi_query_field_is_refused():
    """ChatGLM-6B v1's config has no multi_query_attention field (and 2D positions)"""
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    cfg = _chatglm3_6b_json()
    del cfg['multi_query_attention']
    with pytest.raises(NotImplementedError, match='multi_query_attention'):
        ChatGLMForConditionalGeneration.chatglm_config(cfg)


def test_fused_attention_knob_is_refused(monkeypatch):
    """PIA_ATTN_FUSED: the fused attention kernel has no interleaved RoPE; the model refuses before building anything
    rather than taking the two-kernel path silently"""
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    m = GlmForCausalLM(glm_config('glm', 64), device='cpu')
    monkeypatch.setenv('PIA_ATTN_FUSED', '1')
    with pytest.raises(ValueError, match='PIA_ATTN_FUSED'):
        m._runtime(256, 64)


def test_chatglm_without_multi_query_regroups_per_head_qkv():
    """multi_query_attention=False: query_key_value rows are per head [q_h; k_h; v_h] (weight and bias); every
    tensor of a synthesised THUDM state dict lands on the transformers name it came from"""
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    hf = glm_hf_model('glm', 64, seed=5, num_key_value_heads=6)
    hf_sd = hf.state_dict()
    sd = thudm_state_dict(hf_sd, per_head_dim=64)
    cfg = ChatGLMForConditionalGeneration.chatglm_config(thudm_config(hf.config, multi_query_attention=False))
    assert cfg.num_key_value_heads == 6 and cfg.chatglm_qkv_per_head
    m = ChatGLMForConditionalGeneration(cfg, device='cpu')
    conv = m._convert_checkpoint_keys(sd)
    assert sorted(conv) == sorted(dict(m.named_parameters()))
    for k, v in conv.items():
        assert torch.equal(v, hf_sd[k]), k
    # the same state dict read as [q; k; v] would scramble the heads
    cfg_mqa = ChatGLMForConditionalGeneration.chatglm_config(thudm_config(hf.config, multi_query_group_num=6))
    wrong = ChatGLMForConditionalGeneration(cfg_mqa, device='cpu')._convert_checkpoint_keys(sd)
    assert not torch.equal(wrong['model.layers.0.self_attn.k_proj.weight'], hf_sd['model.layers.0.self_attn.k_proj.weight'])


@pytest.mark.parametrize('kind', ['glm', 'glm4'])
def test_from_pretrained_refuses_the_other_glm_type(tmp_path, kind):
    """a glm4 checkpoint loaded as glm would drop its sandwich norms (and glm as glm4 would lack them): the config's
    model_type must be the class's"""
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import Glm4ForCausalLM, GlmForCausalLM
    glm_config(kind, 64).save_pretrained(str(tmp_path))
    right, wrong = (GlmForCausalLM, Glm4ForCausalLM) if kind == 'glm' else (Glm4ForCausalLM, GlmForCausalLM)
    assert right._pretrained_config(str(tmp_path)).model_type == kind
    with pytest.raises(ValueError, match='model_type'):
        wrong._pretrained_config(str(tmp_path))
