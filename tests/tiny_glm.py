# -*- coding: utf-8 -*-
"""seeded tiny random-init HF GLM models (no checkpoints exist offline), initialised like tests/tiny_qwen2.py (std 0.08,
non-zero q/k/v biases, large k biases):
  * glm_hf_model(hd=128): model_type `glm`, head dim 128, 16 query heads over 2 KV heads (G = 16, as ChatGLM3-6B and
    GLM-4-9B), hidden 2048, rotary_dim 64;
  * glm_hf_model(hd=64): model_type `glm`, head dim 64, 6 query heads over 2 KV heads (odd G = 3), hidden 384,
    rotary_dim 32;
  * glm_hf_model(kind='glm4'): model_type `glm4` with the sandwich norms, whose RMSNorm weights are drawn around 1
    (1 + N(0, 0.1)) so that a missing or misplaced norm shows in the logits."""
import torch

SHAPES = {128: dict(hidden_size=2048, num_attention_heads=16, num_key_value_heads=2, head_dim=128),
          64: dict(hidden_size=384, num_attention_heads=6, num_key_value_heads=2, head_dim=64)}


def glm_config(kind='glm', hd=128, vocab=64, **over):
    from transformers import Glm4Config, GlmConfig
    cls = GlmConfig if kind == 'glm' else Glm4Config
    cfg = cls(vocab_size=vocab, intermediate_size=512, num_hidden_layers=2, max_position_embeddings=1024,
              rms_norm_eps=1e-5, attention_bias=True, tie_word_embeddings=False, bos_token_id=1, eos_token_id=2,
              pad_token_id=0, **SHAPES[hd])
    for k, v in over.items():
        setattr(cfg, k, v)
    cfg._attn_implementation = 'eager'
    return cfg


def glm_hf_model(kind='glm', hd=128, seed=0, dtype=torch.float32, device='cpu', vocab=64, **over):
    from transformers import AutoModelForCausalLM
    torch.manual_seed(seed)
    model = AutoModelForCausalLM.from_config(glm_config(kind, hd, vocab=vocab, **over), attn_implementation='eager')
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() >= 2:
                p.normal_(0.0, 0.08)
            elif kind == 'glm4' and n.endswith('norm.weight'):
                p.normal_(1.0, 0.1)
        for layer in model.model.layers:
            a = layer.self_attn
            a.q_proj.bias.normal_(0.0, 1.0)
            a.k_proj.bias.normal_(0.0, 3.0)
            a.v_proj.bias.normal_(0.0, 1.0)
    return model.to(device=device, dtype=dtype).eval()


def glm_model_class(kind):
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import Glm4ForCausalLM, GlmForCausalLM
    return GlmForCausalLM if kind == 'glm' else Glm4ForCausalLM


def thudm_state_dict(hf_sd, per_head_dim=None):
    """the THUDM (chatglm) names of a transformers GLM state dict: fused query_key_value [q; k; v] (multi-query
    attention) or, given per_head_dim, per head [q_h; k_h; v_h] (multi_query_attention=False, every head its own K / V),
    dense_h_to_4h [gate; up] as they are, plus the rotary inv_freq buffer THUDM checkpoints carry"""
    out = {}
    n_layers = 1 + max(int(k.split('.')[2]) for k in hf_sd if k.startswith('model.layers.'))
    for li in range(n_layers):
        p, q = f'model.layers.{li}.', f'transformer.encoder.layers.{li}.'
        for kind in ('weight', 'bias'):
            parts = [hf_sd[p + f'self_attn.{x}_proj.{kind}'] for x in 'qkv']
            if per_head_dim:
                hd = per_head_dim
                parts = [t[h * hd:(h + 1) * hd] for h in range(parts[0].shape[0] // hd) for t in parts]
            out[q + 'self_attention.query_key_value.' + kind] = torch.cat(parts, 0).contiguous()
        out[q + 'self_attention.dense.weight'] = hf_sd[p + 'self_attn.o_proj.weight']
        out[q + 'input_layernorm.weight'] = hf_sd[p + 'input_layernorm.weight']
        out[q + 'post_attention_layernorm.weight'] = hf_sd[p + 'post_attention_layernorm.weight']
        out[q + 'mlp.dense_h_to_4h.weight'] = hf_sd[p + 'mlp.gate_up_proj.weight']
        out[q + 'mlp.dense_4h_to_h.weight'] = hf_sd[p + 'mlp.down_proj.weight']
    out['transformer.embedding.word_embeddings.weight'] = hf_sd['model.embed_tokens.weight']
    out['transformer.encoder.final_layernorm.weight'] = hf_sd['model.norm.weight']
    out['transformer.output_layer.weight'] = hf_sd['lm_head.weight']
    out['transformer.rotary_pos_emb.inv_freq'] = torch.ones(32)
    return out


def thudm_config(hf_cfg, **over):
    """a ChatGLM2/3-style config.json dict describing the same network as a transformers GlmConfig"""
    rp = hf_cfg.rope_parameters
    cfg = dict(model_type='chatglm', architectures=['ChatGLMModel'], add_bias_linear=False, add_qkv_bias=True,
               apply_query_key_layer_scaling=True, apply_residual_connection_post_layernorm=False,
               attention_softmax_in_fp32=True, bias_dropout_fusion=True, ffn_hidden_size=hf_cfg.intermediate_size,
               fp32_residual_connection=False, hidden_size=hf_cfg.hidden_size, kv_channels=hf_cfg.head_dim,
               layernorm_epsilon=hf_cfg.rms_norm_eps, multi_query_attention=True,
               multi_query_group_num=hf_cfg.num_key_value_heads, num_attention_heads=hf_cfg.num_attention_heads,
               num_layers=hf_cfg.num_hidden_layers, original_rope=True, padded_vocab_size=hf_cfg.vocab_size,
               post_layer_norm=True, rmsnorm=True, seq_length=hf_cfg.max_position_embeddings, use_cache=True,
               torch_dtype='bfloat16', tie_word_embeddings=False, eos_token_id=2, pad_token_id=0,
               rope_ratio=rp['rope_theta'] / 10000.0)
    cfg.update(over)
    return cfg
