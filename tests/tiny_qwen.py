# -*- coding: utf-8 -*-
"""Seeded tiny Qwen (v1) models (no checkpoints exist offline) and an fp32 torch restatement of the Qwen forward
written from the math, with explicit positions.  The config is a Qwen config.json dict with a small seq_length (64),
so that ordinary test prompts pass it: dynamic NTK (alpha > 1) and log-n scaling are both live.  4 heads of 128,
c_attn biases, w1 / w2 of intermediate_size // 2 each."""
import math

import torch
from torch.nn import functional as F

SEQ_LENGTH = 64


def tiny_config(vocab=200, layers=2, seq_length=SEQ_LENGTH, heads=4, head_dim=128, **over):
    hidden = heads * head_dim
    cfg = dict(model_type='qwen', architectures=['QWenLMHeadModel'], vocab_size=vocab, hidden_size=hidden,
               intermediate_size=1024, num_hidden_layers=layers, num_attention_heads=heads, kv_channels=head_dim,
               layer_norm_epsilon=1e-6, rotary_emb_base=10000, rotary_pct=1.0, seq_length=seq_length,
               max_position_embeddings=8192, use_dynamic_ntk=True, use_logn_attn=True, no_bias=True, bf16=True,
               tie_word_embeddings=False, eos_token_id=2, pad_token_id=0, bos_token_id=1)
    cfg.update(over)
    return cfg


def model_class():
    from painlessinferenceacceleration_b200.models.qwen.modeling_qwen import QWenLMHeadModel
    return QWenLMHeadModel


def tiny_model(seed=0, device='cuda:0', std=0.08, **over):
    from painlessinferenceacceleration_b200.models.qwen.modeling_qwen import qwen_config
    return model_class()(qwen_config(tiny_config(**over)), device=torch.device(device)).init_weights(seed=seed, std=std)


def qwen_state_dict(sd):
    """our (Llama-named) state dict -> Qwen checkpoint names (transformer.h.*, c_attn = [q; k; v] weight and bias,
    w2 = gate, w1 = up)"""
    out = {}
    simple = {'input_layernorm.weight': 'ln_1.weight', 'post_attention_layernorm.weight': 'ln_2.weight',
              'self_attn.o_proj.weight': 'attn.c_proj.weight', 'mlp.gate_proj.weight': 'mlp.w2.weight',
              'mlp.up_proj.weight': 'mlp.w1.weight', 'mlp.down_proj.weight': 'mlp.c_proj.weight'}
    for k, v in sd.items():
        if k == 'model.embed_tokens.weight':
            out['transformer.wte.weight'] = v
        elif k == 'model.norm.weight':
            out['transformer.ln_f.weight'] = v
        elif k.startswith('model.layers.'):
            li, _, rest = k[len('model.layers.'):].partition('.')
            pre = f'transformer.h.{li}.'
            if rest.startswith('self_attn.q_proj.'):
                kind = rest.rsplit('.', 1)[1]
                base = f'model.layers.{li}.self_attn.'
                out[pre + 'attn.c_attn.' + kind] = torch.cat([sd[base + f'{n}.{kind}'] for n in
                                                              ('q_proj', 'k_proj', 'v_proj')], 0)
            elif rest.startswith('self_attn.k_proj.') or rest.startswith('self_attn.v_proj.'):
                continue
            else:
                out[pre + simple[rest]] = v
        else:
            out[k] = v
    return out


def ntk_alpha_ref(L, seq_length):
    """modeling_qwen.py:724-726"""
    return max(2 ** math.ceil(math.log(L / seq_length, 2) + 1) - 1, 1)


def _rms(x, w, eps):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def ref_forward(sd, cfg, ids, pos, allowed, alpha, dtype=torch.float32):
    """the Qwen forward over tokens `ids` [T] at positions `pos` [T] with a boolean visibility matrix allowed [T, T]
    (row attends column), NTK alpha `alpha`, every op in `dtype` (float32: the truth; bfloat16: an eager restatement
    that rounds per op, RoPE in fp32 rounded once as the reference does); sd: Llama-named weights.  Returns logits
    [T, V] fp32"""
    H, hid = cfg['num_attention_heads'], cfg['hidden_size']
    D = hid // H
    S = cfg['seq_length']
    eps = cfg['layer_norm_epsilon']
    w = {k: v.to(dtype) for k, v in sd.items()}
    dev = ids.device
    x = w['model.embed_tokens.weight'][ids]
    T = ids.shape[0]
    base = cfg['rotary_emb_base'] * alpha ** (D / (D - 2))
    inv = 1.0 / (base ** (torch.arange(0, D, 2, device=dev, dtype=torch.float64) / D))
    ang = pos.to(torch.float64)[:, None] * inv[None]
    cos = torch.cat([ang.cos(), ang.cos()], -1)[:, None, :].float()
    sin = torch.cat([ang.sin(), ang.sin()], -1)[:, None, :].float()
    logn = torch.tensor([math.log(p + 1, S) if p + 1 > S else 1.0 for p in pos.tolist()], device=dev)
    logn = logn.to(dtype)[:, None, None] if cfg.get('use_logn_attn', True) else None

    def rope(t):
        r = torch.cat([-t[..., D // 2:], t[..., :D // 2]], -1)
        return (t.float() * cos + r.float() * sin).to(dtype)

    for li in range(cfg['num_hidden_layers']):
        p = f'model.layers.{li}.'
        h = _rms(x, w[p + 'input_layernorm.weight'], eps)
        q = (h @ w[p + 'self_attn.q_proj.weight'].t() + w[p + 'self_attn.q_proj.bias']).view(T, H, D)
        k = (h @ w[p + 'self_attn.k_proj.weight'].t() + w[p + 'self_attn.k_proj.bias']).view(T, H, D)
        v = (h @ w[p + 'self_attn.v_proj.weight'].t() + w[p + 'self_attn.v_proj.bias']).view(T, H, D)
        q, k = rope(q), rope(k)
        if logn is not None:
            q = q * logn
        s = torch.einsum('ihd,jhd->hij', q.float(), k.float()) / math.sqrt(D)
        s = s.masked_fill(~allowed[None], float('-inf'))
        a = torch.softmax(s, -1).to(dtype)
        o = torch.einsum('hij,jhd->ihd', a, v).reshape(T, hid)
        x = x + o @ w[p + 'self_attn.o_proj.weight'].t()
        h = _rms(x, w[p + 'post_attention_layernorm.weight'], eps)
        up = h @ w[p + 'mlp.up_proj.weight'].t()      # w1
        gate = h @ w[p + 'mlp.gate_proj.weight'].t()  # w2
        x = x + (up * F.silu(gate)) @ w[p + 'mlp.down_proj.weight'].t()
    x = _rms(x, w['model.norm.weight'], eps)
    return (x @ w['lm_head.weight'].t()).float()


def causal_logits(sd, cfg, ids, alpha, dtype=torch.float32):
    """plain causal forward over ids [T] at positions 0..T-1"""
    T = ids.shape[0]
    allowed = torch.tril(torch.ones((T, T), dtype=torch.bool, device=ids.device))
    return ref_forward(sd, cfg, ids, torch.arange(T, device=ids.device), allowed, alpha, dtype)
