# -*- coding: utf-8 -*-
"""Seeded tiny Baichuan models (no checkpoints exist offline) and an fp32 torch restatement of the Baichuan forward
written from the math, with explicit positions:
  * '13b' / '2_13b': ALiBi, 5 heads of 128 (a head count that is not a power of two), no RoPE;
  * '7b': Llama RoPE (bf16 tables); '2_7b': fp32 RoPE; 4 heads of 128;
  * '2_*': the lm_head rows L2-normalised (NormHead).
Configs are Baichuan config.json dicts (model_max_length for the ALiBi members, max_position_embeddings for the RoPE
ones)."""
import math

import torch
from torch.nn import functional as F

KINDS = ('7b', '13b', '2_7b', '2_13b')


def tiny_config(kind, vocab=200, layers=2):
    heads = 5 if kind in ('13b', '2_13b') else 4
    cfg = dict(model_type='baichuan', vocab_size=vocab, hidden_size=128 * heads, intermediate_size=512,
               num_hidden_layers=layers, num_attention_heads=heads, hidden_act='silu', rms_norm_eps=1e-6,
               bos_token_id=1, eos_token_id=2, pad_token_id=0, tie_word_embeddings=False)
    if kind in ('13b', '2_13b'):
        cfg['model_max_length'] = 1024
    else:
        cfg['max_position_embeddings'] = 1024
        if kind == '2_7b':
            cfg['model_max_length'] = 1024
    return cfg


def model_class(kind, batch=False):
    if kind == '7b':
        from painlessinferenceacceleration_b200.models.baichuan_7b.modeling_baichuan import BaiChuanForCausalLM as C
    elif kind == '13b':
        from painlessinferenceacceleration_b200.models.baichuan_13b.modeling_baichuan import BaichuanForCausalLM as C
    elif kind == '2_13b':
        from painlessinferenceacceleration_b200.models.baichuan2_13b.modeling_baichuan import BaichuanForCausalLM as C
    elif batch:
        from painlessinferenceacceleration_b200.models.baichuan2_7b.modeling_baichuan_batch import \
            BaichuanForCausalLM as C
    else:
        from painlessinferenceacceleration_b200.models.baichuan2_7b.modeling_baichuan import BaichuanForCausalLM as C
    if batch and kind != '2_7b':   # the batched loop over the other members, mixed in as the Baichuan2-7B class does
        from painlessinferenceacceleration_b200.common.pretrained_model_batch import LookaheadPreTrainedModel as Loop
        C = type(C.__name__, (Loop, C), {})
    return C


def tiny_model(kind, seed=0, device='cuda:0', batch=False, std=0.08):
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    cls = model_class(kind, batch)
    return cls(baichuan_config(tiny_config(kind)), device=torch.device(device)).init_weights(seed=seed, std=std)


def w_pack_state_dict(sd):
    """our (Llama-named) state dict -> Baichuan checkpoint names: q / k / v rows fused into self_attn.W_pack.weight"""
    out = {}
    for k, v in sd.items():
        if k.endswith('self_attn.q_proj.weight'):
            pre = k[:-len('q_proj.weight')]
            out[pre + 'W_pack.weight'] = torch.cat([v, sd[pre + 'k_proj.weight'], sd[pre + 'v_proj.weight']], 0)
        elif k.endswith('self_attn.k_proj.weight') or k.endswith('self_attn.v_proj.weight'):
            continue
        else:
            out[k] = v
    return out


def slopes_f64(n):
    """ALiBi slopes from the definition: 2^(-8 i / n), i = 1..n, for a power of two n; otherwise those of the largest
    power of two c < n followed by the odd-indexed slopes 2^(-8 (2 i - 1) / (2 c)) of 2c heads, i = 1..n - c"""
    c = 2 ** int(math.floor(math.log2(n)))
    s = [2.0 ** (-8.0 * (i + 1) / c) for i in range(c)]
    s += [2.0 ** (-8.0 * (2 * i + 1) / (2 * c)) for i in range(n - c)]
    return s


def _rms(x, w, eps):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def ref_forward(sd, cfg, kind, ids, pos, allowed, dtype=torch.float32):
    """the Baichuan forward over tokens `ids` [T] at positions `pos` [T] with a boolean visibility matrix
    allowed [T, T] (row attends column), every op in `dtype` (float32: the truth; bfloat16: an eager restatement that
    rounds per op); sd: Llama-named weights.  Returns logits [T, V] fp32"""
    H = cfg['num_attention_heads']
    hid = cfg['hidden_size']
    D = hid // H
    eps = cfg['rms_norm_eps']
    w = {k: v.to(dtype) for k, v in sd.items()}
    dev = ids.device
    x = w['model.embed_tokens.weight'][ids]
    T = ids.shape[0]
    pos_f = pos.to(torch.float32)
    if kind in ('13b', '2_13b'):
        sl = torch.tensor(slopes_f64(H), dtype=torch.float64, device=dev).to(torch.float32)
        bias = sl[:, None, None] * (pos_f[None, None, :] - pos_f[None, :, None])   # [H, T, T]
    else:
        inv = 1.0 / (10000 ** (torch.arange(0, D, 2, device=dev, dtype=torch.float32) / D))
        ang = pos_f[:, None] * inv[None]
        cos = torch.cat([ang.cos(), ang.cos()], -1)[:, None, :]
        sin = torch.cat([ang.sin(), ang.sin()], -1)[:, None, :]
        if kind == '7b':
            cos, sin = cos.to(dtype), sin.to(dtype)

    def rope(t):
        r = torch.cat([-t[..., D // 2:], t[..., :D // 2]], -1)
        if kind == '2_7b':   # fp32 arithmetic, one rounding
            return (t.float() * cos + r.float() * sin).to(dtype)
        return t * cos + r * sin

    for li in range(cfg['num_hidden_layers']):
        p = f'model.layers.{li}.'
        h = _rms(x, w[p + 'input_layernorm.weight'], eps)
        q = (h @ w[p + 'self_attn.q_proj.weight'].t()).view(T, H, D)
        k = (h @ w[p + 'self_attn.k_proj.weight'].t()).view(T, H, D)
        v = (h @ w[p + 'self_attn.v_proj.weight'].t()).view(T, H, D)
        if kind not in ('13b', '2_13b'):
            q, k = rope(q), rope(k)
        s = torch.einsum('ihd,jhd->hij', q.float(), k.float()) / math.sqrt(D)
        if kind in ('13b', '2_13b'):
            s = s + bias
        s = s.masked_fill(~allowed[None], float('-inf'))
        a = torch.softmax(s, -1).to(dtype)
        o = torch.einsum('hij,jhd->ihd', a, v).reshape(T, hid)
        x = x + o @ w[p + 'self_attn.o_proj.weight'].t()
        h = _rms(x, w[p + 'post_attention_layernorm.weight'], eps)
        g = h @ w[p + 'mlp.gate_proj.weight'].t()
        u = h @ w[p + 'mlp.up_proj.weight'].t()
        x = x + (F.silu(g) * u) @ w[p + 'mlp.down_proj.weight'].t()
    x = _rms(x, w['model.norm.weight'], eps)
    return (x @ w['lm_head.weight'].t()).float()


def causal_logits(sd, cfg, kind, ids, dtype=torch.float32):
    """plain causal forward over ids [T] at positions 0..T-1"""
    T = ids.shape[0]
    allowed = torch.tril(torch.ones((T, T), dtype=torch.bool, device=ids.device))
    return ref_forward(sd, cfg, kind, ids, torch.arange(T, device=ids.device), allowed, dtype)
