# -*- coding: utf-8 -*-
"""Qwen (v1: Qwen-1.8B / 7B / 14B / 72B, HF model_type `qwen`) with the lookahead patch (reference:
models/qwen/modeling_qwen.py, `QWenLMHeadModel`).  The network is the Llama decoder with a biased fused QKV
projection (Qwen2's, `attn.c_attn` = [q; k; v] split on load) and three Qwen-specific pieces:
  * RoPE in fp32 with fp32 cos / sin tables built on the CPU op for op as `RotaryEmbedding.update_rotary_pos_emb_cache`
    (:1184-1206), one bf16 rounding after the rotation (`apply_rotary_pos_emb` :1222-1237): k_rope_kv_append's fp32
    instance.
  * dynamic NTK, fixed per request (:716-730): the prefill (no past) sets alpha = max(2^ceil(log2(L / seq_length) + 1)
    - 1, 1) from its input length L, the RoPE base becomes base * alpha^(d / (d - 2)), and every decode step of the
    request keeps that alpha.  `_start_request` copies the tables of the request's alpha into the runtime's tables in
    place, so captured prefill and step graphs keep their pointers.
  * log-n attention scaling (:223-227, :374-380): after RoPE each query row is multiplied, in bf16, by
    log(pos + 1, seq_length) once pos + 1 > seq_length (pia_rope_f32_logn_kv_append).  The reference's table has 32767
    entries, so max_length is limited to 32767 with use_logn_attn.
RoPE and log-n are taken at TREE positions, max(P - pad, 0) + depth, where the reference slices both by cache column
(:355-362, :377-379); DESIGN.md section 7 records the deviation.  The MLP is w1(x) * silu(w2(x)) (:441-445): w2 is the
gate, w1 the up projection.  RMSNorm multiplies the bf16 input by an fp32 rsqrt and the weight, rounding once
(:1262-1266).  The fused RoPE-inside-attention kernel (PIA_ATTN_FUSED) has neither fp32 RoPE nor log-n and is refused.

config.json is read as JSON: AutoConfig would need trust_remote_code, which runs code shipped with the checkpoint.
Configs this decoder cannot run raise and name the field."""
import json
import math
import os

import torch

from ...common import ops
from ..llama.modeling_llama import LlamaForCausalLM
from ..qwen2.modeling_qwen2 import Qwen2Model

LOGN_ENTRIES = 32767   # the reference's logn_list: range(1, 32768)
ENDOFTEXT = 151643     # <|endoftext|> of Qwen's tokenizer, its eos / pad when the config names none


def qwen_config(cfg):
    """Qwen config.json dict -> a transformers LlamaConfig of the same network, carrying seq_length, use_dynamic_ntk
    and use_logn_attn"""
    from transformers import LlamaConfig
    if cfg.get('model_type') != 'qwen':
        raise ValueError(f'config model_type={cfg.get("model_type")!r} is not a Qwen (v1) checkpoint (model_type '
                         "'qwen'; Qwen1.5 / Qwen2 checkpoints load through models.qwen2)")
    for field in ('quantization_config', 'quantization_bit'):
        if cfg.get(field):
            raise NotImplementedError(f'qwen config {field}={cfg[field]!r}: quantised (GPTQ Int4 / Int8) Qwen checkpoints '
                                      "are not supported (load the bf16 checkpoint, optionally with quantization='fp8')")
    for field in ('vocab_size', 'hidden_size', 'intermediate_size', 'num_hidden_layers', 'num_attention_heads',
                  'seq_length'):
        if field not in cfg:
            raise ValueError(f'qwen config has no {field}')
    heads, hidden = int(cfg['num_attention_heads']), int(cfg['hidden_size'])
    if hidden % heads:
        raise ValueError(f'qwen config num_attention_heads={heads} does not divide hidden_size={hidden}')
    if float(cfg.get('rotary_pct', 1.0)) != 1.0:
        raise NotImplementedError(f'qwen config rotary_pct={cfg["rotary_pct"]}: only rotary_pct = 1 (RoPE over the '
                                  'whole head) is supported')
    if not cfg.get('no_bias', True):
        raise NotImplementedError('qwen config no_bias=False: biases on c_proj / w1 / w2 are not supported')
    kv_channels = cfg.get('kv_channels', hidden // heads)
    if int(kv_channels) != hidden // heads:
        raise NotImplementedError(f'qwen config kv_channels={kv_channels}: only kv_channels = hidden_size / '
                                  f'num_attention_heads = {hidden // heads} is supported')
    inter = int(cfg['intermediate_size'])
    if inter % 2:
        raise ValueError(f'qwen config intermediate_size={inter} is odd: w1 and w2 are intermediate_size // 2 wide each')
    c = LlamaConfig(vocab_size=int(cfg['vocab_size']), hidden_size=hidden, intermediate_size=inter // 2,
                    num_hidden_layers=int(cfg['num_hidden_layers']), num_attention_heads=heads,
                    num_key_value_heads=heads, max_position_embeddings=int(cfg.get('max_position_embeddings', 8192)),
                    rms_norm_eps=float(cfg.get('layer_norm_epsilon', 1e-6)),
                    rope_theta=float(cfg.get('rotary_emb_base', 10000)),
                    tie_word_embeddings=bool(cfg.get('tie_word_embeddings', False)),
                    bos_token_id=cfg.get('bos_token_id', ENDOFTEXT), eos_token_id=cfg.get('eos_token_id', ENDOFTEXT),
                    pad_token_id=cfg.get('pad_token_id', ENDOFTEXT))
    c.rotary_emb_base = cfg.get('rotary_emb_base', 10000)   # as given: the reference's base is a python number
    c.seq_length = int(cfg['seq_length'])
    c.use_dynamic_ntk = bool(cfg.get('use_dynamic_ntk', True))
    c.use_logn_attn = bool(cfg.get('use_logn_attn', True))
    return c


def ntk_alpha(input_len, seq_length, use_dynamic_ntk=True):
    """the NTK alpha of a request whose prefill has `input_len` tokens (modeling_qwen.py:719-728)"""
    if not use_dynamic_ntk:
        return 1.0
    context_value = math.log(input_len / seq_length, 2) + 1
    return max(2 ** math.ceil(context_value) - 1, 1)


def rope_tables_f32(dim, base, alpha, max_pos):
    """fp32 cos / sin [max_pos, dim / 2] of RotaryEmbedding.update_rotary_pos_emb_cache (:1187-1205) at ntk_alpha
    `alpha`, on the CPU, op for op (a row does not depend on how many rows are built)"""
    base = base * alpha ** (dim / (dim - 2))
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim))
    seq = torch.arange(max_pos)
    freqs = torch.outer(seq.type_as(inv_freq), inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos(), emb.sin()
    return cos[:, :dim // 2].contiguous(), sin[:, :dim // 2].contiguous()


def logn_table(seq_length, max_pos):
    """bf16 [max_pos]: entry p = log(p + 1, seq_length) if p + 1 > seq_length else 1, computed in float64, stored as
    fp32 and cast to bf16, the path of the reference's logn_tensor (:223-227, :375-376)"""
    vals = [math.log(i, seq_length) if i > seq_length else 1 for i in range(1, max_pos + 1)]
    return torch.tensor(vals).to(torch.bfloat16)


class QWenLMHeadModel(LlamaForCausalLM):
    """module tree and parameter names are Llama's (checkpoint names are translated on load)"""
    model_cls = Qwen2Model   # the Llama decoder with biases on q / k / v
    int4_checkpoints = False   # quantization_config is refused by the config check
    rmsnorm_rounding = ops.ROUND_ONCE   # (weight * (x * rsqrt(var + eps))).to(bf16): one rounding (:1262-1266)

    @staticmethod
    def qwen_config(cfg):
        return qwen_config(cfg)

    @classmethod
    def _pretrained_config(cls, path):
        with open(os.path.join(path, 'config.json')) as f:
            return qwen_config(json.load(f))

    def _convert_checkpoint_keys(self, sd):
        """Qwen checkpoint names -> Llama names: transformer.wte / ln_f, h.{i}.ln_1 / ln_2, attn.c_attn (weight and bias
        [q; k; v], :203, :347-349) split into q / k / v, attn.c_proj -> o_proj, mlp.w2 -> gate_proj, mlp.w1 ->
        up_proj (w1(x) * silu(w2(x)), :441-445), mlp.c_proj -> down_proj; rotary inv_freq buffers dropped"""
        hid = self.config.hidden_size
        simple = {'ln_1.weight': 'input_layernorm.weight', 'ln_2.weight': 'post_attention_layernorm.weight',
                  'attn.c_proj.weight': 'self_attn.o_proj.weight', 'mlp.w2.weight': 'mlp.gate_proj.weight',
                  'mlp.w1.weight': 'mlp.up_proj.weight', 'mlp.c_proj.weight': 'mlp.down_proj.weight'}
        out = {}
        for k, v in sd.items():
            if k.endswith('rotary_emb.inv_freq'):
                continue
            if k == 'transformer.wte.weight':
                out['model.embed_tokens.weight'] = v
            elif k == 'transformer.ln_f.weight':
                out['model.norm.weight'] = v
            elif k.startswith('transformer.h.'):
                li, _, rest = k[len('transformer.h.'):].partition('.')
                pre = f'model.layers.{li}.'
                if rest in ('attn.c_attn.weight', 'attn.c_attn.bias'):
                    kind = rest.rsplit('.', 1)[1]
                    want = (3 * hid, hid) if kind == 'weight' else (3 * hid,)
                    if tuple(v.shape) != want:
                        raise ValueError(f'{k}: shape {tuple(v.shape)}, expected {want}')
                    for j, name in enumerate(('q_proj', 'k_proj', 'v_proj')):
                        out[f'{pre}self_attn.{name}.{kind}'] = v[j * hid:(j + 1) * hid]
                elif rest in simple:
                    out[pre + simple[rest]] = v
                else:
                    out[k] = v
            else:
                out[k] = v
        return out

    # ------------------------------------------------------------------ tables / runtime
    def _head_dim(self):
        return self.config.hidden_size // self.config.num_attention_heads

    def _host_rope(self, alpha, max_pos):
        """the fp32 tables of one alpha on the host, cached per (alpha, length)"""
        cache = self.__dict__.setdefault('_rope_host', {})
        key = (alpha, int(max_pos))
        if key not in cache:
            cache[key] = rope_tables_f32(self._head_dim(), self.config.rotary_emb_base, alpha, max_pos)
        return cache[key]

    def rope_tables(self, max_pos):
        """the tables at alpha 1 (a new runtime's; _start_request switches them per request)"""
        cos, sin = self._host_rope(1.0, max_pos)
        return cos.to(self.device), sin.to(self.device)

    def _check_fused_attn(self):
        if os.environ.get('PIA_ATTN_FUSED', '0') != '0':
            raise ValueError(f'{type(self).__name__} needs fp32 RoPE and log-n query scaling, which the fused attention '
                             'kernel does not have: unset PIA_ATTN_FUSED')
        super()._check_fused_attn()

    def _runtime(self, max_seq, max_nodes, n_slots=1, keep_cache=False):
        self._check_fused_attn()   # before anything is captured
        rt = super()._runtime(max_seq, max_nodes, n_slots, keep_cache)
        if getattr(rt, 'ntk_alpha', None) is None:   # a new runtime: its tables are alpha 1's
            rt.ntk_alpha = 1.0
            rt.logn_scale = None
            if self.config.use_logn_attn:   # one device table per runtime, made outside any capture
                rt.logn_scale = logn_table(self.config.seq_length, rt.rope_cos.shape[0]).to(rt.device)
        return rt

    def _start_request(self, rt, input_len, max_length=None):
        """a request's prefill of `input_len` tokens (left padding included) fixes its NTK alpha; the runtime's tables
        are rewritten in place when the alpha changes (nothing is in flight between requests)"""
        c = self.config
        if c.use_logn_attn and max_length is not None and max_length > LOGN_ENTRIES:
            raise ValueError(f'max_length={max_length}: with use_logn_attn the log-n table covers {LOGN_ENTRIES} '
                             'positions (modeling_qwen.py:223-227)')
        alpha = ntk_alpha(input_len, c.seq_length, c.use_dynamic_ntk)
        if alpha != rt.ntk_alpha:
            cos, sin = self._host_rope(alpha, rt.rope_cos.shape[0])
            rt.rope_cos.copy_(cos)
            rt.rope_sin.copy_(sin)
            rt.ntk_alpha = alpha


__all__ = ['QWenLMHeadModel', 'qwen_config', 'ntk_alpha', 'rope_tables_f32', 'logn_table']
