# -*- coding: utf-8 -*-
"""The Baichuan family with the lookahead patch (reference: models/baichuan_7b, baichuan_13b, baichuan2_7b,
baichuan2_13b).  Every member is the Llama decoder (RMSNorm, SwiGLU MLP, no biases, MHA) with q / k / v fused into one
`self_attn.W_pack` weight [q; k; v]; they differ in three places, each a class flag here:
  * alibi: Baichuan-13B and Baichuan2-13B have no RoPE; every score gets a per-head linear position bias
    slope_h * (kpos - qpos) (slopes: baichuan_13b/modeling_baichuan.py:25-36 `_get_interleave`).  The bias is taken at
    TREE positions (the reference's BLOOM patch, bloom/modeling_bloom.py:170), so every draft node's verify logits equal
    a causal forward over prefix + root-to-node path; DESIGN.md section 7 records how this differs from the reference's
    Baichuan-13B lookahead mask (:317-323).  K / V are appended through k_rope_kv_append with identity tables (x * 1 +
    rot(x) * 0, exact), and the tree attention kernel's ALiBi instance adds the bias (pia_tree_attn_alibi_fwd).
  * norm_head: Baichuan2's lm_head rows are L2-normalised (`NormHead`, baichuan2_13b/modeling_baichuan.py:504-521).
    The reference normalises the weight in place on its first eval forward; here the same op (F.normalize in the model
    dtype, on the GPU) runs once when the weights are set: from_pretrained, init_weights, build_fp8.
  * rope_fp32: Baichuan2-7B rotates in fp32 with fp32 cos / sin tables and rounds once
    (baichuan2_7b/modeling_baichuan.py:112-155): k_rope_kv_append's fp32 instance (pia_rope_f32_kv_append).
    Baichuan-7B rotates like Llama (bf16 tables, every op rounded).
The fused RoPE-inside-attention kernel (PIA_ATTN_FUSED) has neither ALiBi nor fp32 RoPE and is refused for those models.

config.json is read as JSON: AutoConfig would need trust_remote_code, which runs code shipped with the checkpoint.
Configs this decoder cannot run raise and name the field."""
import json
import os

import torch
from torch.nn import functional as F

from ...common import ops
from ..llama.modeling_llama import LlamaForCausalLM


def baichuan_config(cfg):
    """Baichuan config.json dict -> a transformers LlamaConfig of the same network.  The RoPE members name their
    context length max_position_embeddings, the ALiBi ones model_max_length (Baichuan2-7B carries both)"""
    from transformers import LlamaConfig
    act = cfg.get('hidden_act', 'silu')
    if act != 'silu':
        raise NotImplementedError(f'baichuan config hidden_act={act!r}: only silu is supported')
    for field in ('quantization_config', 'quantization_bit'):
        if cfg.get(field):
            raise NotImplementedError(f'baichuan config {field}={cfg[field]!r}: quantised Baichuan checkpoints are not '
                                      "supported (load the bf16 checkpoint, optionally with quantization='fp8')")
    for field in ('vocab_size', 'hidden_size', 'intermediate_size', 'num_hidden_layers', 'num_attention_heads'):
        if field not in cfg:
            raise ValueError(f'baichuan config has no {field}')
    heads, hidden = int(cfg['num_attention_heads']), int(cfg['hidden_size'])
    if hidden % heads:
        raise ValueError(f'baichuan config num_attention_heads={heads} does not divide hidden_size={hidden}')
    kv = cfg.get('num_key_value_heads')
    if kv not in (None, heads):
        raise NotImplementedError(f'baichuan config num_key_value_heads={kv}: Baichuan models are multi-head '
                                  f'(num_key_value_heads = num_attention_heads = {heads})')
    mpe = cfg.get('max_position_embeddings') or cfg.get('model_max_length') or 4096
    c = LlamaConfig(vocab_size=int(cfg['vocab_size']), hidden_size=hidden,
                    intermediate_size=int(cfg['intermediate_size']), num_hidden_layers=int(cfg['num_hidden_layers']),
                    num_attention_heads=heads, num_key_value_heads=heads, max_position_embeddings=int(mpe),
                    rms_norm_eps=float(cfg.get('rms_norm_eps', 1e-6)),
                    tie_word_embeddings=bool(cfg.get('tie_word_embeddings', False)),
                    bos_token_id=cfg.get('bos_token_id', 1), eos_token_id=cfg.get('eos_token_id', 2),
                    pad_token_id=cfg.get('pad_token_id', 0))
    c.model_max_length = int(cfg.get('model_max_length') or mpe)
    return c


class BaichuanBase(LlamaForCausalLM):
    """shared base of the four Baichuan classes; module tree and parameter names are Llama's (the checkpoint's
    W_pack is split into q / k / v on load)"""
    int4_checkpoints = False   # quantization_config is refused by the config check
    alibi = False       # Baichuan-13B, Baichuan2-13B: ALiBi instead of RoPE
    norm_head = False   # Baichuan2: L2-normalised lm_head rows
    rope_fp32 = False   # Baichuan2-7B: fp32 cos / sin tables and arithmetic
    # every member's RMSNorm casts x_hat to bf16, then multiplies by the weight (baichuan_7b/modeling_baichuan.py:84-91)
    rmsnorm_rounding = ops.ROUND_TWICE

    def __init__(self, config, device=None, dtype=torch.bfloat16):
        hd = config.hidden_size // config.num_attention_heads
        if self.alibi and hd != 128:
            raise ValueError(f'{type(self).__name__}: hidden_size / num_attention_heads = {hd}; the ALiBi tree '
                             'attention is built for head dim 128 only')
        super().__init__(config, device=device, dtype=dtype)

    @staticmethod
    def baichuan_config(cfg):
        return baichuan_config(cfg)

    @classmethod
    def _pretrained_config(cls, path):
        with open(os.path.join(path, 'config.json')) as f:
            cfg = json.load(f)
        if cfg.get('model_type') != 'baichuan':
            raise ValueError(f'{path}: model_type {cfg.get("model_type")!r} is not a Baichuan checkpoint')
        return baichuan_config(cfg)

    # ------------------------------------------------------------------ weights
    @torch.no_grad()
    def normalize_lm_head(self):
        """NormHead: lm_head rows to unit L2 norm, F.normalize in the model dtype on the model's device (what the
        reference's NormHead does to its weight on the first eval forward); no-op for the other members"""
        if self.norm_head:
            w = self.lm_head.weight
            w.copy_(F.normalize(w))
        return self

    @torch.no_grad()
    def init_weights(self, seed=0, std=0.02):
        super().init_weights(seed=seed, std=std)
        return self.normalize_lm_head()

    @classmethod
    def from_pretrained(cls, path, torch_dtype=torch.bfloat16, device=None, quantization=None, **kwargs):
        model = super().from_pretrained(path, torch_dtype=torch_dtype, device=device, quantization=quantization,
                                        **kwargs)
        return model.normalize_lm_head()

    @classmethod
    def build_fp8(cls, config, fill_rest, fill_weight, device=None):
        return super().build_fp8(config, fill_rest, fill_weight, device=device).normalize_lm_head()

    def _convert_checkpoint_keys(self, sd):
        """self_attn.W_pack.weight [3 * hidden, hidden] = [q; k; v] -> q_proj / k_proj / v_proj (reference
        baichuan2_7b/modeling_baichuan.py:208-212); the rotary inv_freq buffers some checkpoints carry are dropped"""
        hid = self.config.hidden_size
        out = {}
        for k, v in sd.items():
            if k.endswith('self_attn.W_pack.weight'):
                if tuple(v.shape) != (3 * hid, hid):
                    raise ValueError(f'{k}: shape {tuple(v.shape)}, expected {(3 * hid, hid)}')
                pre = k[:-len('W_pack.weight')]
                out[pre + 'q_proj.weight'], out[pre + 'k_proj.weight'], out[pre + 'v_proj.weight'] = \
                    v[:hid], v[hid:2 * hid], v[2 * hid:]
            elif k.endswith('rotary_emb.inv_freq'):
                continue
            else:
                out[k] = v
        return out

    # ------------------------------------------------------------------ tables / runtime
    def rope_tables(self, max_pos):
        hd = self.config.hidden_size // self.config.num_attention_heads
        dev = self.device
        if self.alibi:   # identity rotation: k_rope_kv_append copies q and appends K / V unchanged
            return (torch.ones((max_pos, hd // 2), dtype=torch.bfloat16, device=dev),
                    torch.zeros((max_pos, hd // 2), dtype=torch.bfloat16, device=dev))
        if not self.rope_fp32:
            return super().rope_tables(max_pos)
        # Baichuan2-7B's RotaryEmbedding (:112-121), on the CPU over max_position_embeddings positions as the reference
        # builds it (so that the same elementwise cos / sin evaluations produce the tables), fp32 throughout
        n = max(int(max_pos), int(self.config.max_position_embeddings))
        inv_freq = 1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))
        t = torch.arange(n, dtype=torch.float32)
        freqs = torch.outer(t, inv_freq)
        emb = torch.cat((freqs, freqs), dim=-1)
        cos, sin = emb.cos()[:max_pos, :hd // 2], emb.sin()[:max_pos, :hd // 2]
        return cos.contiguous().to(dev), sin.contiguous().to(dev)

    def _check_fused_attn(self):
        if (self.alibi or self.rope_fp32) and os.environ.get('PIA_ATTN_FUSED', '0') != '0':
            what = 'ALiBi' if self.alibi else 'fp32 RoPE'
            raise ValueError(f'{type(self).__name__} needs {what}, which the fused attention kernel does not have: '
                             'unset PIA_ATTN_FUSED')
        super()._check_fused_attn()

    def _runtime(self, max_seq, max_nodes, n_slots=1, keep_cache=False):
        self._check_fused_attn()   # before anything is captured
        rt = super()._runtime(max_seq, max_nodes, n_slots, keep_cache)
        if self.alibi:   # the slopes in a device buffer of the model, made outside any capture
            if getattr(self, 'alibi_slopes', None) is None or self.alibi_slopes.device != rt.device:
                self.alibi_slopes = ops.alibi_slopes(self.config.num_attention_heads).to(rt.device)
            rt.alibi_slopes = self.alibi_slopes
        return rt
