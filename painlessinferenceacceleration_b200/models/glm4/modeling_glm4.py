# -*- coding: utf-8 -*-
"""GLM-family decoders with the lookahead patch: HF model_type `glm` (GLM-4-9B(-chat)-hf) and `glm4` (GLM-4-9B-0414,
GLM-4-32B-0414, GLM-Z1).  ChatGLM2/3-6B checkpoints in THUDM's own format load into the same decoder through
models/chatglm (reference: models/chatglm/modeling_chatglm.py; lookahead positions :815 = rowsum(mask) - 1, the
Llama patch).

The decoder is Qwen2's (Llama with biases on q/k/v, none on o) except in three places:
  * RoPE rotates only the first rotary_dim = head_dim * partial_rotary_factor dims of every q / k head, in interleaved
    pairs (2i, 2i+1) with frequency i (reference :156-169; transformers' glm apply_rotary_pos_emb); the other dims
    pass through.  k_rope_kv_append's GLM instance (pia_rope_interleaved_kv_append) does it, tables
    [max_pos, rotary_dim / 2].  The fused RoPE-inside-attention kernel (PIA_ATTN_FUSED) has no such layout and is
    refused.
  * The MLP keeps HF's fused `gate_up_proj` weight [gate; up] (HF computes up * silu(gate)): it is the fused gate/up
    GEMM operand as it stands.
  * glm4 only: "sandwich" norms, `post_self_attn_layernorm` on the attention output and `post_mlp_layernorm` on the MLP
    output, each before its residual add.
Query heads per KV head are 16 (ChatGLM3-6B, GLM-4-9B: 32 over 2) or 6 (GLM-4-32B: 48 over 8); tree attention packs
any group.  Only the default RoPE type is supported."""
import torch
from torch import nn

from ...common import ops
from ..llama.modeling_llama import Fp8Linear, Fp8Rows, LlamaDecoderLayer, LlamaForCausalLM, LlamaModel, LlamaRMSNorm


class GlmMLP(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        kw = dict(bias=False, device=device, dtype=dtype)
        self.gate_up_proj = nn.Linear(cfg.hidden_size, 2 * cfg.intermediate_size, **kw)
        self.down_proj = nn.Linear(cfg.intermediate_size, cfg.hidden_size, **kw)


class GlmDecoderLayer(LlamaDecoderLayer):
    def _qkv_bias(self, cfg):
        # q/k/v biases unless the config turns them off (attention_bias, True for every published GLM)
        return bool(getattr(cfg, 'attention_bias', True))

    def _make_mlp(self, cfg, device, dtype):
        return GlmMLP(cfg, device, dtype)


class Glm4DecoderLayer(GlmDecoderLayer):
    def __init__(self, cfg, device, dtype):
        super().__init__(cfg, device, dtype)
        self.post_self_attn_layernorm = LlamaRMSNorm(cfg.hidden_size, cfg.rms_norm_eps, device, dtype)
        self.post_mlp_layernorm = LlamaRMSNorm(cfg.hidden_size, cfg.rms_norm_eps, device, dtype)


class GlmModel(LlamaModel):
    layer_cls = GlmDecoderLayer


class Glm4Model(LlamaModel):
    layer_cls = Glm4DecoderLayer


class GlmForCausalLM(LlamaForCausalLM):
    model_cls = GlmModel
    model_type = 'glm'
    rotary_interleaved = True
    rmsnorm_rounding = ops.ROUND_TWICE   # transformers' GlmRMSNorm / Glm4RMSNorm: weight * hidden_states.to(input_dtype)

    _fp8_params = ('self_attn.q_proj.weight', 'self_attn.k_proj.weight', 'self_attn.v_proj.weight',
                   'self_attn.o_proj.weight', 'mlp.gate_up_proj.weight', 'mlp.down_proj.weight')

    @classmethod
    def _pretrained_config(cls, path):
        """HF config of the checkpoint; it must be this class's model_type: a glm4 checkpoint loaded as glm would drop
        its sandwich norms, a glm one loaded as glm4 would miss them"""
        config = super()._pretrained_config(path)
        mt = getattr(config, 'model_type', None)
        if mt != cls.model_type:
            other = {'glm': 'GlmForCausalLM', 'glm4': 'Glm4ForCausalLM'}.get(mt)
            raise ValueError(f'{path}: model_type {mt!r} is not {cls.model_type!r}'
                             + (f'; load it with {other}' if other else ''))
        return config

    def _rope_parameters(self):
        """(rope type, theta, partial_rotary_factor) from the config attributes or transformers-5 rope_parameters"""
        c = self.config
        rp = getattr(c, 'rope_parameters', None) or {}
        scaling = getattr(c, 'rope_scaling', None) or {}
        rtype = rp.get('rope_type') or scaling.get('rope_type') or scaling.get('type') or 'default'
        theta = float(getattr(c, 'rope_theta', None) or rp.get('rope_theta', 10000.0))
        # GlmConfig defaults the factor to 0.5 when a checkpoint does not name it
        factor = float(getattr(c, 'partial_rotary_factor', None) or rp.get('partial_rotary_factor', 0.5))
        return rtype, theta, factor

    def geometry(self):
        g = super().geometry()
        g['rotary_dim'] = int(g['head_dim'] * self._rope_parameters()[2])
        return g

    def rope_tables(self, max_pos):
        """cos / sin [max_pos, rotary_dim / 2] bf16: the first half of what GlmRotaryEmbedding.forward returns (fp32
        angles over the rotary dims, then cast to the model dtype); its apply_rotary_pos_emb repeats each entry for the
        pair (2i, 2i+1).  Only the default RoPE type exists for GLM here."""
        rtype, theta, _ = self._rope_parameters()
        if rtype != 'default':
            raise ValueError(f'Unknown RoPE scaling type {rtype}: GLM models support the default RoPE only')
        dim = self.geometry()['rotary_dim']
        dev = self.device
        inv_freq = 1.0 / (theta ** (torch.arange(0, dim, 2, dtype=torch.int64).float().to(dev) / dim))
        pos = torch.arange(max_pos, device=dev).float()
        freqs = pos[:, None] * inv_freq[None, :]
        return freqs.cos().to(torch.bfloat16).contiguous(), freqs.sin().to(torch.bfloat16).contiguous()

    def _runtime(self, max_seq, max_nodes, n_slots=1, keep_cache=False):
        self._check_fused_attn()   # before anything is captured
        rt = super()._runtime(max_seq, max_nodes, n_slots, keep_cache)
        if self.sandwich_norms:    # the post norms' output, outside any capture
            for b in (rt.decode_bufs, rt.prefill_bufs):
                if getattr(b, 'post_norm', None) is None:
                    b.post_norm = torch.zeros_like(b.y)
        return rt

    # the fused gate/up weight is the checkpoint's own gate_up_proj: nothing to concatenate
    def _fuse_mlp(self, layer):
        layer.mlp.gate_up_weight = layer.mlp.gate_up_proj.weight.data

    def _quantize_mlp(self, layer):
        m = layer.mlp
        gu = Fp8Linear(m.gate_up_weight, interleaved=True)
        m.gate_up_fp8 = gu
        m.gate_up_proj = Fp8Rows(gu, 0, gu.shape[0])
        m.gate_up_weight = None
        m.down_proj = Fp8Linear(m.down_proj.weight.data)


class Glm4ForCausalLM(GlmForCausalLM):
    model_cls = Glm4Model
    model_type = 'glm4'
    sandwich_norms = True


__all__ = ['GlmForCausalLM', 'Glm4ForCausalLM']
