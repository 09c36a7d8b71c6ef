# -*- coding: utf-8 -*-
"""Llama with the lookahead patch, H100-native.

Reference: /root/reference/lookahead/lookahead/models/llama/modeling_llama.py
  patch :584-588 (rank-4 mask -> position_ids = rowsum-1, additive mask), attention :243-308, RoPE :93-169,
  RMSNorm :76-90, MLP :172-186, LM head :768-769.
The module tree and parameter names are HF's (so checkpoints load unchanged); the forward over a draft of
<= 64/128 tree nodes runs on static buffers:  fused QKV / gate-up cuBLAS GEMMs + libpia_b200 kernels
(rmsnorm+residual, rope+kv-append into a preallocated cache, wgmma tree attention, silu*mul).  The rank-4 mask
is never built: `mask` is the per-node ancestor bit set, the prefix is implicit."""
import glob
import json
import math
import os

import torch
from torch import nn

from ...common import ops
from ...common.pretrained_model import LookaheadPreTrainedModel


class LlamaRMSNorm(nn.Module):
    def __init__(self, hidden_size, eps=1e-6, device=None, dtype=None):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size, device=device, dtype=dtype))
        self.variance_epsilon = eps


class LlamaAttention(nn.Module):
    def __init__(self, cfg, device, dtype, qkv_bias=False):
        super().__init__()
        hd = cfg.hidden_size // cfg.num_attention_heads
        kv = getattr(cfg, 'num_key_value_heads', None) or cfg.num_attention_heads
        kw = dict(bias=False, device=device, dtype=dtype)
        qkw = dict(kw, bias=qkv_bias)
        self.q_proj = nn.Linear(cfg.hidden_size, cfg.num_attention_heads * hd, **qkw)
        self.k_proj = nn.Linear(cfg.hidden_size, kv * hd, **qkw)
        self.v_proj = nn.Linear(cfg.hidden_size, kv * hd, **qkw)
        self.o_proj = nn.Linear(cfg.num_attention_heads * hd, cfg.hidden_size, **kw)


class LlamaMLP(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        kw = dict(bias=False, device=device, dtype=dtype)
        self.gate_proj = nn.Linear(cfg.hidden_size, cfg.intermediate_size, **kw)
        self.up_proj = nn.Linear(cfg.hidden_size, cfg.intermediate_size, **kw)
        self.down_proj = nn.Linear(cfg.intermediate_size, cfg.hidden_size, **kw)


def _gate_up_order(w, inverse=False, vec=False):
    """[..., gate (I rows); up (I rows), K] <-> the SiLU*up epilogue's row order (ops.interleave_gate_up), for any
    leading dims (stacked experts); vec: per-row values [..., 2I] (the scales)"""
    x = w.unsqueeze(-1) if vec else w
    two_i, K = x.shape[-2:]
    lead = x.shape[:-2]
    if inverse:
        y = x.reshape(*lead, two_i // 128, 2, 64, K).transpose(-4, -3)
    else:
        y = x.reshape(*lead, 2, two_i // 128, 64, K).transpose(-4, -3)
    y = y.reshape(*lead, two_i, K).contiguous()
    return y.squeeze(-1) if vec else y


class Fp8Linear(nn.Module):
    """fp8 (e4m3) weight of one projection, or of G stacked ones (the MoE experts), stored once, in the fp8 GEMM's
    HBM-tiled layout: `qweight` uint8 (ops.tile_weight_fp8), `scale` fp32, one per stored row (ops.quantize_fp8).
    `interleaved`: a fused gate/up weight whose rows are stored in the SiLU*up epilogue's order."""

    def __init__(self, w, interleaved=False):
        super().__init__()
        self.shape = tuple(w.shape)
        self.interleaved = interleaved
        if interleaved:   # quantisation is per row, so reordering rows first gives the same codes and scales
            w = _gate_up_order(w)
        q, s = ops.quantize_fp8(w)
        self.qweight = nn.Parameter(ops.tile_weight_fp8(q), requires_grad=False)
        self.scale = nn.Parameter(s, requires_grad=False)

    def codes(self):
        """(q e4m3 [..., N, K], s fp32 [..., N]) in the checkpoint's row order"""
        q, s = ops.untile_weight_fp8(self.qweight), self.scale.data
        if self.interleaved:
            q = _gate_up_order(q.view(torch.uint8), inverse=True).view(torch.float8_e4m3fn)
            s = _gate_up_order(s, inverse=True, vec=True)
        return q, s

    def dequantize(self):
        """the weight the fp8 GEMM multiplies with: float(q) * s, fp32"""
        q, s = self.codes()
        return q.float() * s.unsqueeze(-1)


class Fp8Rows(nn.Module):
    """rows [r0, r1) of a fused Fp8Linear under their HF name (q_proj / k_proj / v_proj, gate_proj / up_proj); the
    bytes belong to the fused weight, `bias` (Qwen2) stays the bf16 parameter it was"""

    def __init__(self, fused, r0, r1, bias=None):
        super().__init__()
        self._fused = (fused,)   # a tuple: not a submodule, its parameters are counted once
        self.r0, self.r1 = r0, r1
        self.shape = (r1 - r0, fused.shape[-1])
        self.bias = bias

    def codes(self):
        q, s = self._fused[0].codes()
        return q[self.r0:self.r1], s[self.r0:self.r1]

    def dequantize(self):
        q, s = self.codes()
        return q.float() * s.unsqueeze(-1)


class Int4Linear(nn.Module):
    """4-bit weight of one projection, as a GPTQ / compressed-tensors checkpoint stores it, in the int4 GEMM's layout:
    `qweight` uint8 (ops.tile_weight_w4 of the codes), `scale` [G, N] in the checkpoint's scale dtype, `zero` uint8
    [G, N] zero points (G = K / group_size).  `interleaved`: a fused gate/up weight whose rows (with their scales and zero
    points) are stored in the SiLU*up epilogue's order."""

    def __init__(self, u, s, z, group_size, interleaved=False):
        super().__init__()
        self.shape = tuple(u.shape)
        self.group_size = int(group_size)
        self.interleaved = interleaved
        if interleaved:
            u, s, z = _gate_up_order(u), _gate_up_order(s), _gate_up_order(z)
        self.qweight = nn.Parameter(ops.tile_weight_w4(u), requires_grad=False)
        self.scale = nn.Parameter(s.t().contiguous(), requires_grad=False)
        self.zero = nn.Parameter(z.t().contiguous(), requires_grad=False)

    def codes(self):
        """(u uint8 [N, K], s [N, G], z uint8 [N, G]) in the checkpoint's row order"""
        u = ops.untile_weight_w4(self.qweight, self.shape[1])
        s, z = self.scale.data.t(), self.zero.data.t()
        if self.interleaved:
            u, s, z = (_gate_up_order(t, inverse=True) for t in (u, s, z))
        return u, s.contiguous(), z.contiguous()

    def dequantize(self):
        """the weight the int4 GEMM multiplies with (ops.dequantize_w4), bf16 [N, K]"""
        return ops.dequantize_w4(*self.codes(), self.group_size)

    def gemm(self, x, **kw):
        return ops.Gemm.w4(self.qweight, self.scale, self.zero, self.group_size, x, **kw)


class Int4Rows(Fp8Rows):
    """rows [r0, r1) of a fused Int4Linear under their HF name; `bias` (Qwen2) stays the bf16 parameter it was"""

    def codes(self):
        u, s, z = self._fused[0].codes()
        return u[self.r0:self.r1], s[self.r0:self.r1], z[self.r0:self.r1]

    def dequantize(self):
        return ops.dequantize_w4(*self.codes(), self._fused[0].group_size)


def _w4_spec(config):
    """the int4 layout a checkpoint's quantization_config describes -> dict(format='gptq' | 'compressed-tensors',
    group_size (None: channel-wise), sym); ValueError naming the field for anything the int4 GEMM does not run"""
    q = getattr(config, 'quantization_config', None)
    q = q.to_dict() if hasattr(q, 'to_dict') else dict(q)
    method = q.get('quant_method')
    if method == 'gptq':
        if q.get('bits') != 4:
            raise ValueError(f'quantization_config.bits={q.get("bits")!r}: only 4-bit GPTQ checkpoints are supported')
        if q.get('desc_act'):
            raise ValueError('quantization_config.desc_act=True: act-order GPTQ checkpoints are not supported')
        if (q.get('checkpoint_format') or 'gptq') != 'gptq':
            raise ValueError(f'quantization_config.checkpoint_format={q.get("checkpoint_format")!r}: only the v1 '
                             "'gptq' format (zero points stored minus one) is supported")
        if q.get('lm_head'):
            raise ValueError('quantization_config.lm_head=True: a quantised lm_head is not supported')
        gs, sym = q.get('group_size', 128), q.get('sym', True)
    elif method == 'compressed-tensors':
        if q.get('format') != 'pack-quantized':
            raise ValueError(f'quantization_config.format={q.get("format")!r}: only compressed-tensors '
                             "'pack-quantized' int4 checkpoints are supported")
        groups = list((q.get('config_groups') or {}).values())
        if not groups:
            raise ValueError('quantization_config.config_groups is empty')
        w = groups[0].get('weights') or {}
        for g in groups:
            if g.get('weights') != w:
                raise ValueError('quantization_config.config_groups: groups with different weight schemes are not '
                                 'supported')
            if g.get('input_activations') is not None:
                raise ValueError('quantization_config.config_groups.input_activations: only weight-only (W4A16) '
                                 'checkpoints are supported')
            if g.get('targets') != ['Linear']:
                raise ValueError(f'quantization_config.config_groups.targets={g.get("targets")!r}: only Linear targets '
                                 'are supported')
        if w.get('num_bits') != 4:
            raise ValueError(f'quantization_config weights.num_bits={w.get("num_bits")!r}: only 4-bit weights are '
                             'supported')
        if w.get('type', 'int') != 'int':
            raise ValueError(f'quantization_config weights.type={w.get("type")!r}: only int weights are supported')
        if w.get('actorder') not in (None, False):
            raise ValueError(f'quantization_config weights.actorder={w.get("actorder")!r}: act-order is not supported')
        strategy = w.get('strategy')
        if strategy not in ('group', 'channel'):
            raise ValueError(f'quantization_config weights.strategy={strategy!r}: only group and channel are supported')
        if w.get('dynamic'):
            raise ValueError('quantization_config weights.dynamic=True is not supported')
        ignore = q.get('ignore') or []
        if not any(i == 'lm_head' or (i.startswith('re:') and 'lm_head' in i) for i in ignore):
            raise ValueError(f'quantization_config.ignore={ignore!r} does not hold lm_head: a quantised lm_head is not '
                             'supported')
        gs, sym = (w.get('group_size') if strategy == 'group' else -1), w.get('symmetric', True)
    else:
        raise ValueError(f'quantization_config.quant_method={method!r}: only gptq and compressed-tensors '
                         '(pack-quantized) 4-bit checkpoints are supported')
    if gs in (None, -1):
        gs = None
    elif int(gs) <= 0 or int(gs) % 128:
        raise ValueError(f'quantization_config group_size={gs}: the int4 GEMM takes groups of a multiple of 128 '
                         'weights (or channel-wise scales)')
    c = config
    hd = c.hidden_size // c.num_attention_heads
    kv = getattr(c, 'num_key_value_heads', None) or c.num_attention_heads
    for field, v in (('hidden_size', c.hidden_size), ('intermediate_size', c.intermediate_size),
                     ('num_attention_heads * head_dim', c.num_attention_heads * hd),
                     ('num_key_value_heads * head_dim', kv * hd)):
        if v % 128:
            raise ValueError(f'{field}={v}: int4 weights need every projection dimension divisible by 128')
        if gs is not None and field in ('hidden_size', 'intermediate_size') and v % int(gs):
            raise ValueError(f'{field}={v} is not a multiple of quantization_config group_size={gs}')
    return dict(format=method, group_size=int(gs) if gs is not None else None, sym=bool(sym))


class LlamaDecoderLayer(nn.Module):
    qkv_bias = False   # biases on q/k/v (Qwen2); o_proj never has one

    def __init__(self, cfg, device, dtype):
        super().__init__()
        self.self_attn = LlamaAttention(cfg, device, dtype, qkv_bias=self._qkv_bias(cfg))
        self.mlp = self._make_mlp(cfg, device, dtype)
        self.input_layernorm = LlamaRMSNorm(cfg.hidden_size, cfg.rms_norm_eps, device, dtype)
        self.post_attention_layernorm = LlamaRMSNorm(cfg.hidden_size, cfg.rms_norm_eps, device, dtype)

    def _qkv_bias(self, cfg):
        """whether q/k/v carry biases: the class's flag (a family may read it from the config instead)"""
        return self.qkv_bias

    def _make_mlp(self, cfg, device, dtype):
        return LlamaMLP(cfg, device, dtype)


class LlamaModel(nn.Module):
    layer_cls = LlamaDecoderLayer

    def __init__(self, cfg, device, dtype):
        super().__init__()
        self.embed_tokens = nn.Embedding(cfg.vocab_size, cfg.hidden_size, device=device, dtype=dtype)
        self.layers = nn.ModuleList([self.layer_cls(cfg, device, dtype) for _ in range(cfg.num_hidden_layers)])
        self.norm = LlamaRMSNorm(cfg.hidden_size, cfg.rms_norm_eps, device, dtype)


class LlamaForCausalLM(LookaheadPreTrainedModel):
    model_cls = LlamaModel
    rotary_interleaved = False   # GLM: RoPE on the first geometry()['rotary_dim'] dims of a head, in (2i, 2i+1) pairs
    sandwich_norms = False       # GLM-4-0414: RMSNorm of each sublayer's output before its residual add
    # where RMSNorm rounds the normalised value: once, bf16(w * x_hat) (llama/modeling_llama.py:90), or twice,
    # bf16(w * bf16(x_hat)) (the families whose norm casts x_hat to bf16 before the weight multiply; DESIGN.md)
    rmsnorm_rounding = ops.ROUND_ONCE
    # whether from_pretrained reads GPTQ / compressed-tensors int4 checkpoints (the Llama decoder's projections);
    # families that refuse or ignore quantization_config set False
    int4_checkpoints = True

    def __init__(self, config, device=None, dtype=torch.bfloat16):
        super().__init__(config)
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else 'meta'
        assert dtype == torch.bfloat16, 'the H100 path computes in bf16'
        self.model = self.model_cls(config, device, dtype)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False, device=device, dtype=dtype)
        self._fused = False
        self._fp8 = False
        self._w4 = False
        for p_ in self.parameters():  # inference only: no autograd state on the hot path
            p_.requires_grad_(False)

    # ------------------------------------------------------------------ weights
    @torch.no_grad()
    def init_weights(self, seed=0, std=0.02):
        """random-init weights of the configured shape (there are no checkpoints offline)"""
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed)
        for name, p in self.named_parameters():
            if name.endswith('layernorm.weight') or name.endswith('norm.weight'):
                p.fill_(1.0)
            else:
                p.normal_(0.0, std, generator=gen)
        return self

    @staticmethod
    def _shards(path):
        files = sorted(glob.glob(os.path.join(path, '*.safetensors')))
        if files:
            from safetensors.torch import load_file
            return (load_file(f) for f in files)
        return (torch.load(f, map_location='cpu') for f in sorted(glob.glob(os.path.join(path, 'pytorch_model*.bin'))))

    @classmethod
    def from_pretrained(cls, path, torch_dtype=torch.bfloat16, device=None, quantization=None, **kwargs):
        """HF checkpoint directory (config.json + *.safetensors / pytorch_model*.bin) -> model on the GPU.
        quantization='fp8': the decoder projections become fp8 weights as they arrive (see quantize_fp8); the bf16
        decoder never exists on the GPU.  A GPTQ or compressed-tensors int4 checkpoint (config.quantization_config) is
        loaded as it is stored, one layer at a time, onto the int4 GEMM (see _w4_spec for what is accepted)."""
        if quantization not in (None, 'fp8'):
            raise ValueError(f'quantization={quantization!r}: only None and \'fp8\' are supported')
        config = cls._pretrained_config(path)
        if cls.int4_checkpoints and getattr(config, 'quantization_config', None):
            spec = _w4_spec(config)
            if quantization is not None:
                raise ValueError(f'quantization={quantization!r}: this checkpoint is already quantised '
                                 f'({spec["format"]} int4); load it with quantization=None')
            return cls._from_pretrained_w4(path, config, spec, device)
        if quantization == 'fp8':
            return cls._from_pretrained_fp8(path, config, device)
        model = cls(config, device=device, dtype=torch_dtype)
        own = dict(model.named_parameters())
        seen = set()
        shards = cls._shards(path)
        with torch.no_grad():
            for sd in shards:
                for k, v in model._convert_checkpoint_keys(sd).items():
                    if k in own:
                        own[k].copy_(v.to(torch_dtype))
                        seen.add(k)
        if 'lm_head.weight' not in seen and getattr(config, 'tie_word_embeddings', False):
            with torch.no_grad():
                model.lm_head.weight.copy_(model.model.embed_tokens.weight)
            seen.add('lm_head.weight')
        missing = [k for k in own if k not in seen]
        if missing:
            raise RuntimeError(f'checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}')
        return model

    @classmethod
    def _pretrained_config(cls, path):
        """the config of a checkpoint directory (HF format: AutoConfig)"""
        from transformers import AutoConfig
        return AutoConfig.from_pretrained(path)

    # the parameters of a decoder layer that fp8 mode quantises (relative to the layer)
    _fp8_params = ('self_attn.q_proj.weight', 'self_attn.k_proj.weight', 'self_attn.v_proj.weight',
                   'self_attn.o_proj.weight', 'mlp.gate_proj.weight', 'mlp.up_proj.weight', 'mlp.down_proj.weight')

    @classmethod
    def _fp8_skeleton(cls, config, device):
        """the model on the meta device with everything but the quantised projections allocated (uninitialised) on
        the GPU.  Returns (model, {name: allocated parameter}, layer_of(name) -> layer index of a quantised projection
        or None, materialise(name) -> that projection allocated in bf16 on the GPU)"""
        dev = device if device is not None else torch.device('cuda', torch.cuda.current_device())
        model = cls(config, device='meta')

        def layer_of(name):
            parts = name.split('.')
            if name.startswith('model.layers.') and '.'.join(parts[3:]) in cls._fp8_params:
                return int(parts[2])
            return None

        def materialise(name):
            mod_name, _, pname = name.rpartition('.')
            mod = model.get_submodule(mod_name)
            old = getattr(mod, pname)
            setattr(mod, pname, nn.Parameter(torch.empty(old.shape, dtype=old.dtype, device=dev), requires_grad=False))
            return getattr(mod, pname)

        own = {name: materialise(name) for name, _ in list(model.named_parameters()) if layer_of(name) is None}
        return model, own, layer_of, materialise

    @classmethod
    @torch.no_grad()
    def build_fp8(cls, config, fill_rest, fill_weight, device=None):
        """An fp8 model without a checkpoint and without its bf16 decoder ever existing: fill_rest(model) initialises
        the parameters that stay bf16 (the quantised projections are still meta tensors then, and may be skipped);
        then, one layer at a time, fill_weight(name, tensor) fills each projection in a bf16 buffer (HF names, e.g.
        'model.layers.3.self_attn.q_proj.weight'), which is fused, quantised and freed.  Gives the bytes of
        quantize_fp8() on a bf16 model filled the same way."""
        model, _, _, materialise = cls._fp8_skeleton(config, device)
        fill_rest(model)
        for li, layer in enumerate(model.model.layers):
            for p in cls._fp8_params:
                name = f'model.layers.{li}.{p}'
                fill_weight(name, materialise(name))
            model._fuse_layer(layer)
            model._quantize_layer(layer)
        model._fused = True
        model._fp8 = True
        return model

    @classmethod
    @torch.no_grad()
    def _from_pretrained_fp8(cls, path, config, device):
        """The model is built on the meta device; everything but the quantised projections is allocated on the GPU up
        front.  A layer's projections wait on the host until the layer is complete, then that one layer is allocated
        in bf16, filled, fused and quantised, so the GPU holds the fp8 model plus at most one bf16 layer."""
        model, own, layer_of, materialise = cls._fp8_skeleton(config, device)
        n_layers = len(model.model.layers)
        pending = {li: {} for li in range(n_layers)}
        seen = set()
        for sd in cls._shards(path):
            for k, v in model._convert_checkpoint_keys(sd).items():
                li = layer_of(k)
                if li is not None and li in pending:
                    pending[li][k] = v
                    if len(pending[li]) == len(cls._fp8_params):
                        for name, t in pending.pop(li).items():
                            materialise(name).copy_(t.to(torch.bfloat16))
                        layer = model.model.layers[li]
                        model._fuse_layer(layer)
                        model._quantize_layer(layer)
                elif k in own:
                    own[k].copy_(v.to(torch.bfloat16))
                    seen.add(k)
        if 'lm_head.weight' not in seen and getattr(config, 'tie_word_embeddings', False):
            model.lm_head.weight.copy_(model.model.embed_tokens.weight)
            seen.add('lm_head.weight')
        missing = [k for k in own if k not in seen]
        missing += [f'model.layers.{li}.{p}' for li, got in pending.items() for p in cls._fp8_params
                    if f'model.layers.{li}.{p}' not in got]
        if missing:
            raise RuntimeError(f'checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}')
        model._fused = True
        model._fp8 = True
        return model

    # ------------------------------------------------------------------ int4 (GPTQ / compressed-tensors) weights
    _W4_PARTS = {'compressed-tensors': ('weight_packed', 'weight_scale', 'weight_shape', 'weight_zero_point',
                                        'weight_g_idx'),
                 'gptq': ('qweight', 'qzeros', 'scales', 'g_idx')}

    @classmethod
    def _w4_unpack(cls, spec, t, name):
        """one projection's checkpoint tensors {part: tensor} -> (u, s, z, group size) (ops' internal form)"""
        if spec['format'] == 'gptq':
            if 'qweight' not in t or 'qzeros' not in t or 'scales' not in t:
                raise RuntimeError(f'checkpoint is missing GPTQ tensors of {name}: has {sorted(t)}')
            out = ops.unpack_gptq_w4(t['qweight'], t['qzeros'], t['scales'], t.get('g_idx'))
        else:
            if 'weight_g_idx' in t:
                raise ValueError(f'{name}.weight_g_idx: act-order compressed-tensors checkpoints are not supported')
            if 'weight_packed' not in t or 'weight_scale' not in t or (not spec['sym'] and 'weight_zero_point' not in t):
                raise RuntimeError(f'checkpoint is missing compressed-tensors tensors of {name}: has {sorted(t)}')
            out = ops.unpack_compressed_tensors_w4(t['weight_packed'], t['weight_scale'], t.get('weight_shape'),
                                                   t.get('weight_zero_point') if not spec['sym'] else None)
        gs = spec['group_size'] or out[0].shape[1]
        if out[3] != gs:
            raise ValueError(f'{name}: the stored scales give group size {out[3]}, quantization_config says {gs}')
        return out

    def _install_w4_layer(self, layer, w):
        """the layer's projections from {'q_proj': (u, s, z, gs), ...}: q|k|v and gate|up fused by rows (with their
        scales and zero points), the HF names become Int4Rows views of the fused weights"""
        a, m = layer.self_attn, layer.mlp
        cat = lambda names, i: torch.cat([w[n][i] for n in names], dim=0).contiguous()
        qkv_names = ('q_proj', 'k_proj', 'v_proj')
        for names in (qkv_names, ('gate_proj', 'up_proj')):
            if len({w[n][3] for n in names}) != 1:
                raise ValueError(f'{"/".join(names)} have different group sizes: they cannot be fused')
        nq, nk = w['q_proj'][0].shape[0], w['k_proj'][0].shape[0]
        qkv = Int4Linear(cat(qkv_names, 0), cat(qkv_names, 1), cat(qkv_names, 2), w['q_proj'][3])
        a.qkv_w4 = qkv
        a.qkv_bias = None
        if a.q_proj.bias is not None:
            a.qkv_bias = torch.cat([a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data]).contiguous()
        a.q_proj = Int4Rows(qkv, 0, nq, a.q_proj.bias)
        a.k_proj = Int4Rows(qkv, nq, nq + nk, a.k_proj.bias)
        a.v_proj = Int4Rows(qkv, nq + nk, qkv.shape[0], a.v_proj.bias)
        a.qkv_weight = None
        a.o_proj = Int4Linear(*w['o_proj'])
        ni = w['gate_proj'][0].shape[0]
        gu_names = ('gate_proj', 'up_proj')
        gu = Int4Linear(cat(gu_names, 0), cat(gu_names, 1), cat(gu_names, 2), w['gate_proj'][3], interleaved=True)
        m.gate_up_w4 = gu
        m.gate_proj, m.up_proj = Int4Rows(gu, 0, ni), Int4Rows(gu, ni, 2 * ni)
        m.gate_up_weight = None
        m.down_proj = Int4Linear(*w['down_proj'])

    @classmethod
    @torch.no_grad()
    def _from_pretrained_w4(cls, path, config, spec, device):
        """As _from_pretrained_fp8: everything but the decoder projections is allocated up front; a layer's packed
        tensors wait on the host until the layer is complete, then they are unpacked and tiled on the GPU, so no bf16
        projection ever exists there."""
        model, own, layer_of, _ = cls._fp8_skeleton(config, device)
        dev = model.model.norm.weight.device
        parts = cls._W4_PARTS[spec['format']]
        need = {'qweight', 'qzeros', 'scales'} if spec['format'] == 'gptq' else \
            {'weight_packed', 'weight_scale', 'weight_shape'} | (set() if spec['sym'] else {'weight_zero_point'})
        pending = {li: {} for li in range(len(model.model.layers))}
        seen = set()

        def complete(li):
            return all(need <= pending[li].get(f'model.layers.{li}.{p[:-len(".weight")]}', {}).keys()
                       for p in cls._fp8_params)

        def finish(li):
            got = pending.pop(li)
            w = {}
            for p in cls._fp8_params:
                name = f'model.layers.{li}.{p[:-len(".weight")]}'
                w[p.rsplit('.', 2)[-2]] = cls._w4_unpack(spec, {k: v.to(dev) for k, v in got.get(name, {}).items()},
                                                         name)
            model._install_w4_layer(model.model.layers[li], w)

        for sd in cls._shards(path):
            for k, v in model._convert_checkpoint_keys(sd).items():
                base, _, part = k.rpartition('.')
                li = layer_of(base + '.weight') if part in parts else None
                if li is not None and li in pending:
                    pending[li].setdefault(base, {})[part] = v
                elif part in parts and k.startswith(('lm_head.', 'model.embed_tokens.')):
                    raise ValueError(f'{k}: a quantised {k.split(".")[0]} is not supported (it stays bf16)')
                elif k in own:
                    own[k].copy_(v.to(torch.bfloat16))
                    seen.add(k)
            # layers are finished at the end of a shard, so that an optional tensor (g_idx) stored after the required
            # ones in the same shard is not missed
            for li in [li for li in pending if complete(li)]:
                finish(li)
        if 'lm_head.weight' not in seen and getattr(config, 'tie_word_embeddings', False):
            model.lm_head.weight.copy_(model.model.embed_tokens.weight)
            seen.add('lm_head.weight')
        missing = [k for k in own if k not in seen]
        missing += [f'model.layers.{li}.* ({sorted(got)[:2]})' for li, got in pending.items()]
        if missing:
            raise RuntimeError(f'checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}')
        model._fused = True
        model._w4 = True
        return model

    @classmethod
    @torch.no_grad()
    def build_w4(cls, config, fill_rest, fill_codes, device=None):
        """An int4 model without a checkpoint (synthetic weights, e.g. the benchmark's 70B shape): fill_rest(model)
        initialises the parameters that stay bf16 (the projections are still meta tensors then); then, one layer at a
        time, fill_codes(name, (N, K)) returns each projection's (u, s, z, group size) in ops' internal form on the
        GPU (HF names, e.g. 'model.layers.3.self_attn.q_proj.weight')."""
        model, _, _, _ = cls._fp8_skeleton(config, device)
        fill_rest(model)
        for li, layer in enumerate(model.model.layers):
            w = {}
            for p in cls._fp8_params:
                mod = layer.get_submodule(p[:-len('.weight')])
                w[p.rsplit('.', 2)[-2]] = fill_codes(f'model.layers.{li}.{p}', tuple(mod.weight.shape))
            model._install_w4_layer(layer, w)
        model._fused = True
        model._w4 = True
        return model

    def _w4_plans(self, b):
        """int4 GEMM plans of one activation buffer set, on the buffers (as _fp8_plans); the bf16 GEMM selection knobs
        are refused"""
        plans = getattr(b, 'w4_plans', None)
        if plans is not None:
            return plans
        if os.environ.get('PIA_GEMM', '1') == '0' or 'PIA_GEMM_SET' in os.environ:
            raise ValueError('this model holds int4 weights, which only the int4 GEMM runs: PIA_GEMM=0 / PIA_GEMM_SET '
                             'do not apply')
        b.fp8_out = torch.zeros((b.rows, self.config.hidden_size), dtype=torch.bfloat16, device=b.y.device)
        if getattr(b, 'act', None) is None or b.act.shape[0] != b.rows:
            b.act = torch.zeros((b.rows, self.config.intermediate_size), dtype=torch.bfloat16, device=b.y.device)
        n_sm = torch.cuda.get_device_properties(b.y.device).multi_processor_count
        plans = {'layers': []}
        for layer in self.model.layers:
            a, m = layer.self_attn, layer.mlp
            bias = a.qkv_bias.float() if a.qkv_bias is not None else None
            # the int4 GEMM's k chunk is 256 wide: _fp8_split's rule over chunks of that size
            split = lambda w: self._fp8_split(torch.empty((w.shape[0], -(-w.shape[1] // 256) * 128), device='meta'), n_sm)
            plans['layers'].append({
                'qkv': a.qkv_w4.gemm(b.y, bias=bias, split_k=split(a.qkv_w4), out=b.qkv),
                'o': a.o_proj.gemm(b.attn, split_k=split(a.o_proj), out=b.fp8_out),
                'gate_up_silu': m.gate_up_w4.gemm(b.y, out=b.act).set_silu(),
                'down': m.down_proj.gemm(b.act, split_k=split(m.down_proj), out=b.fp8_out)})
        b.w4_plans = plans
        return plans

    def _convert_checkpoint_keys(self, sd):
        """checkpoint tensor names -> this module tree's names (identity for Llama / Mistral)"""
        return sd

    def fuse(self):
        """QKV and gate/up weights (and the QKV biases, if any) into single GEMM operands; the HF-named parameters
        become views of them"""
        if self._fused:
            return
        for layer in self.model.layers:
            self._fuse_layer(layer)
        self._fused = True

    def _fuse_layer(self, layer):
        a = layer.self_attn
        w = torch.cat([a.q_proj.weight.data, a.k_proj.weight.data, a.v_proj.weight.data], dim=0).contiguous()
        nq, nk = a.q_proj.weight.shape[0], a.k_proj.weight.shape[0]
        a.q_proj.weight.data, a.k_proj.weight.data, a.v_proj.weight.data = w[:nq], w[nq:nq + nk], w[nq + nk:]
        a.qkv_weight = w
        a.qkv_bias = None
        if a.q_proj.bias is not None:
            bias = torch.cat([a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data]).contiguous()
            a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data = bias[:nq], bias[nq:nq + nk], bias[nq + nk:]
            a.qkv_bias = bias
        self._fuse_mlp(layer)

    def _fuse_mlp(self, layer):
        m = layer.mlp
        w = torch.cat([m.gate_proj.weight.data, m.up_proj.weight.data], dim=0).contiguous()
        ni = m.gate_proj.weight.shape[0]
        m.gate_proj.weight.data, m.up_proj.weight.data = w[:ni], w[ni:]
        m.gate_up_weight = w

    # ------------------------------------------------------------------ fp8 (e4m3) weight-only mode
    def _fp8_weight_shapes(self, layer):
        """(name, shape) of every weight of a fused layer that fp8 mode quantises"""
        a, m = layer.self_attn, layer.mlp
        return [('qkv', a.qkv_weight.shape), ('o_proj', a.o_proj.weight.shape), ('gate_up', m.gate_up_weight.shape),
                ('down_proj', m.down_proj.weight.shape)]

    @torch.no_grad()
    def quantize_fp8(self):
        """Convert the decoder projections (fused q/k/v, o, fused gate/up, down; Mixtral's experts) to per-row e4m3
        weights with fp32 scales (ops.quantize_fp8), in place and one layer at a time: each bf16 weight is freed once
        its fp8 copy exists.  Embeddings, lm_head, norms, the router and QKV biases stay bf16.  Every weight must have
        both dimensions divisible by 128; otherwise ValueError before anything is converted."""
        if self._fp8:
            return self
        if self._w4:
            raise ValueError('quantize_fp8(): this model holds int4 weights from its checkpoint; they cannot be '
                             're-quantised to fp8')
        self.fuse()
        for li, layer in enumerate(self.model.layers):
            for name, shape in self._fp8_weight_shapes(layer):
                if shape[-1] % 128 or shape[-2] % 128:
                    raise ValueError(f'layer {li} {name} {tuple(shape)}: fp8 weights need both dimensions divisible by 128')
        self._rt = None                               # drops the bf16 GEMM plans and the buffers bound to them
        self.__dict__.pop('_tiled_weights', None)     # and the bf16 HBM-tiled copies
        for layer in self.model.layers:
            self._quantize_layer(layer)
        self._fp8 = True
        return self

    def _quantize_layer(self, layer):
        a = layer.self_attn
        nq, nk = a.q_proj.weight.shape[0], a.k_proj.weight.shape[0]
        qkv = Fp8Linear(a.qkv_weight)
        a.qkv_fp8 = qkv
        a.q_proj = Fp8Rows(qkv, 0, nq, a.q_proj.bias)
        a.k_proj = Fp8Rows(qkv, nq, nq + nk, a.k_proj.bias)
        a.v_proj = Fp8Rows(qkv, nq + nk, qkv.shape[0], a.v_proj.bias)
        a.qkv_weight = None
        a.o_proj = Fp8Linear(a.o_proj.weight.data)
        self._quantize_mlp(layer)

    def _quantize_mlp(self, layer):
        m = layer.mlp
        ni = m.gate_proj.weight.shape[0]
        gu = Fp8Linear(m.gate_up_weight, interleaved=True)
        m.gate_up_fp8 = gu
        m.gate_proj, m.up_proj = Fp8Rows(gu, 0, ni), Fp8Rows(gu, ni, 2 * ni)
        m.gate_up_weight = None
        m.down_proj = Fp8Linear(m.down_proj.weight.data)

    @staticmethod
    def _fp8_split(w, n_sm):
        """K splits of an fp8 plan: 1 when the 128-row tiles alone come close to filling the SMs (or the plan uses the
        SiLU epilogue), else the smallest 2 / 4 / 8-CTA cluster split that does (cluster splits add the bias once and
        write bf16)"""
        tiles, chunks = w.shape[-2] // 128, w.shape[-1] // 128
        want = (n_sm * 7) // 8
        if tiles >= want:
            return 1
        best = 1
        for s in (2, 4, 8):
            if chunks >= s and -(-chunks // -(-chunks // s)) == s:
                best = s
                if tiles * s >= want:
                    break
        return -best if best > 1 else 1

    def _fp8_plans(self, b):
        """fp8 GEMM plans of one activation buffer set (the decode rows or the prefill pass's 256), on the buffers;
        there is no other path for fp8 weights, so the bf16 GEMM selection knobs are refused"""
        plans = getattr(b, 'fp8_plans', None)
        if plans is not None:
            return plans
        if os.environ.get('PIA_GEMM', '1') == '0' or 'PIA_GEMM_SET' in os.environ:
            raise ValueError('this model holds fp8 weights, which only the fp8 GEMM runs: PIA_GEMM=0 / PIA_GEMM_SET '
                             'do not apply')
        hid = self.config.hidden_size
        b.fp8_out = torch.zeros((b.rows, hid), dtype=torch.bfloat16, device=b.y.device)
        n_sm = torch.cuda.get_device_properties(b.y.device).multi_processor_count
        plans = {'layers': [self._layer_fp8_plans(layer, b, n_sm) for layer in self.model.layers]}
        b.fp8_plans = plans
        return plans

    def _attn_fp8_plans(self, layer, b, n_sm):
        a = layer.self_attn
        qkv, o = a.qkv_fp8, a.o_proj
        bias = a.qkv_bias.float() if a.qkv_bias is not None else None
        return {'qkv': ops.Gemm.fp8(qkv.qweight, qkv.scale, b.y, bias=bias, split_k=self._fp8_split(qkv, n_sm),
                                    out=b.qkv),
                'o': ops.Gemm.fp8(o.qweight, o.scale, b.attn, split_k=self._fp8_split(o, n_sm), out=b.fp8_out)}

    def _layer_fp8_plans(self, layer, b, n_sm):
        m = layer.mlp
        plans = self._attn_fp8_plans(layer, b, n_sm)
        if getattr(b, 'act', None) is None or b.act.shape[0] != b.rows:
            b.act = torch.zeros((b.rows, self.config.intermediate_size), dtype=torch.bfloat16, device=b.y.device)
        plans['gate_up_silu'] = ops.Gemm.fp8(m.gate_up_fp8.qweight, m.gate_up_fp8.scale, b.y, out=b.act).set_silu()
        plans['down'] = ops.Gemm.fp8(m.down_proj.qweight, m.down_proj.scale, b.act,
                                     split_k=self._fp8_split(m.down_proj, n_sm), out=b.fp8_out)
        return plans

    # ------------------------------------------------------------------ geometry / tables
    def geometry(self):
        c = self.config
        hd = c.hidden_size // c.num_attention_heads
        if getattr(c, 'head_dim', None) not in (None, hd):   # the projections are built hidden_size wide per head set
            raise ValueError(f'config head_dim {c.head_dim} differs from hidden_size // num_attention_heads = {hd}; '
                             'only configs where the two are equal are supported')
        return dict(n_layers=c.num_hidden_layers, hidden=c.hidden_size, n_q_heads=c.num_attention_heads,
                    n_kv_heads=getattr(c, 'num_key_value_heads', None) or c.num_attention_heads, head_dim=hd,
                    inter=c.intermediate_size, vocab=c.vocab_size)

    def rope_tables(self, max_pos):
        """cos/sin exactly as LlamaRotaryEmbedding.forward returns them (reference :100, :111-127): fp32 angles,
        then cast to the model dtype"""
        c = self.config
        hd = c.hidden_size // c.num_attention_heads
        rp = getattr(c, 'rope_parameters', None) or {}
        theta = float(getattr(c, 'rope_theta', None) or rp.get('rope_theta', 10000.0))
        scaling = getattr(c, 'rope_scaling', None) or ({k: v for k, v in rp.items() if k != 'rope_theta'} if rp else None)
        rtype = (scaling or {}).get('rope_type', (scaling or {}).get('type', 'default')) if scaling else 'default'
        dev = self.device
        inv_freq = 1.0 / (theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float().to(dev) / hd))
        pos = torch.arange(max_pos, device=dev).float()
        if rtype in (None, 'default'):
            pass
        elif rtype == 'linear':      # LlamaLinearScalingRotaryEmbedding (reference :130-146): t / factor
            pos = pos / float(scaling['factor'])
        elif rtype == 'dynamic':     # LlamaDynamicNTKScalingRotaryEmbedding (reference :149-169): base grows with seq_len
            factor, mpe = float(scaling['factor']), int(c.max_position_embeddings)
            if max_pos > mpe:
                base = theta * ((factor * max_pos / mpe) - (factor - 1)) ** (hd / (hd - 2))
                inv_freq = 1.0 / (base ** (torch.arange(0, hd, 2, dtype=torch.int64).float().to(dev) / hd))
        elif rtype == 'llama3':      # Llama 3.1 / 3.2: long wavelengths / factor, a smooth blend between the two bounds
            # (transformers' _compute_llama3_parameters, op for op, so the bf16 tables come out bit for bit; attention
            # factor 1)
            factor, low, high = float(scaling['factor']), float(scaling['low_freq_factor']), float(scaling['high_freq_factor'])
            old_ctx = scaling.get('original_max_position_embeddings') or c.max_position_embeddings
            low_freq_wavelen, high_freq_wavelen = old_ctx / low, old_ctx / high
            wavelen = 2 * math.pi / inv_freq
            inv_freq_llama = torch.where(wavelen > low_freq_wavelen, inv_freq / factor, inv_freq)
            smooth_factor = (old_ctx / wavelen - low) / (high - low)
            smoothed_inv_freq = (1 - smooth_factor) * inv_freq_llama / factor + smooth_factor * inv_freq_llama
            is_medium_freq = ~(wavelen < high_freq_wavelen) * ~(wavelen > low_freq_wavelen)
            inv_freq = torch.where(is_medium_freq, smoothed_inv_freq, inv_freq_llama)
        else:                        # the reference raises on unknown types as well (:241 `Unknown RoPE scaling type`)
            raise ValueError(f'Unknown RoPE scaling type {rtype}')
        freqs = pos[:, None] * inv_freq[None, :]
        return freqs.cos().to(torch.bfloat16).contiguous(), freqs.sin().to(torch.bfloat16).contiguous()

    # ------------------------------------------------------------------ weight-streaming GEMM plans (decode rows)
    def _gemm_plans(self, rt):
        """wgmma weight-streaming GEMMs (csrc/gemm_ws.cu) for the 64-row decode buffers: HBM-tiled copies of the
        fused weights, one plan per (weight, activation buffer).  Prefill passes (256 rows) stay on cuBLAS."""
        plans = getattr(rt, 'gemm_plans', None)
        if plans is not None:
            return plans
        if self._fp8 or self._w4:   # fp8 / int4 weights: their plans of both buffer sets, built here, outside any capture
            mk = self._fp8_plans if self._fp8 else self._w4_plans
            mk(rt.decode_bufs)
            mk(rt.prefill_bufs)
            rt.gemm_plans = False
            return False
        import os
        if os.environ.get('PIA_GEMM', '1') == '0' or rt.max_nodes != 64:
            rt.gemm_plans = False
            return False
        b = rt.decode_bufs
        g = rt.g
        dev = b.y.device
        b.gu = torch.zeros((b.rows, 2 * g['inter']), dtype=torch.bfloat16, device=dev)
        b.act = torch.zeros((b.rows, g['inter']), dtype=torch.bfloat16, device=dev)
        plans = {'layers': []}
        for layer in self.model.layers:
            plans['layers'].append(self._layer_gemm_plans(layer, b))
        plans['lm_head'] = self._mk_gemm(self.lm_head.weight.data, b.y)
        rt.gemm_plans = plans
        return plans

    def _layer_gemm_plans(self, layer, b):
        """Which projections go through k_gemm_ws is decided by measurement (H100 80GB HBM3 SXM, 700 W; Llama-2-7B
        shapes; whole verify forward as one CUDA graph, scripts/microbench.py --forward-only, us per forward): gate_up
        only 6179; gate_up with the SiLU*up epilogue + down 6249; gate_up + down as a 4-CTA cluster split-K (fp32
        partials reduced through DSMEM) 6353; + o (cluster 4) 6622; + qkv (cluster 2) 6795 - on the narrow
        projections (32 / 96 weight tiles on 132 SMs) cuBLAS is faster.  PIA_GEMM_SET overrides the set."""
        import os
        want = os.environ.get('PIA_GEMM_SET', 'gate_up').split(',')
        if ('qkv' in want or 'qkv2' in want) and layer.self_attn.qkv_bias is not None:
            raise ValueError('PIA_GEMM_SET names qkv, but this model has QKV biases and k_gemm_ws has no bias epilogue')
        plans = {}
        if 'gate_up_silu' in want and layer.mlp.gate_up_weight.shape[0] % 256 == 0:
            # SiLU(gate) * up in the GEMM epilogue: every 128-row weight tile holds 64 gate rows + the 64 up rows of the same
            # columns (ops.interleave_gate_up), the plan writes act [rows, inter] directly
            cache = self.__dict__.setdefault('_tiled_weights', {})
            key = ('gate_up_silu', layer.mlp.gate_up_weight.data_ptr())
            if key not in cache:
                cache[key] = ops.tile_weight(ops.interleave_gate_up(layer.mlp.gate_up_weight))
            plans['gate_up_silu'] = ops.Gemm(cache[key], b.y, tiled=True).set_silu()
        elif 'gate_up' in want or 'gate_up_silu' in want:
            plans['gate_up'] = self._mk_gemm(layer.mlp.gate_up_weight, b.y)
        if 'qkv' in want:
            plans['qkv'] = self._mk_gemm(layer.self_attn.qkv_weight, b.y)
        sk = int(os.environ.get('PIA_GEMM_SPLIT', '-4'))   # > 1: fp32 slices summed by the next rmsnorm; < -1: cluster
        if 'qkv2' in want:
            plans['qkv'] = self._mk_gemm(layer.self_attn.qkv_weight, b.y, split_k=-2)
        if 'o' in want:
            plans['o'] = self._mk_gemm(layer.self_attn.o_proj.weight.data, b.attn, split_k=sk)
        if 'down' in want and layer.mlp.down_proj.weight.shape[1] % 64 == 0 and layer.mlp.down_proj.weight.shape[1] >= 64 * abs(sk):
            plans['down'] = self._mk_gemm(layer.mlp.down_proj.weight.data, b.act, split_k=sk)
        for name in os.environ.get('PIA_GEMM_NOPDL', '').split(','):   # experiment knob: plain kernel boundaries
            if name in plans:
                plans[name].set_pdl(False)
        return plans

    def _mk_gemm(self, w, x, split_k=1):
        """HBM-tiled copy of the weight when its row count allows it (N % 128 == 0), else the row-major tensor.
        The tiled copies belong to the model (one per weight), not to a runtime: rebuilding the runtime for a longer
        max_seq or another slot count must not duplicate 9 GB of weights"""
        if w.shape[0] % 128 == 0:
            cache = self.__dict__.setdefault('_tiled_weights', {})
            key = (w.data_ptr(), tuple(w.shape))
            if key not in cache:
                cache[key] = ops.tile_weight(w)
            return ops.Gemm(cache[key], x, split_k=split_k, tiled=True)
        return ops.Gemm(w.contiguous(), x, split_k=split_k)

    # ------------------------------------------------------------------ weight prefetch beside the small kernels
    def _prefetch_cfg(self, rt):
        """PIA_PREFETCH="o_frac,gate_up_frac,down_frac,gbytes_per_s" (0 disables): which share of the next
        projections' weights is pulled into L2 on a side stream while RoPE + tree attention (o, gate_up) and
        SiLU*up (down) keep HBM idle; the step is weight-streaming bound, so HBM time hidden here comes straight
        off the step.  Decode steps only."""
        cfg = getattr(rt, 'prefetch_cfg', None)
        if cfg is None:
            import os
            spec = os.environ.get('PIA_PREFETCH', '0')
            v = [float(t) for t in spec.split(',')] if spec not in ('', '0') else []
            cfg = False
            if v and torch.cuda.is_available():
                v = (v + [0.0] * 4)[:4]
                cfg = dict(o=v[0], gate_up=v[1], down=v[2], rate=v[3], side=torch.cuda.Stream(device=self.device))
            rt.prefetch_cfg = cfg
        return cfg

    @staticmethod
    def _prefetch(pf, jobs):
        """fork: the side stream picks up after the kernels launched so far and issues the prefetch jobs"""
        main = torch.cuda.current_stream()
        pf['side'].wait_stream(main)
        with torch.cuda.stream(pf['side']):
            for (t, frac, tile_bytes) in jobs:
                if frac <= 0:
                    continue
                total = t.numel() * t.element_size()
                if tile_bytes:   # HBM-tiled weight: the first share of every tile (= its first k chunks)
                    rb = max(16384, int(tile_bytes * min(frac, 1.0)) // 16384 * 16384)
                    ops.l2_prefetch(t, n_ranges=total // tile_bytes, stride_bytes=tile_bytes, range_bytes=min(rb, tile_bytes),
                                    gbytes_per_s=pf['rate'])
                else:
                    ops.l2_prefetch(t, range_bytes=int(total * min(frac, 1.0)) // 16 * 16, gbytes_per_s=pf['rate'])
        pf['dirty'] = True

    def _check_fused_attn(self):
        """the fused RoPE-inside-attention kernel (PIA_ATTN_FUSED) rotates in the half-split layout only"""
        if self.rotary_interleaved and os.environ.get('PIA_ATTN_FUSED', '0') != '0':
            raise ValueError(f'{type(self).__name__} rotates interleaved pairs (GLM RoPE), which the fused attention '
                             'kernel does not: unset PIA_ATTN_FUSED')

    # ------------------------------------------------------------------ the verify forward on static buffers
    def _mlp(self, rt, layer, y, plans=None, pf=None, b=None):
        """returns (x, parts): the MLP output as a bf16 tensor or as fp32 split-K slices for the next rmsnorm.
        b: the buffer set y belongs to (default: the decode buffers)"""
        m = layer.mlp
        if plans:
            b = b if b is not None else rt.decode_bufs
            rows = y.shape[0]   # 64 for the bf16 plans; every buffer row for the fp8 plans
            if 'gate_up_silu' in plans:
                plans['gate_up_silu'].run(rows, out=b.act)
            else:
                if 'gate_up' in plans:
                    plans['gate_up'].run(64, out=b.gu)
                else:
                    torch.mm(y, m.gate_up_weight.t(), out=b.gu)
                if pf:
                    self._prefetch(pf, [(m.down_proj.weight, pf['down'], 0)])
                ops.silu_mul(b.gu, b.act)
            if 'down' in plans:
                o = plans['down'].run(rows)
                return (o, None) if plans['down'].splits == 1 else (None, o)
            return torch.mm(b.act, m.down_proj.weight.t()), None
        gu = torch.mm(y, m.gate_up_weight.t())
        act = torch.empty((gu.shape[0], gu.shape[1] // 2), dtype=gu.dtype, device=gu.device)
        ops.silu_mul(gu, act)
        return torch.mm(act, m.down_proj.weight.t()), None

    def _verify_layers(self, rt, bufs=None, last_only=False):
        """embed -> decoder layers -> final norm -> lm_head over the rows described by `bufs` (default: the decode
        buffers = the drafts of the request slots in rt.ids / rt.mask / rt.n on top of rt.prefix_len cached tokens;
        bufs.slots says which slot owns which rows).  A prefill pass uses wider buffers holding several 64-row chain
        chunks (one table slot each): the GEMMs run once over all rows.  Writes bufs.logits (skipped when
        last_only)."""
        self.fuse()
        b = bufs if bufs is not None else rt.decode_bufs
        g = rt.g
        eps = self.config.rms_norm_eps
        ops.embed_gather(self.model.embed_tokens.weight, b.ids, b.n_total, b.h)
        if self._fp8:   # every projection of every buffer set on the fp8 plans, over all rows of the buffers
            plans, rows = self._fp8_plans(b), b.rows
        elif self._w4:  # likewise on the int4 plans
            plans, rows = self._w4_plans(b), b.rows
        else:
            plans, rows = (self._gemm_plans(rt) if b is rt.decode_bufs else False), 64
        pf = self._prefetch_cfg(rt) if plans and not (self._fp8 or self._w4) else False
        fused_attn = b is rt.decode_bufs and os.environ.get('PIA_ATTN_FUSED', '0') != '0' and \
            (b.slots.batch == 1 or b.slots.kv_slot_stride != 0)
        if fused_attn:
            self._check_fused_attn()
        rotary_dim = g['rotary_dim'] if self.rotary_interleaved else None
        alibi = getattr(rt, 'alibi_slopes', None)   # ALiBi models (Baichuan-13B): the slopes on the device
        logn = getattr(rt, 'logn_scale', None)      # Qwen's log-n query scaling: a bf16 table on the device
        x, parts, resid_in = b.h, None, None  # norm(x | parts, resid_in) -> (resid = x + resid_in, y = norm(resid))

        rnd = self.rmsnorm_rounding

        def norm(w):
            if parts is not None:
                ops.rmsnorm_partials(parts, resid_in, w, eps, b.resid, b.y, rounding=rnd)
            else:
                ops.rmsnorm(x, resid_in, w, eps, b.resid, b.y, rounding=rnd)

        def post_norm(w):   # a sublayer output normalised alone (no residual), into b.post_norm
            if parts is not None:
                ops.rmsnorm_partials(parts, None, w, eps, None, b.post_norm, rounding=rnd)
            else:
                ops.rmsnorm(x, None, w, eps, None, b.post_norm, rounding=rnd)
            return b.post_norm, None

        for li, layer in enumerate(self.model.layers):
            lp = plans['layers'][li] if plans else None
            norm(layer.input_layernorm.weight)
            a = layer.self_attn
            if lp and 'qkv' in lp:
                lp['qkv'].run(rows, out=b.qkv)
            elif a.qkv_bias is not None:   # bias added in fp32 before the one bf16 rounding, as F.linear does
                torch.addmm(a.qkv_bias, b.y, a.qkv_weight.t(), out=b.qkv)
            else:
                torch.mm(b.y, a.qkv_weight.t(), out=b.qkv)
            if pf and lp and 'gate_up' in lp:
                gw = lp['gate_up'].weight
                self._prefetch(pf, [(a.o_proj.weight, pf['o'], 0),
                                    (gw, pf['gate_up'], gw.shape[1] * gw.shape[2] * gw.shape[3] * 2 if gw.dim() == 4 else 0)])
            # every request slot / prefill chunk of the table in one launch each (pia_slots_t)
            if fused_attn:   # decode steps: RoPE + KV append happen inside the attention kernel
                rt.plan.forward_fused(li, b.qkv, b.mask, b.slots, rt.rope_cos, rt.rope_sin, b.attn)
            else:            # prefill chunks share one cache: append first, then attend
                ops.rope_kv_append(b.qkv, b.mask, b.slots, g['n_q_heads'], g['n_kv_heads'], g['head_dim'], rt.rope_cos,
                                   rt.rope_sin, b.q, rt.k_layer(li, b.kv_slot), rt.v_layer(li, b.kv_slot), rt.max_seq,
                                   rotary_dim=rotary_dim, q_scale=logn)
                rt.plan.forward(li, b.q, b.mask, b.slots, b.attn, alibi_slopes=alibi)
            if lp and 'o' in lp:
                o = lp['o'].run(rows)
                x, parts, resid_in = (o, None, b.resid) if lp['o'].splits == 1 else (None, o, b.resid)
            else:
                x, parts, resid_in = torch.mm(b.attn, a.o_proj.weight.t()), None, b.resid
            if self.sandwich_norms:
                x, parts = post_norm(layer.post_self_attn_layernorm.weight)
            norm(layer.post_attention_layernorm.weight)
            x, parts = self._mlp(rt, layer, b.y, lp, pf, b=b)
            if self.sandwich_norms:
                x, parts = post_norm(layer.post_mlp_layernorm.weight)
        if pf and pf.pop('dirty', False):  # join the side stream (required before a capture ends)
            torch.cuda.current_stream().wait_stream(pf['side'])
        if last_only:
            return
        norm(self.model.norm.weight)
        if b.logits is not None:
            if plans and 'lm_head' in plans:
                plans['lm_head'].run(64, out=b.logits)
            else:
                torch.mm(b.y, self.lm_head.weight.t(), out=b.logits)


class LlamaPreTrainedModel(LookaheadPreTrainedModel):
    pass
