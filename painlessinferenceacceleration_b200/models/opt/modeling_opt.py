# -*- coding: utf-8 -*-
"""OPT (OPT-125m ... OPT-66B, HF model_type `opt`) with the lookahead patch, H100-native (reference:
models/opt/modeling_opt.py).

The module tree and parameter names are HF's: `model.decoder.{embed_tokens, embed_positions, project_in?,
project_out?, layers.N.{self_attn.{q,k,v,out}_proj, self_attn_layer_norm, fc1, fc2, final_layer_norm},
final_layer_norm?}` and `lm_head` tied to `embed_tokens`.  One pre-LN decoder layer of the verify forward:
  pia_layernorm (+ the residual add) -> q|k|v addmm with the concatenated bias -> pia_kv_append_qscale (no rotation;
  q written as bf16(q * head_dim**-0.5), HF's `q_proj(h) * self.scaling`, K / V appended) -> k_tree_attn at softmax
  scale 1 -> out_proj addmm -> pia_layernorm (+ residual) -> fc1 addmm -> ReLU -> fc2 addmm.
The post-LN variant (`do_layer_norm_before=False`, OPT-350m) normalises after each residual add and has no final
LayerNorm; `project_in` / `project_out` (`word_embed_proj_dim != hidden_size`) stay bf16.

Positions are OPT's learned absolute embeddings (`OPTLearnedPositionalEmbedding`, offset 2) taken at tree positions,
pia_learned_pos_embed: every draft node's verify logits equal a causal forward over prefix + root-to-node path.  A
request whose max_length exceeds max_position_embeddings is refused before anything runs, so positions are never
clamped on a real request.

Head dims 64 and 128 run natively; any other (OPT-2.7B: 80) runs zero-padded to 128: the QKV GEMM stays at the
checkpoint's width and the append kernel writes the padded q / K / V itself; the attention output is gathered back to
[rows, H * d] before out_proj, so the streamed weight bytes stay the checkpoint's.  Because q arrives pre-scaled, the
attention runs with scale_mul = sqrt(D), which gives the kernel's log2-domain scale exactly log2(e) for D = 64 and 128.

fp8 (quantize_fp8, from_pretrained(quantization='fp8'), build_fp8): q|k|v, out_proj, fc1 and fc2 become per-row e4m3
weights on the fp8 GEMM with their biases in fp32 in its epilogue, fc1 with the ReLU epilogue.  Embeddings, positions,
lm_head, LayerNorms and project_in / project_out stay bf16.  In bf16 mode the biased projections run on cuBLAS, as
BLOOM's do."""
import math
import os

import torch
from torch import nn

from ...common import ops
from ...common.pretrained_model import LookaheadPreTrainedModel
from ..llama.modeling_llama import Fp8Linear, Fp8Rows, LlamaForCausalLM

PAD_D = 128
POS_OFFSET = 2   # OPTLearnedPositionalEmbedding.offset
LN_EPS = 1e-5    # HF builds OPT's LayerNorms with nn.LayerNorm's default eps


def check_opt_config(config):
    """raise, naming the field, for an OPT config this decoder cannot run"""
    mt = getattr(config, 'model_type', None)
    if mt != 'opt':
        raise ValueError(f'model_type {mt!r} is not an OPT config')
    act = getattr(config, 'activation_function', 'relu')
    if act != 'relu':
        raise NotImplementedError(f'opt config activation_function={act!r}: only relu is supported (Galactica\'s '
                                  'gelu is not)')
    if not getattr(config, 'enable_bias', True):
        raise NotImplementedError('opt config enable_bias=False: the projections are built with biases')
    if not getattr(config, 'layer_norm_elementwise_affine', True):
        raise NotImplementedError('opt config layer_norm_elementwise_affine=False: the LayerNorms are built with '
                                  'weight and bias')
    q = getattr(config, 'quantization_config', None)
    if q:
        raise NotImplementedError(f'opt config quantization_config={q!r}: quantised OPT checkpoints are not '
                                  'supported (fp8 is quantised on load: quantization=\'fp8\')')
    H, E = config.num_attention_heads, config.hidden_size
    if E % H:
        raise ValueError(f'opt config hidden_size={E} is not a multiple of num_attention_heads={H}')
    if E // H > PAD_D:
        raise ValueError(f'opt config head dim hidden_size / num_attention_heads = {E // H}: at most {PAD_D} is '
                         'supported')
    if (E // H) % 8:
        raise ValueError(f'opt config head dim {E // H}: a multiple of 8 is needed')


class OPTAttention(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        E = cfg.hidden_size
        kw = dict(bias=True, device=device, dtype=dtype)
        self.q_proj, self.k_proj, self.v_proj = nn.Linear(E, E, **kw), nn.Linear(E, E, **kw), nn.Linear(E, E, **kw)
        self.out_proj = nn.Linear(E, E, **kw)


class OPTDecoderLayer(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        E = cfg.hidden_size
        kw = dict(device=device, dtype=dtype)
        self.self_attn = OPTAttention(cfg, device, dtype)
        self.self_attn_layer_norm = nn.LayerNorm(E, eps=LN_EPS, **kw)
        self.fc1 = nn.Linear(E, cfg.ffn_dim, bias=True, **kw)
        self.fc2 = nn.Linear(cfg.ffn_dim, E, bias=True, **kw)
        self.final_layer_norm = nn.LayerNorm(E, eps=LN_EPS, **kw)


class OPTDecoder(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        E, P = cfg.hidden_size, cfg.word_embed_proj_dim
        kw = dict(device=device, dtype=dtype)
        self.embed_tokens = nn.Embedding(cfg.vocab_size, P, **kw)
        self.embed_positions = nn.Embedding(cfg.max_position_embeddings + POS_OFFSET, E, **kw)
        self.project_out = nn.Linear(E, P, bias=False, **kw) if P != E else None
        self.project_in = nn.Linear(P, E, bias=False, **kw) if P != E else None
        # HF: only a pre-LN model has one, unless _remove_final_layer_norm (old checkpoints) says otherwise
        pre = cfg.do_layer_norm_before and not getattr(cfg, '_remove_final_layer_norm', False)
        self.final_layer_norm = nn.LayerNorm(E, eps=LN_EPS, **kw) if pre else None
        self.layers = nn.ModuleList([OPTDecoderLayer(cfg, device, dtype) for _ in range(cfg.num_hidden_layers)])


class OPTModel(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        self.decoder = OPTDecoder(cfg, device, dtype)


class OPTForCausalLM(LookaheadPreTrainedModel):
    # the parameters of a decoder layer that fp8 mode quantises (relative to the layer)
    _fp8_params = ('self_attn.q_proj.weight', 'self_attn.k_proj.weight', 'self_attn.v_proj.weight',
                   'self_attn.out_proj.weight', 'fc1.weight', 'fc2.weight')

    def __init__(self, config, device=None, dtype=torch.bfloat16):
        check_opt_config(config)
        super().__init__(config)
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else 'meta'
        assert dtype == torch.bfloat16, 'the H100 path computes in bf16'
        self.model = OPTModel(config, device, dtype)
        self.lm_head = nn.Linear(config.word_embed_proj_dim, config.vocab_size, bias=False, device=device, dtype=dtype)
        if getattr(config, 'tie_word_embeddings', True):
            self.lm_head.weight = self.model.decoder.embed_tokens.weight
        self._fused = False
        self._fp8 = False
        for p_ in self.parameters():
            p_.requires_grad_(False)

    @property
    def head_dim(self):
        return self.config.hidden_size // self.config.num_attention_heads

    @property
    def attn_head_dim(self):
        """the head width the tree attention kernel runs at: 64 and 128 natively, the rest zero-padded to 128"""
        return self.head_dim if self.head_dim in (64, PAD_D) else PAD_D

    # ------------------------------------------------------------------ weights
    @torch.no_grad()
    def init_weights(self, seed=0, std=0.02):
        """random weights of the configured shape: LayerNorm weights 1, biases 0, the rest N(0, std^2)"""
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed)
        for name, p in self.named_parameters():
            if 'layer_norm' in name:
                p.fill_(1.0 if name.endswith('weight') else 0.0)
            elif name.endswith('bias'):
                p.zero_()
            else:
                p.normal_(0.0, std, generator=gen)
        return self

    def _convert_checkpoint_keys(self, sd):
        """checkpoint names with the `model.decoder.` (OPTForCausalLM), `decoder.` (OPTModel) or no (OPTDecoder)
        prefix -> this module tree's; a tied model ignores a stored lm_head"""
        tied = self.lm_head.weight is self.model.decoder.embed_tokens.weight
        out = {}
        for k, v in sd.items():
            if k == 'lm_head.weight':
                if tied:
                    continue
            elif k.startswith('decoder.'):
                k = 'model.' + k
            elif not k.startswith('model.decoder.'):
                k = 'model.decoder.' + k
            out[k] = v
        return out

    @torch.no_grad()
    def load_hf_state_dict(self, sd, _seen=None):
        """copy an HF OPT state dict (any of the three prefixes) into this model; raises if a tensor of the model is
        missing (unless _seen collects the names over several shards)"""
        own = dict(self.named_parameters())
        seen = set() if _seen is None else _seen
        for k, v in self._convert_checkpoint_keys(sd).items():
            if k in own:
                if tuple(v.shape) != tuple(own[k].shape):
                    raise ValueError(f'{k}: shape {tuple(v.shape)}, expected {tuple(own[k].shape)}')
                own[k].copy_(v.to(own[k].dtype))
                seen.add(k)
        if _seen is None:
            self._check_complete(seen, own)
        return self

    @staticmethod
    def _check_complete(seen, own):
        missing = [k for k in own if k not in seen]
        if missing:
            raise RuntimeError(f'checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}')

    @classmethod
    def _pretrained_config(cls, path):
        from transformers import AutoConfig
        cfg = AutoConfig.from_pretrained(path)
        if cfg.model_type != 'opt':
            raise ValueError(f'{path}: model_type {cfg.model_type!r} is not an OPT checkpoint')
        return cfg

    @classmethod
    def from_pretrained(cls, path, torch_dtype=torch.bfloat16, device=None, quantization=None, **kwargs):
        """HF checkpoint directory (config.json + *.safetensors / pytorch_model*.bin; the Hub's fp16 tensors are
        converted to bf16) -> model on the GPU.  quantization='fp8': the decoder projections become fp8 weights one
        layer at a time as they arrive; the bf16 decoder never exists on the GPU."""
        if quantization not in (None, 'fp8'):
            raise ValueError(f'quantization={quantization!r}: only None and \'fp8\' are supported')
        config = cls._pretrained_config(path)
        if quantization == 'fp8':
            return cls._from_pretrained_fp8(path, config, device)
        model = cls(config, device=device, dtype=torch_dtype)
        seen = set()
        for sd in LlamaForCausalLM._shards(path):
            model.load_hf_state_dict(sd, _seen=seen)
        model._check_complete(seen, dict(model.named_parameters()))
        return model

    # ------------------------------------------------------------------ fused q|k|v
    def fuse(self):
        """q / k / v weights and biases into single GEMM operands; the HF-named parameters become views of them"""
        if self._fused:
            return
        for layer in self.model.decoder.layers:
            self._fuse_layer(layer)
        self._fused = True

    @staticmethod
    def _fuse_layer(layer):
        a = layer.self_attn
        E = a.q_proj.weight.shape[0]
        w = torch.cat([a.q_proj.weight.data, a.k_proj.weight.data, a.v_proj.weight.data], dim=0).contiguous()
        b = torch.cat([a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data]).contiguous()
        a.q_proj.weight.data, a.k_proj.weight.data, a.v_proj.weight.data = w[:E], w[E:2 * E], w[2 * E:]
        a.q_proj.bias.data, a.k_proj.bias.data, a.v_proj.bias.data = b[:E], b[E:2 * E], b[2 * E:]
        a.qkv_weight, a.qkv_bias = w, b

    # ------------------------------------------------------------------ fp8 (e4m3) weight-only mode
    @torch.no_grad()
    def quantize_fp8(self):
        """Convert q|k|v, out_proj, fc1 and fc2 of every layer to per-row e4m3 weights with fp32 scales
        (ops.quantize_fp8), in place and one layer at a time.  Biases, embeddings, positions, lm_head, LayerNorms and
        project_in / project_out stay bf16.  Both dimensions of every weight must be multiples of 128; otherwise
        ValueError before anything is converted."""
        if self._fp8:
            return self
        E, F = self.config.hidden_size, self.config.ffn_dim
        for shape in ((3 * E, E), (E, E), (F, E), (E, F)):
            if shape[0] % 128 or shape[1] % 128:
                raise ValueError(f'fp8 weights need both dimensions divisible by 128, got {shape} (hidden_size={E}, '
                                 f'ffn_dim={F})')
        self.fuse()
        self._rt = None   # drops the buffers of the bf16 path
        for layer in self.model.decoder.layers:
            self._quantize_layer(layer)
        self._fp8 = True
        return self

    @staticmethod
    def _quantize_layer(layer):
        a = layer.self_attn
        E = a.q_proj.weight.shape[0]
        qkv = Fp8Linear(a.qkv_weight)
        a.qkv_fp8 = qkv
        a.q_proj = Fp8Rows(qkv, 0, E, a.q_proj.bias)
        a.k_proj = Fp8Rows(qkv, E, 2 * E, a.k_proj.bias)
        a.v_proj = Fp8Rows(qkv, 2 * E, 3 * E, a.v_proj.bias)
        a.qkv_weight = None
        for parent, name in ((a, 'out_proj'), (layer, 'fc1'), (layer, 'fc2')):
            lin = getattr(parent, name)
            f = Fp8Linear(lin.weight.data)
            f.bias = lin.bias   # the bf16 bias keeps its HF name
            setattr(parent, name, f)

    @classmethod
    def _fp8_skeleton(cls, config, device):
        """the model on the meta device with everything but the quantised projections allocated (uninitialised) on
        the GPU; returns (model, {name: allocated parameter}, layer_of(name), materialise(name))"""
        dev = device if device is not None else torch.device('cuda', torch.cuda.current_device())
        model = cls(config, device='meta')

        def layer_of(name):
            parts = name.split('.')
            if name.startswith('model.decoder.layers.') and '.'.join(parts[4:]) in cls._fp8_params:
                return int(parts[3])
            return None

        def materialise(name):
            mod_name, _, pname = name.rpartition('.')
            mod = model.get_submodule(mod_name)
            old = getattr(mod, pname)
            setattr(mod, pname, nn.Parameter(torch.empty(old.shape, dtype=old.dtype, device=dev), requires_grad=False))
            return getattr(mod, pname)

        own = {name: materialise(name) for name, _ in list(model.named_parameters()) if layer_of(name) is None}
        if model.lm_head.weight is not model.model.decoder.embed_tokens.weight and \
                getattr(config, 'tie_word_embeddings', True):
            model.lm_head.weight = model.model.decoder.embed_tokens.weight   # materialise broke the tie
            own.pop('lm_head.weight', None)
        return model, own, layer_of, materialise

    @classmethod
    @torch.no_grad()
    def build_fp8(cls, config, fill_rest, fill_weight, device=None):
        """An fp8 model without a checkpoint and without its bf16 decoder ever existing (an OPT-66B shape fits one
        80 GB card only this way): fill_rest(model) initialises the parameters that stay bf16; then, one layer at a
        time, fill_weight(name, tensor) fills each projection weight in a bf16 buffer (HF names), which is fused,
        quantised and freed."""
        model, _, _, materialise = cls._fp8_skeleton(config, device)
        fill_rest(model)
        for li, layer in enumerate(model.model.decoder.layers):
            for p in cls._fp8_params:
                name = f'model.decoder.layers.{li}.{p}'
                fill_weight(name, materialise(name))
            cls._fuse_layer(layer)
            cls._quantize_layer(layer)
        model._fused = model._fp8 = True
        return model

    @classmethod
    @torch.no_grad()
    def _from_pretrained_fp8(cls, path, config, device):
        """everything but the quantised projections is allocated on the GPU up front; a layer's projections wait on
        the host until the layer is complete, then that one layer is allocated in bf16, filled, fused and quantised"""
        model, own, layer_of, materialise = cls._fp8_skeleton(config, device)
        n_layers = len(model.model.decoder.layers)
        pending = {li: {} for li in range(n_layers)}
        seen = set()
        for sd in LlamaForCausalLM._shards(path):
            for k, v in model._convert_checkpoint_keys(sd).items():
                li = layer_of(k)
                if li is not None and li in pending:
                    pending[li][k] = v
                    if len(pending[li]) == len(cls._fp8_params):
                        for name, t in pending.pop(li).items():
                            materialise(name).copy_(t.to(torch.bfloat16))
                        layer = model.model.decoder.layers[li]
                        cls._fuse_layer(layer)
                        cls._quantize_layer(layer)
                elif k in own:
                    own[k].copy_(v.to(torch.bfloat16))
                    seen.add(k)
        missing = [k for k in own if k not in seen]
        missing += [f'model.decoder.layers.{li}.{p}' for li, got in pending.items() for p in cls._fp8_params
                    if f'model.decoder.layers.{li}.{p}' not in got]
        if missing:
            raise RuntimeError(f'checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}')
        model._fused = model._fp8 = True
        return model

    def _fp8_plans(self, b, s):
        """fp8 GEMM plans of one activation buffer set, made once per buffer set outside any capture"""
        plans = getattr(b, 'opt_fp8_plans', None)
        if plans is not None:
            return plans
        n_sm = torch.cuda.get_device_properties(b.y.device).multi_processor_count
        pre = self.config.do_layer_norm_before
        attn = s['attn'] if s['attn'] is not None else b.attn   # out_proj's input: H * d wide
        plans = []
        for layer in self.model.decoder.layers:
            a = layer.self_attn
            qkv = a.qkv_fp8
            bias = torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias]).float()
            lp = {'qkv': ops.Gemm.fp8(qkv.qweight, qkv.scale, b.y if pre else b.h, bias=bias,
                                      split_k=LlamaForCausalLM._fp8_split(qkv, n_sm), out=s['qkv'])}
            for name, lin, x, out in (('o', a.out_proj, attn, s['o']), ('fc1', layer.fc1, b.y, s['act']),
                                      ('fc2', layer.fc2, s['act'], s['o'])):
                lp[name] = ops.Gemm.fp8(lin.qweight, lin.scale, x, bias=lin.bias.float(),
                                        split_k=LlamaForCausalLM._fp8_split(lin, n_sm), out=out)
            lp['fc1'].set_relu()
            plans.append(lp)
        b.opt_fp8_plans = plans
        return plans

    # ------------------------------------------------------------------ geometry / tables / runtime
    def geometry(self):
        c = self.config
        return dict(n_layers=c.num_hidden_layers, hidden=c.hidden_size, n_q_heads=c.num_attention_heads,
                    n_kv_heads=c.num_attention_heads, head_dim=self.attn_head_dim, inter=c.ffn_dim,
                    vocab=c.vocab_size)

    def rope_tables(self, max_pos):
        """OPT has no rotation: the append kernel reads no tables"""
        return None, None

    def check_max_length(self, max_length):
        """positions are learned up to max_position_embeddings: a longer request is refused, never clamped"""
        limit = self.config.max_position_embeddings
        if max_length is not None and int(max_length) > limit:
            raise ValueError(f'max_length={int(max_length)} exceeds the model\'s max_position_embeddings={limit}: OPT '
                             'has no learned position beyond it')

    def _start_request(self, rt, input_len, max_length=None):
        self.check_max_length(input_len)
        self.check_max_length(max_length)

    def _check_knobs(self):
        if os.environ.get('PIA_ATTN_FUSED', '0') != '0':
            raise ValueError(f'{type(self).__name__} has no RoPE for the fused attention kernel to apply and a '
                             'pre-scaled query: unset PIA_ATTN_FUSED')
        for knob in ('PIA_GEMM', 'PIA_GEMM_SET'):
            if knob in os.environ:
                raise ValueError(f'{knob} is set, but OPT runs its biased projections on cuBLAS (bf16) or on the fp8 '
                                 'GEMM with a bias epilogue and has no weight-streaming plan for it to select: unset it')

    def _runtime(self, max_seq, max_nodes, n_slots=1, keep_cache=False):
        self._check_knobs()   # before anything is captured
        rt = super()._runtime(max_seq, max_nodes, n_slots, keep_cache)
        for b in (rt.decode_bufs, rt.prefill_bufs):   # scratch of the verify forward, made outside any capture
            if getattr(b, 'opt', None) is None:
                b.opt = self._scratch(b.rows, rt.device)
            if self._fp8:
                self._fp8_plans(b, b.opt)
        return rt

    def _scratch(self, rows, dev):
        c = self.config
        E, H, P = c.hidden_size, c.num_attention_heads, c.word_embed_proj_dim
        bf = dict(dtype=torch.bfloat16, device=dev)
        s = dict(qkv=torch.zeros((rows, 3 * E), **bf), o=torch.zeros((rows, E), **bf),
                 act=torch.zeros((rows, c.ffn_dim), **bf))
        s['attn'] = torch.zeros((rows, E), **bf) if self.attn_head_dim != self.head_dim else None
        if P != E:   # project_in's input and project_out's output
            s['emb'] = torch.zeros((rows, P), **bf)
            s['out'] = torch.zeros((rows, P), **bf)
        return s

    # ------------------------------------------------------------------ the verify forward on static buffers
    def _verify_layers(self, rt, bufs=None, last_only=False):
        self.fuse()
        b = bufs if bufs is not None else rt.decode_bufs
        c = self.config
        H, d, D, eps = c.num_attention_heads, self.head_dim, self.attn_head_dim, LN_EPS
        rows = b.rows
        s = b.opt
        dec = self.model.decoder
        pre = c.do_layer_norm_before
        q_mul = d ** -0.5                 # OPTAttention.scaling, a python float taken as fp32 by the kernel
        scale_mul = math.sqrt(D)          # the query is pre-scaled: the softmax scale is exactly 1
        attn = s['attn'] if s['attn'] is not None else b.attn
        plans = b.opt_fp8_plans if self._fp8 else None
        # embeddings: tokens (project_in) + learned positions at tree positions
        if dec.project_in is None:
            ops.learned_pos_embed(dec.embed_tokens.weight, b.ids, dec.embed_positions.weight, POS_OFFSET, b.mask,
                                  b.slots, b.h)
        else:
            ops.embed_gather(dec.embed_tokens.weight, b.ids, b.n_total, s['emb'])
            torch.mm(s['emb'], dec.project_in.weight.t(), out=b.h)
            ops.learned_pos_embed(None, None, dec.embed_positions.weight, POS_OFFSET, b.mask, b.slots, b.h)
        x, resid_in = b.h, None
        n_layers = len(dec.layers)
        for li, layer in enumerate(dec.layers):
            a = layer.self_attn
            lp = plans[li] if plans is not None else None
            if pre:   # y = LN(x + resid), resid updated in place
                ln = layer.self_attn_layer_norm
                ops.layernorm(x, resid_in, ln.weight, ln.bias, eps, b.resid, b.y)
            qkv_in = b.y if pre else b.h
            if lp is not None:
                lp['qkv'].run(rows)
            else:
                torch.addmm(a.qkv_bias, qkv_in, a.qkv_weight.t(), out=s['qkv'])
            ops.kv_append(s['qkv'], b.mask, b.slots, H, H, d, D, q_mul, b.q, rt.k_layer(li, b.kv_slot),
                          rt.v_layer(li, b.kv_slot), rt.max_seq)
            rt.plan.forward(li, b.q, b.mask, b.slots, b.attn, scale_mul=scale_mul)
            if s['attn'] is not None:
                s['attn'].view(rows, H, d).copy_(b.attn.view(rows, H, D)[:, :, :d])
            if lp is not None:
                lp['o'].run(rows)
            else:
                torch.addmm(a.out_proj.bias, attn, a.out_proj.weight.t(), out=s['o'])
            if pre:
                ln = layer.final_layer_norm
                ops.layernorm(s['o'], b.resid, ln.weight, ln.bias, eps, b.resid, b.y)
            else:   # post-LN: h = LN(h + attn) -> b.y
                ln = layer.self_attn_layer_norm
                ops.layernorm(s['o'], b.h, ln.weight, ln.bias, eps, None, b.y)
            if lp is not None:
                lp['fc1'].run(rows)
                lp['fc2'].run(rows)
            else:
                torch.addmm(layer.fc1.bias, b.y, layer.fc1.weight.t(), out=s['act'])
                torch.relu_(s['act'])
                torch.addmm(layer.fc2.bias, s['act'], layer.fc2.weight.t(), out=s['o'])
            if pre:
                x, resid_in = s['o'], b.resid
            else:   # h = LN(y + mlp): the next layer's input in b.h, the last layer's output in b.y (in place)
                ln = layer.final_layer_norm
                ops.layernorm(s['o'], b.y, ln.weight, ln.bias, eps, None, b.y if li == n_layers - 1 else b.h)
        if last_only:
            return
        # the final hidden state (before project_out) in b.y, where the prefill pass leaves its last row
        if pre and dec.final_layer_norm is not None:
            ops.layernorm(x, resid_in, dec.final_layer_norm.weight, dec.final_layer_norm.bias, eps, b.resid, b.y)
        elif pre:
            torch.add(x, resid_in, out=b.y)
        if b.logits is not None:
            torch.mm(self._project_out(b.y, s.get('out')), self.lm_head.weight.t(), out=b.logits)

    def _project_out(self, h, out=None):
        po = self.model.decoder.project_out
        return h if po is None else torch.mm(h, po.weight.t(), out=out)

    def _prefill_logits(self, rt, prompt_len, slot=0, row=0):
        """prefill of slot `slot` + the last prompt row's logits into rt.logits[row], through project_out if any"""
        y = self._prefill_kv(rt, prompt_len, slot)
        torch.mm(self._project_out(y), self.lm_head.weight.t(), out=rt.logits[row:row + 1])
