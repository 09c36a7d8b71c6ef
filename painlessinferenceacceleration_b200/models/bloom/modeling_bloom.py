# -*- coding: utf-8 -*-
"""BLOOM / BLOOMZ with the lookahead patch, H100-native (reference: models/bloom/modeling_bloom.py).

The module tree and parameter names are HF's (`transformer.word_embeddings`, `transformer.word_embeddings_layernorm`,
`transformer.h.N.{input_layernorm, self_attention.query_key_value, self_attention.dense, post_attention_layernorm,
mlp.dense_h_to_4h, mlp.dense_4h_to_h}`, `transformer.ln_f`, `lm_head` tied to the word embeddings unless the config
unties it).  One decoder layer of the verify forward:
  pia_layernorm (+ the residual add, dropout_add :504 / :539) -> QKV addmm (bias added before the one bf16 rounding, as
  F.linear does) -> k_rope_kv_append with identity tables (x * 1 + rot(x) * 0, exact: BLOOM has no RoPE) ->
  pia_tree_attn_alibi_fwd -> dense addmm -> pia_layernorm (+ residual) -> dense_h_to_4h addmm -> pia_bloom_gelu in
  place -> dense_4h_to_h addmm.
The ALiBi bias is taken at tree positions, which is what the reference's BLOOM patch does (:170, `(mask.cumsum(-1) - 1)
* mask`), so every draft node's verify logits equal a causal forward over prefix + root-to-node path.  The four biased
projections stay on cuBLAS: k_gemm_ws has no bias epilogue.

The ALiBi tree attention kernel is built for head dim 128.  Narrower heads (bloom-560m: 64, bloom-3b: 80, bloom-1b1:
96) run on it zero-padded to 128: the QKV GEMM runs at the checkpoint's width and its output is copied into the padded
[rows, 3H, 128] layout (the padding columns are zero from allocation on and never written), the attention output is
gathered back to [rows, H * d] before `dense`, and the softmax scale 1/sqrt(128) is corrected by scale_mul =
sqrt(128 / d).  The kernel adds the bias after the scale, so padding leaves it unchanged.  Padding the activations
rather than the weights keeps the streamed weight bytes exactly the checkpoint's.

The checkpoint's query_key_value rows are per head [q_h; k_h; v_h] (HF `_reshape`: view(H, 3, d)); they are re-laid
as [q heads | k heads | v heads] when the weights are set (load_hf_state_dict / from_pretrained), so the parameter of
this class holds the regrouped rows."""
import math
import os

import torch
from torch import nn

from ...common import ops
from ...common.pretrained_model import LookaheadPreTrainedModel
from ..llama.modeling_llama import LlamaForCausalLM

PAD_D = 128


def check_bloom_config(config):
    """raise, naming the field, for a BLOOM config this decoder cannot run"""
    mt = getattr(config, 'model_type', None)
    if mt != 'bloom':
        raise ValueError(f'model_type {mt!r} is not a BLOOM config')
    if getattr(config, 'apply_residual_connection_post_layernorm', False):
        raise NotImplementedError('bloom config apply_residual_connection_post_layernorm=True: the residual is taken '
                                  'before the LayerNorm here, as in every published BLOOM checkpoint')
    if getattr(config, 'pretraining_tp', 1) > 1 and getattr(config, 'slow_but_exact', False):
        raise NotImplementedError(f'bloom config slow_but_exact=True with pretraining_tp={config.pretraining_tp}: the '
                                  'sliced dense projections are not supported (set slow_but_exact=False)')
    q = getattr(config, 'quantization_config', None)
    if q:
        raise NotImplementedError(f'bloom config quantization_config={q!r}: quantised BLOOM checkpoints are not '
                                  'supported')
    H, E = config.n_head, config.hidden_size
    if E % H:
        raise ValueError(f'bloom config hidden_size={E} is not a multiple of n_head={H}')
    if E // H > PAD_D:
        raise ValueError(f'bloom config head dim hidden_size / n_head = {E // H}: at most {PAD_D} is supported')


def regroup_qkv(t, n_head):
    """query_key_value weight [3 H d, E] (or bias [3 H d]) from per-head [q_h; k_h; v_h] to [q heads | k heads |
    v heads]"""
    d = t.shape[0] // (3 * n_head)
    return t.reshape(n_head, 3, d, *t.shape[1:]).transpose(0, 1).reshape(t.shape).contiguous()


class BloomAttention(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        E = cfg.hidden_size
        self.query_key_value = nn.Linear(E, 3 * E, bias=True, device=device, dtype=dtype)
        self.dense = nn.Linear(E, E, bias=True, device=device, dtype=dtype)


class BloomMLP(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        E = cfg.hidden_size
        self.dense_h_to_4h = nn.Linear(E, 4 * E, bias=True, device=device, dtype=dtype)
        self.dense_4h_to_h = nn.Linear(4 * E, E, bias=True, device=device, dtype=dtype)


class BloomBlock(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        kw = dict(eps=cfg.layer_norm_epsilon, device=device, dtype=dtype)
        self.input_layernorm = nn.LayerNorm(cfg.hidden_size, **kw)
        self.self_attention = BloomAttention(cfg, device, dtype)
        self.post_attention_layernorm = nn.LayerNorm(cfg.hidden_size, **kw)
        self.mlp = BloomMLP(cfg, device, dtype)


class BloomModel(nn.Module):
    def __init__(self, cfg, device, dtype):
        super().__init__()
        kw = dict(eps=cfg.layer_norm_epsilon, device=device, dtype=dtype)
        self.word_embeddings = nn.Embedding(cfg.vocab_size, cfg.hidden_size, device=device, dtype=dtype)
        self.word_embeddings_layernorm = nn.LayerNorm(cfg.hidden_size, **kw)
        self.h = nn.ModuleList([BloomBlock(cfg, device, dtype) for _ in range(cfg.n_layer)])
        self.ln_f = nn.LayerNorm(cfg.hidden_size, **kw)


class BloomForCausalLM(LookaheadPreTrainedModel):
    def __init__(self, config, device=None, dtype=torch.bfloat16):
        check_bloom_config(config)
        super().__init__(config)
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else 'meta'
        assert dtype == torch.bfloat16, 'the H100 path computes in bf16'
        self.transformer = BloomModel(config, device, dtype)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False, device=device, dtype=dtype)
        if getattr(config, 'tie_word_embeddings', True):
            self.lm_head.weight = self.transformer.word_embeddings.weight
        self.alibi_slopes = None
        for p_ in self.parameters():
            p_.requires_grad_(False)

    @property
    def head_dim(self):
        return self.config.hidden_size // self.config.n_head

    # ------------------------------------------------------------------ weights
    @torch.no_grad()
    def init_weights(self, seed=0, std=0.02):
        """random weights of the configured shape: LayerNorm weights 1, biases 0, the rest N(0, std^2)"""
        gen = torch.Generator(device=self.device)
        gen.manual_seed(seed)
        for name, p in self.named_parameters():
            if 'layernorm' in name or '.ln_f.' in name:
                p.fill_(1.0 if name.endswith('weight') else 0.0)
            elif name.endswith('bias'):
                p.zero_()
            else:
                p.normal_(0.0, std, generator=gen)
        return self

    def _convert_checkpoint_keys(self, sd):
        """checkpoint names with or without the `transformer.` prefix (BloomModel saves none, BloomForCausalLM does);
        query_key_value rows regrouped to [q | k | v]; a tied model ignores a stored lm_head"""
        tied = self.lm_head.weight is self.transformer.word_embeddings.weight
        out = {}
        for k, v in sd.items():
            if k == 'lm_head.weight':
                if tied:
                    continue
            elif not k.startswith('transformer.'):
                k = 'transformer.' + k
            if k.endswith('self_attention.query_key_value.weight') or k.endswith('self_attention.query_key_value.bias'):
                v = regroup_qkv(v, self.config.n_head)
            out[k] = v
        return out

    @torch.no_grad()
    def load_hf_state_dict(self, sd, _seen=None):
        """copy an HF BLOOM state dict (checkpoint layout, with or without the `transformer.` prefix) into this model;
        raises if a tensor of the model is missing (unless _seen collects the names over several shards)"""
        own = dict(self.named_parameters())
        seen = set() if _seen is None else _seen
        for k, v in self._convert_checkpoint_keys(sd).items():
            if k in own:
                if tuple(v.shape) != tuple(own[k].shape):
                    raise ValueError(f'{k}: shape {tuple(v.shape)}, expected {tuple(own[k].shape)}')
                own[k].copy_(v.to(own[k].dtype))
                seen.add(k)
        if _seen is None:
            self._check_complete(seen)
        return self

    def _check_complete(self, seen):
        missing = [k for k in dict(self.named_parameters()) if k not in seen]
        if missing:
            raise RuntimeError(f'checkpoint is missing {len(missing)} tensors, e.g. {missing[:4]}')

    @classmethod
    def _pretrained_config(cls, path):
        from transformers import AutoConfig
        cfg = AutoConfig.from_pretrained(path)
        if cfg.model_type != 'bloom':
            raise ValueError(f'{path}: model_type {cfg.model_type!r} is not a BLOOM checkpoint')
        return cfg

    @classmethod
    def from_pretrained(cls, path, torch_dtype=torch.bfloat16, device=None, quantization=None, **kwargs):
        """HF checkpoint directory (config.json + *.safetensors / pytorch_model*.bin) -> model on the GPU"""
        if quantization is not None:
            raise NotImplementedError(f'quantization={quantization!r}: {cls.__name__} has no fp8 weight mode')
        model = cls(cls._pretrained_config(path), device=device, dtype=torch_dtype)
        seen = set()
        for sd in LlamaForCausalLM._shards(path):
            model.load_hf_state_dict(sd, _seen=seen)
        model._check_complete(seen)
        return model

    # ------------------------------------------------------------------ geometry / tables / runtime
    def geometry(self):
        c = self.config
        return dict(n_layers=c.n_layer, hidden=c.hidden_size, n_q_heads=c.n_head, n_kv_heads=c.n_head,
                    head_dim=PAD_D, inter=4 * c.hidden_size, vocab=c.vocab_size)

    def rope_tables(self, max_pos):
        """identity rotation: k_rope_kv_append then only copies q and appends K / V"""
        dev = self.device
        return (torch.ones((max_pos, PAD_D // 2), dtype=torch.bfloat16, device=dev),
                torch.zeros((max_pos, PAD_D // 2), dtype=torch.bfloat16, device=dev))

    def fuse(self):
        """nothing to fuse: the QKV rows are regrouped when the weights are set"""

    def _check_knobs(self):
        if os.environ.get('PIA_ATTN_FUSED', '0') != '0':
            raise ValueError(f'{type(self).__name__} needs ALiBi, which the fused attention kernel does not have: '
                             'unset PIA_ATTN_FUSED')
        for knob in ('PIA_GEMM', 'PIA_GEMM_SET'):
            if knob in os.environ:
                raise ValueError(f'{knob} is set, but BLOOM runs its biased projections on cuBLAS and has no '
                                 'weight-streaming GEMM plan for it to select: unset it')

    def _runtime(self, max_seq, max_nodes, n_slots=1, keep_cache=False):
        self._check_knobs()   # before anything is captured
        rt = super()._runtime(max_seq, max_nodes, n_slots, keep_cache)
        if self.alibi_slopes is None or self.alibi_slopes.device != rt.device:
            self.alibi_slopes = ops.alibi_slopes(self.config.n_head).to(rt.device)
        rt.alibi_slopes = self.alibi_slopes
        for b in (rt.decode_bufs, rt.prefill_bufs):   # scratch of the verify forward, made outside any capture
            if getattr(b, 'bloom', None) is None:
                b.bloom = self._scratch(b.rows, rt.device)
        return rt

    def _scratch(self, rows, dev):
        c = self.config
        E, d = c.hidden_size, self.head_dim
        bf = dict(dtype=torch.bfloat16, device=dev)
        s = dict(o=torch.zeros((rows, E), **bf), act=torch.zeros((rows, 4 * E), **bf))
        if d != PAD_D:   # checkpoint-width QKV output and attention input of dense
            s['qkv'] = torch.zeros((rows, 3 * E), **bf)
            s['attn'] = torch.zeros((rows, E), **bf)
        return s

    # ------------------------------------------------------------------ the verify forward on static buffers
    def _verify_layers(self, rt, bufs=None, last_only=False):
        b = bufs if bufs is not None else rt.decode_bufs
        c = self.config
        H, d, eps = c.n_head, self.head_dim, c.layer_norm_epsilon
        rows = b.rows
        s = b.bloom
        tr = self.transformer
        padded = d != PAD_D
        scale_mul = math.sqrt(PAD_D / d)
        ops.embed_gather(tr.word_embeddings.weight, b.ids, b.n_total, b.h)
        wl = tr.word_embeddings_layernorm
        ops.layernorm(b.h, None, wl.weight, wl.bias, eps, None, b.h)
        x, resid_in = b.h, None
        for li, blk in enumerate(tr.h):
            a = blk.self_attention
            ops.layernorm(x, resid_in, blk.input_layernorm.weight, blk.input_layernorm.bias, eps, b.resid, b.y)
            if padded:
                torch.addmm(a.query_key_value.bias, b.y, a.query_key_value.weight.t(), out=s['qkv'])
                b.qkv.view(rows, 3 * H, PAD_D)[:, :, :d].copy_(s['qkv'].view(rows, 3 * H, d))
            else:
                torch.addmm(a.query_key_value.bias, b.y, a.query_key_value.weight.t(), out=b.qkv)
            ops.rope_kv_append(b.qkv, b.mask, b.slots, H, H, PAD_D, rt.rope_cos, rt.rope_sin, b.q,
                               rt.k_layer(li, b.kv_slot), rt.v_layer(li, b.kv_slot), rt.max_seq)
            rt.plan.forward(li, b.q, b.mask, b.slots, b.attn, scale_mul=scale_mul, alibi_slopes=rt.alibi_slopes)
            if padded:
                s['attn'].view(rows, H, d).copy_(b.attn.view(rows, H, PAD_D)[:, :, :d])
                attn = s['attn']
            else:
                attn = b.attn
            torch.addmm(a.dense.bias, attn, a.dense.weight.t(), out=s['o'])
            ln = blk.post_attention_layernorm
            ops.layernorm(s['o'], b.resid, ln.weight, ln.bias, eps, b.resid, b.y)
            m = blk.mlp
            torch.addmm(m.dense_h_to_4h.bias, b.y, m.dense_h_to_4h.weight.t(), out=s['act'])
            ops.bloom_gelu(s['act'])
            torch.addmm(m.dense_4h_to_h.bias, s['act'], m.dense_4h_to_h.weight.t(), out=s['o'])
            x, resid_in = s['o'], b.resid
        if last_only:
            return
        ops.layernorm(x, resid_in, tr.ln_f.weight, tr.ln_f.bias, eps, b.resid, b.y)
        if b.logits is not None:
            torch.mm(b.y, self.lm_head.weight.t(), out=b.logits)
