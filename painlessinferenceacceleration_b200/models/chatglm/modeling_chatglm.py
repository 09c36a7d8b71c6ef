# -*- coding: utf-8 -*-
"""ChatGLM2-6B / ChatGLM3-6B (and their -32k variants) in THUDM's checkpoint format (config.json `model_type: chatglm`,
tensors under `transformer.*`), with the lookahead patch (reference: models/chatglm/modeling_chatglm.py,
models/chatglm3/modeling_chatglm.py; positions :815 = rowsum(mask) - 1).  The network is the GLM decoder of
models/glm4 (RMSNorm, q/k/v biases, multi-query groups, interleaved RoPE on the first half of each head, SwiGLU over a
fused [gate; up] weight), so this class only translates the config and the tensor names.

config.json is read as JSON: AutoConfig would need trust_remote_code, which runs code shipped with the checkpoint.
Configs of a different network raise, naming the field: ChatGLM-6B v1 (2D positions), LayerNorm instead of RMSNorm,
biases on the dense projections, the residual taken after the norm, no final norm, the original (half-split) RoPE,
THUDM's int4 / int8 quantised weights and prefix tuning (pre_seq_len).

apply_query_key_layer_scaling multiplies the scores by `coeff` = layer number and divides 1/sqrt(d) by it too, and the
fp32 softmax (attention_softmax_in_fp32) divides it back out: the math is plain 1/sqrt(d) scaling, which is what the
tree attention kernel computes."""
import json
import os
import types

from ...common import ops
from ..glm4.modeling_glm4 import GlmForCausalLM

_LAYER = 'transformer.encoder.layers.'


def _glm_config(cfg):
    """THUDM chatglm config dict -> a transformers GlmConfig of the same network"""
    from transformers import GlmConfig
    c = types.SimpleNamespace(**cfg)

    def need(field, want):
        if field in cfg and cfg[field] != want:
            raise NotImplementedError(f'chatglm config {field}={cfg[field]!r}: only {field}={want!r} is the GLM decoder '
                                      'this model runs')

    if 'position_encoding_2d' in cfg or 'multi_query_attention' not in cfg:
        raise NotImplementedError('chatglm config with position_encoding_2d / without multi_query_attention: ChatGLM-6B '
                                  'v1 (2D positions) is not supported')
    need('rmsnorm', True)
    need('add_bias_linear', False)
    need('apply_residual_connection_post_layernorm', False)
    need('post_layer_norm', True)
    need('original_rope', True)
    if cfg.get('quantization_bit', 0) not in (0, None):
        raise NotImplementedError(f'chatglm config quantization_bit={cfg["quantization_bit"]}: THUDM int4 / int8 '
                                  'checkpoints are not supported (load the bf16 checkpoint, optionally with '
                                  "quantization='fp8')")
    if cfg.get('pre_seq_len') is not None:
        raise NotImplementedError(f'chatglm config pre_seq_len={cfg["pre_seq_len"]}: prefix tuning is not supported')
    heads, hidden = c.num_attention_heads, c.hidden_size
    kv_ch = int(cfg.get('kv_channels', 128))            # ChatGLMConfig's defaults
    if kv_ch * heads != hidden:
        raise ValueError(f'chatglm config kv_channels={kv_ch}: only kv_channels = hidden_size / num_attention_heads '
                         f'({hidden // heads}) is supported')
    mqa = bool(cfg['multi_query_attention'])
    kv_heads = int(cfg.get('multi_query_group_num', 1)) if mqa else heads
    theta = 10000.0 * float(cfg.get('rope_ratio', 1) or 1)
    return GlmConfig(vocab_size=c.padded_vocab_size, hidden_size=hidden, intermediate_size=c.ffn_hidden_size,
                     num_hidden_layers=c.num_layers, num_attention_heads=heads, num_key_value_heads=kv_heads,
                     head_dim=kv_ch, max_position_embeddings=int(cfg.get('seq_length', 2048)),
                     rms_norm_eps=float(cfg.get('layernorm_epsilon', 1e-5)),
                     attention_bias=bool(cfg.get('add_qkv_bias', False)),
                     rope_parameters={'rope_type': 'default', 'rope_theta': theta, 'partial_rotary_factor': 0.5},
                     tie_word_embeddings=False, pad_token_id=cfg.get('pad_token_id', 0),
                     eos_token_id=cfg.get('eos_token_id', 2), bos_token_id=cfg.get('bos_token_id', None),
                     # without multi-query attention query_key_value rows are per head [q_h; k_h; v_h] (reference
                     # :393-399); with it, [q; k; v]
                     chatglm_qkv_per_head=not mqa)


class ChatGLMForConditionalGeneration(GlmForCausalLM):
    """THUDM-format ChatGLM2/3 checkpoints on the GLM decoder.  Built from a GlmConfig (use from_pretrained(path) for a
    checkpoint directory, or chatglm_config(dict) for a config.json already read); module tree and parameter names
    are transformers' GlmForCausalLM's."""
    # THUDM's RMSNorm rounds once, (weight * hidden_states).to(input_dtype) (chatglm/modeling_chatglm.py:187,
    # chatglm3/modeling_chatglm.py:196), unlike transformers' GlmRMSNorm that GlmForCausalLM follows
    rmsnorm_rounding = ops.ROUND_ONCE

    @staticmethod
    def chatglm_config(cfg):
        return _glm_config(cfg)

    @classmethod
    def _pretrained_config(cls, path):
        with open(os.path.join(path, 'config.json')) as f:
            cfg = json.load(f)
        if cfg.get('model_type') != 'chatglm':
            raise ValueError(f'{path}: model_type {cfg.get("model_type")!r} is not a THUDM chatglm checkpoint')
        return _glm_config(cfg)

    def _convert_checkpoint_keys(self, sd):
        """THUDM tensor names -> transformers' GLM names.  With multi-query attention (every ChatGLM2/3 checkpoint)
        query_key_value rows are [q; k; v], the fused layout of this module tree; without it they are per head
        [q_0; k_0; v_0; q_1; ...] (reference :393-399) and are regrouped.  dense_h_to_4h rows are [gate; up] as here;
        rotary_pos_emb.inv_freq is recomputed"""
        g = self.geometry()
        hd = g['head_dim']
        nq, nk = g['n_q_heads'] * hd, g['n_kv_heads'] * hd
        per_head = bool(getattr(self.config, 'chatglm_qkv_per_head', False))
        out = {}
        simple = {'input_layernorm.weight': 'input_layernorm.weight',
                  'post_attention_layernorm.weight': 'post_attention_layernorm.weight',
                  'self_attention.dense.weight': 'self_attn.o_proj.weight',
                  'mlp.dense_h_to_4h.weight': 'mlp.gate_up_proj.weight',
                  'mlp.dense_4h_to_h.weight': 'mlp.down_proj.weight'}
        for k, v in sd.items():
            if k == 'transformer.embedding.word_embeddings.weight':
                out['model.embed_tokens.weight'] = v
            elif k == 'transformer.encoder.final_layernorm.weight':
                out['model.norm.weight'] = v
            elif k == 'transformer.output_layer.weight':
                out['lm_head.weight'] = v
            elif k.endswith('rotary_pos_emb.inv_freq'):
                continue
            elif k.startswith(_LAYER):
                li, _, rest = k[len(_LAYER):].partition('.')
                pre = f'model.layers.{li}.'
                if rest.startswith('self_attention.query_key_value.'):
                    kind = rest.rsplit('.', 1)[1]   # weight | bias
                    if per_head:   # [np, 3, hn, ...] -> [3, np * hn, ...]
                        v = v.view(g['n_q_heads'], 3, hd, *v.shape[1:]).transpose(0, 1).reshape(v.shape)
                    out[pre + 'self_attn.q_proj.' + kind] = v[:nq]
                    out[pre + 'self_attn.k_proj.' + kind] = v[nq:nq + nk]
                    out[pre + 'self_attn.v_proj.' + kind] = v[nq + nk:]
                elif rest in simple:
                    out[pre + simple[rest]] = v
                else:
                    raise ValueError(f'unexpected chatglm tensor {k}')
            else:
                raise ValueError(f'unexpected chatglm tensor {k}')
        return out
