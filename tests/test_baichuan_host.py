# -*- coding: utf-8 -*-
"""Baichuan family, host side: the ALiBi slopes, the config translation and its refusals, the W_pack split, the class
flags and the new C ABI symbols."""
import json
import os
import re

import numpy as np
import pytest
import torch

from tests.tiny_baichuan import KINDS, model_class, slopes_f64, tiny_config, w_pack_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('h', list(range(1, 65)))
def test_alibi_slopes_match_bloom(h):
    """ops.alibi_slopes(h) is the definition computed in float64 and rounded once, and equals transformers' BLOOM
    slopes (the same formula) to 1 fp32 ulp for the slopes BLOOM takes as base^1 or base^2.  BLOOM rounds the base
    to fp32 before raising it to the power k, which moves its slope by up to k / 2 ulp: the higher powers are
    compared within that bound"""
    from transformers.models.bloom.modeling_bloom import build_alibi_tensor
    from painlessinferenceacceleration_b200.common import ops
    got = ops.alibi_slopes(h)
    assert got.dtype == torch.float32 and got.shape == (h,)
    assert torch.equal(got, torch.tensor(slopes_f64(h), dtype=torch.float64).to(torch.float32))
    bloom = build_alibi_tensor(torch.ones((1, 2)), h, torch.float32)[:, 0, 1]
    a, b = got.numpy(), bloom.numpy()
    ulps = np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))
    c = 2 ** int(np.floor(np.log2(h)))
    power = np.array([i + 1 for i in range(c)] + [2 * i + 1 for i in range(h - c)])   # BLOOM's exponent of slope i
    assert (ulps <= np.maximum(1, np.ceil(power / 2))).all(), (h, ulps.max())
    assert ulps[power <= 2].max(initial=0) <= 1


def test_alibi_slopes_of_the_published_head_counts():
    from painlessinferenceacceleration_b200.common import ops
    s40 = ops.alibi_slopes(40)
    assert s40[0].item() == pytest.approx(2 ** -0.25) and s40[32].item() == pytest.approx(2 ** -0.125)
    assert len(set(s40.tolist())) == 40
    with pytest.raises(ValueError):
        ops.alibi_slopes(0)


def _cfg(**over):
    c = tiny_config('13b')
    c.update(over)
    return c


def test_config_translation():
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    c = baichuan_config(_cfg())
    assert (c.hidden_size, c.num_attention_heads, c.num_key_value_heads) == (640, 5, 5)
    assert c.max_position_embeddings == 1024 and c.model_max_length == 1024 and not c.tie_word_embeddings
    c = baichuan_config(_cfg(model_max_length=4096))   # ALiBi members: model_max_length only
    assert c.max_position_embeddings == 4096
    c = baichuan_config(dict(tiny_config('2_7b'), max_position_embeddings=4096, model_max_length=8192))
    assert c.max_position_embeddings == 4096 and c.model_max_length == 8192
    c = baichuan_config({k: v for k, v in _cfg().items() if k != 'model_max_length'})
    assert c.max_position_embeddings == 4096


@pytest.mark.parametrize('over,field', [(dict(hidden_act='gelu'), 'hidden_act'),
                                        (dict(quantization_config={'bits': 4}), 'quantization_config'),
                                        (dict(num_attention_heads=7), 'num_attention_heads'),
                                        (dict(num_key_value_heads=1), 'num_key_value_heads')])
def test_config_refusals_name_the_field(over, field):
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    with pytest.raises((ValueError, NotImplementedError), match=field):
        baichuan_config(_cfg(**over))


def test_missing_field_and_model_type(tmp_path):
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    c = _cfg()
    del c['intermediate_size']
    with pytest.raises(ValueError, match='intermediate_size'):
        baichuan_config(c)
    (tmp_path / 'config.json').write_text(json.dumps(_cfg(model_type='llama')))
    with pytest.raises(ValueError, match='model_type'):
        model_class('13b')._pretrained_config(str(tmp_path))
    (tmp_path / 'config.json').write_text(json.dumps(_cfg()))
    assert model_class('13b')._pretrained_config(str(tmp_path)).num_attention_heads == 5


def test_alibi_needs_head_dim_128():
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    with pytest.raises(ValueError, match='head dim 128'):
        model_class('13b')(baichuan_config(_cfg(hidden_size=320)), device='meta')
    model_class('7b')(baichuan_config(dict(tiny_config('7b'), hidden_size=256)), device='meta')   # RoPE: any width


def test_w_pack_split_order():
    """W_pack rows are [q; k; v]: the split gives q_proj / k_proj / v_proj in that order, inv_freq buffers dropped"""
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    m = model_class('2_7b')(baichuan_config(tiny_config('2_7b')), device='meta')
    hid = 512
    q, k, v = (torch.full((hid, hid), float(i)) for i in (1, 2, 3))
    sd = w_pack_state_dict({'model.layers.0.self_attn.q_proj.weight': q, 'model.layers.0.self_attn.k_proj.weight': k,
                            'model.layers.0.self_attn.v_proj.weight': v, 'lm_head.weight': torch.zeros(2)})
    assert list(sd) == ['model.layers.0.self_attn.W_pack.weight', 'lm_head.weight']
    sd['model.layers.0.self_attn.rotary_emb.inv_freq'] = torch.ones(64)
    out = m._convert_checkpoint_keys(sd)
    assert set(out) == {'model.layers.0.self_attn.q_proj.weight', 'model.layers.0.self_attn.k_proj.weight',
                        'model.layers.0.self_attn.v_proj.weight', 'lm_head.weight'}
    for name, want in (('q', q), ('k', k), ('v', v)):
        assert torch.equal(out[f'model.layers.0.self_attn.{name}_proj.weight'], want)
    with pytest.raises(ValueError, match='W_pack'):
        m._convert_checkpoint_keys({'model.layers.0.self_attn.W_pack.weight': torch.zeros(hid, hid)})


def test_class_flags_and_names():
    want = {'7b': ('BaiChuanForCausalLM', False, False, False), '13b': ('BaichuanForCausalLM', True, False, False),
            '2_7b': ('BaichuanForCausalLM', False, True, True), '2_13b': ('BaichuanForCausalLM', True, True, False)}
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    for kind in KINDS:
        cls = model_class(kind)
        assert issubclass(cls, LlamaForCausalLM)
        assert (cls.__name__, cls.alibi, cls.norm_head, cls.rope_fp32) == want[kind], kind
    b = model_class('2_7b', batch=True)
    assert b._batch_generation and b.rope_fp32 and b.norm_head


def test_rope_tables_on_the_host():
    """fp32 tables for Baichuan2-7B (cos of the fp32 angles, not cast), bf16 Llama tables for Baichuan-7B, identity
    tables for the ALiBi members"""
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    m = model_class('2_7b')(baichuan_config(tiny_config('2_7b')), device='cpu')
    cos, sin = m.rope_tables(300)
    assert cos.dtype == torch.float32 and cos.shape == (300, 64)
    inv = 1.0 / (10000 ** (torch.arange(0, 128, 2).float() / 128))
    ang = torch.outer(torch.arange(300, dtype=torch.float32), inv)
    assert torch.allclose(cos, ang.cos(), atol=0, rtol=1e-6) and torch.allclose(sin, ang.sin(), atol=1e-7, rtol=1e-6)
    m7 = model_class('7b')(baichuan_config(tiny_config('7b')), device='cpu')
    assert m7.rope_tables(10)[0].dtype == torch.bfloat16
    m13 = model_class('13b')(baichuan_config(tiny_config('13b')), device='cpu')
    c, s = m13.rope_tables(10)
    assert torch.equal(c, torch.ones_like(c)) and torch.equal(s, torch.zeros_like(s))


def test_new_symbols_in_header_and_ctypes_table():
    from painlessinferenceacceleration_b200 import _lib
    hdr = open(os.path.join(ROOT, 'include', 'pia_b200.h')).read()
    for name in ('pia_tree_attn_alibi_fwd', 'pia_rope_f32_kv_append'):
        assert re.search(r'\bint ' + name + r'\(', hdr), name
        assert name in _lib.SYMBOLS
    assert len(_lib.SYMBOLS['pia_tree_attn_alibi_fwd'][1]) == 9
    assert _lib.SYMBOLS['pia_rope_f32_kv_append'][1] == _lib.SYMBOLS['pia_rope_kv_append'][1]
    assert '#define PIA_ABI_VERSION 3' in hdr
