# -*- coding: utf-8 -*-
"""Qwen (v1), host side: the config translation and its refusals, the checkpoint key mapping (c_attn split, w1 / w2
order), the per-request NTK alpha, the fp32 RoPE and bf16 log-n tables against tables recorded from the reference's
own code (tests/golden/qwen_rope_logn.npz, gen_qwen_golden.py), the log-n length limit and the new C ABI symbol."""
import json
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from tests.tiny_qwen import model_class, ntk_alpha_ref, qwen_state_dict, tiny_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'qwen_rope_logn.npz')


def _mod():
    from painlessinferenceacceleration_b200.models.qwen import modeling_qwen
    return modeling_qwen


def _cpu_model(**over):
    m = _mod()
    return model_class()(m.qwen_config(tiny_config(**over)), device='cpu')


def test_import_path_and_class():
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.common import ops
    cls = model_class()
    assert cls.__name__ == 'QWenLMHeadModel' and issubclass(cls, LlamaForCausalLM)
    assert cls.rmsnorm_rounding == ops.ROUND_ONCE   # not Qwen2's ROUND_TWICE
    assert cls.model_cls.layer_cls.qkv_bias


def test_config_translation():
    """Qwen-7B's published config.json fields"""
    qwen7b = dict(model_type='qwen', vocab_size=151936, hidden_size=4096, intermediate_size=22016,
                  num_hidden_layers=32, num_attention_heads=32, kv_channels=128, layer_norm_epsilon=1e-6,
                  rotary_emb_base=10000, rotary_pct=1.0, seq_length=8192, max_position_embeddings=32768,
                  use_dynamic_ntk=True, use_logn_attn=True, no_bias=True, tie_word_embeddings=False)
    c = _mod().qwen_config(qwen7b)
    assert (c.hidden_size, c.intermediate_size, c.num_attention_heads, c.num_key_value_heads) == (4096, 11008, 32, 32)
    assert c.rms_norm_eps == 1e-6 and c.rotary_emb_base == 10000 and c.vocab_size == 151936
    assert c.seq_length == 8192 and c.use_dynamic_ntk and c.use_logn_attn and not c.tie_word_embeddings
    assert c.eos_token_id == 151643
    c = _mod().qwen_config(dict(qwen7b, layer_norm_epsilon=1e-5, rotary_emb_base=1000000, use_logn_attn=False,
                                use_dynamic_ntk=False, seq_length=2048))
    assert c.rms_norm_eps == 1e-5 and c.rotary_emb_base == 1000000 and c.seq_length == 2048
    assert not c.use_logn_attn and not c.use_dynamic_ntk


@pytest.mark.parametrize('over,field', [(dict(model_type='qwen2'), 'model_type'),
                                        (dict(rotary_pct=0.5), 'rotary_pct'),
                                        (dict(no_bias=False), 'no_bias'),
                                        (dict(kv_channels=64), 'kv_channels'),
                                        (dict(intermediate_size=1023), 'intermediate_size'),
                                        (dict(quantization_config={'bits': 4}), 'quantization_config'),
                                        (dict(num_attention_heads=3), 'num_attention_heads')])
def test_config_refusals_name_the_field(over, field):
    with pytest.raises((ValueError, NotImplementedError), match=field):
        _mod().qwen_config(tiny_config(**over))


def test_missing_field_and_pretrained_config(tmp_path):
    c = tiny_config()
    del c['seq_length']
    with pytest.raises(ValueError, match='seq_length'):
        _mod().qwen_config(c)
    (tmp_path / 'config.json').write_text(json.dumps(tiny_config(model_type='llama')))
    with pytest.raises(ValueError, match='model_type'):
        model_class()._pretrained_config(str(tmp_path))
    (tmp_path / 'config.json').write_text(json.dumps(tiny_config()))
    assert model_class()._pretrained_config(str(tmp_path)).seq_length == 64


def test_c_attn_split_order():
    """c_attn rows (weight) and entries (bias) are [q; k; v]; inv_freq buffers are dropped"""
    m = _cpu_model()
    hid = 512
    sd = {'transformer.h.1.attn.c_attn.weight': torch.cat([torch.full((hid, hid), float(i)) for i in (1, 2, 3)]),
          'transformer.h.1.attn.c_attn.bias': torch.cat([torch.full((hid,), float(i)) for i in (4, 5, 6)]),
          'transformer.rotary_emb.inv_freq': torch.ones(64), 'transformer.wte.weight': torch.zeros(3),
          'transformer.ln_f.weight': torch.zeros(4), 'transformer.h.1.ln_1.weight': torch.zeros(5),
          'transformer.h.1.ln_2.weight': torch.zeros(6), 'transformer.h.1.attn.c_proj.weight': torch.zeros(7),
          'lm_head.weight': torch.zeros(8)}
    out = m._convert_checkpoint_keys(sd)
    pre = 'model.layers.1.'
    for name, w, b in (('q_proj', 1, 4), ('k_proj', 2, 5), ('v_proj', 3, 6)):
        assert torch.equal(out[f'{pre}self_attn.{name}.weight'], torch.full((hid, hid), float(w)))
        assert torch.equal(out[f'{pre}self_attn.{name}.bias'], torch.full((hid,), float(b)))
    want = {'model.embed_tokens.weight': 3, 'model.norm.weight': 4, pre + 'input_layernorm.weight': 5,
            pre + 'post_attention_layernorm.weight': 6, pre + 'self_attn.o_proj.weight': 7, 'lm_head.weight': 8}
    for k, numel in want.items():
        assert out[k].numel() == numel, k
    assert not any('inv_freq' in k for k in out)
    with pytest.raises(ValueError, match='c_attn'):
        m._convert_checkpoint_keys({'transformer.h.0.attn.c_attn.weight': torch.zeros(hid, hid)})


def test_w1_w2_map_to_up_and_gate():
    """a CPU MLP with the converted weights computes the reference's w1(x) * silu(w2(x)) -> c_proj"""
    m = _cpu_model()
    g = torch.Generator().manual_seed(0)
    hid, inter = 512, 512
    w1, w2 = torch.randn((inter, hid), generator=g) * 0.05, torch.randn((inter, hid), generator=g) * 0.05
    c_proj = torch.randn((hid, inter), generator=g) * 0.05
    out = m._convert_checkpoint_keys({'transformer.h.0.mlp.w1.weight': w1, 'transformer.h.0.mlp.w2.weight': w2,
                                      'transformer.h.0.mlp.c_proj.weight': c_proj})
    pre = 'model.layers.0.mlp.'
    x = torch.randn((5, hid), generator=g)
    ours = (F.silu(x @ out[pre + 'gate_proj.weight'].t()) * (x @ out[pre + 'up_proj.weight'].t())) @ \
        out[pre + 'down_proj.weight'].t()
    ref = (F.linear(x, w1) * F.silu(F.linear(x, w2))) @ c_proj.t()
    assert torch.allclose(ours, ref, rtol=1e-6, atol=1e-6)
    swapped = (F.silu(F.linear(x, w1)) * F.linear(x, w2)) @ c_proj.t()
    assert not torch.allclose(swapped, ref, rtol=1e-3, atol=1e-3)


def test_state_dict_round_trip():
    """tests/tiny_qwen.qwen_state_dict (the checkpoint writer of the GPU tests) inverts _convert_checkpoint_keys"""
    m = _cpu_model()
    m.init_weights(seed=1)
    sd = m.state_dict()
    back = m._convert_checkpoint_keys(qwen_state_dict(sd))
    assert set(back) == set(sd)
    assert all(torch.equal(back[k], sd[k]) for k in sd)


@pytest.mark.parametrize('S', [64, 2048, 8192])
def test_ntk_alpha(S):
    m = _mod()
    for L in (S - 1, S, S + 1, 2 * S, 2 * S + 1, 4 * S + 1):
        assert m.ntk_alpha(L, S) == ntk_alpha_ref(L, S), (S, L)
    assert [m.ntk_alpha(L, S) for L in (S - 1, S, S + 1, 2 * S, 2 * S + 1, 4 * S + 1)] == [1, 1, 3, 3, 7, 15]
    assert all(m.ntk_alpha(L, S, use_dynamic_ntk=False) == 1 for L in (1, S + 1, 10 * S))


@pytest.mark.parametrize('base', [10000, 1000000])
@pytest.mark.parametrize('alpha', [1, 3, 7, 31])
def test_rope_tables_match_the_reference(base, alpha):
    g = np.load(GOLDEN)
    rows = g['rows']
    for n in (int(rows.max()) + 1, 33000):
        cos, sin = _mod().rope_tables_f32(128, base, alpha, n)
        assert cos.dtype == torch.float32 and cos.shape == (n, 64)
        assert np.array_equal(cos[rows].numpy(), g[f'cos_b{base}_a{alpha}'])
        assert np.array_equal(sin[rows].numpy(), g[f'sin_b{base}_a{alpha}'])


@pytest.mark.parametrize('S', [64, 2048, 8192])
def test_logn_table_matches_the_reference(S):
    g = np.load(GOLDEN)
    pos = g[f'logn_pos_s{S}']
    t = _mod().logn_table(S, 32767)
    assert t.dtype == torch.bfloat16 and t.shape == (32767,)
    assert np.array_equal(t[pos].view(torch.int16).numpy(), g[f'logn_s{S}'])
    # 1 up to position seq_length - 1, then non-decreasing (the first entries past it may round to 1 in bf16)
    assert (t[:S].float() == 1).all() and (t[S:].float() >= 1).all() and (t[2 * S:].float() > 1).all()
    assert (t[1:].float() >= t[:-1].float()).all()


def test_model_tables_switch_with_alpha():
    """rope_tables gives alpha 1's tables; _start_request copies the request's alpha's tables in place, only when the
    alpha changes, and refuses max_length > 32767 with log-n"""
    m = _cpu_model()
    mod = _mod()
    cos, sin = m.rope_tables(300)
    c1, s1 = mod.rope_tables_f32(128, 10000, 1, 300)
    assert torch.equal(cos, c1) and torch.equal(sin, s1)
    rt = SimpleNamespace(rope_cos=cos.clone(), rope_sin=sin.clone(), ntk_alpha=1.0)
    p_cos = rt.rope_cos.data_ptr()
    m._start_request(rt, 129)   # seq_length 64: alpha 7
    c7, s7 = mod.rope_tables_f32(128, 10000, 7, 300)
    assert rt.ntk_alpha == 7 and rt.rope_cos.data_ptr() == p_cos
    assert torch.equal(rt.rope_cos, c7) and torch.equal(rt.rope_sin, s7)
    m._start_request(rt, 10)
    assert rt.ntk_alpha == 1 and torch.equal(rt.rope_cos, c1)
    m._start_request(rt, 10, max_length=32767)
    with pytest.raises(ValueError, match='32767'):
        m._start_request(rt, 10, max_length=32768)
    _cpu_model(use_logn_attn=False)._start_request(rt, 10, max_length=40000)
    off = _cpu_model(use_dynamic_ntk=False)
    off._start_request(rt, 1000)
    assert rt.ntk_alpha == 1


def test_new_symbol_in_header_and_ctypes_table():
    from painlessinferenceacceleration_b200 import _lib
    hdr = open(os.path.join(ROOT, 'include', 'pia_b200.h')).read()
    name = 'pia_rope_f32_logn_kv_append'
    assert re.search(r'\bint ' + name + r'\(', hdr)
    assert 'qwen/modeling_qwen.py:223-227' in hdr
    args = _lib.SYMBOLS[name][1]
    plain = _lib.SYMBOLS['pia_rope_f32_kv_append'][1]
    assert args[:-1] == plain[:-1] + [_lib.vp] and args[-1] == plain[-1]   # + the scale table before the stream
    assert '#define PIA_ABI_VERSION 3' in hdr
