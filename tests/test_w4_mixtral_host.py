# -*- coding: utf-8 -*-
"""Host checks of int4 (GPTQ / compressed-tensors W4A16) Mixtral checkpoints: both unpack paths give every expert's
codes on a CPU load, the per-expert gate/up interleave of the stacked experts, shard and order independence, and every
refusal - none of which touches a GPU."""
import json
import re

import pytest
import torch

from tests import w4_ckpt, w4_moe_ckpt

pytest.importorskip('safetensors')


def _cls():
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    return MixtralForCausalLM


def _check_codes(m, codes):
    I = m.config.intermediate_size
    for li, layer in enumerate(m.model.layers):
        ex = layer.mlp.experts
        gu, dn = ex.gate_up_proj.codes(), ex.down_proj.codes()
        for e in range(m.config.num_local_experts):
            for x, (src, rows) in (('w1', (gu, slice(0, I))), ('w3', (gu, slice(I, 2 * I))), ('w2', (dn, slice(None)))):
                want = codes[f'model.layers.{li}.block_sparse_moe.experts.{e}.{x}']
                for got, w in zip(src, want):
                    assert torch.equal(got[e][rows], w), (li, e, x)
        for p in w4_moe_ckpt.ATTN:
            for got, w in zip(layer.get_submodule(p).codes(), codes[f'model.layers.{li}.{p}']):
                assert torch.equal(got, w), (li, p)


@pytest.mark.parametrize('name', list(w4_moe_ckpt.FIXTURES))
def test_checkpoint_loads_every_experts_codes_on_the_cpu(name, tmp_path):
    """GPTQ and compressed-tensors, sym / asym, group / channel, I = 384, 8 experts: the attention projections' and
    every expert's (u, s, z) read back exactly; the router, norms and embeddings are the checkpoint's bf16 tensors"""
    codes = w4_moe_ckpt.write(name, str(tmp_path))
    m = _cls().from_pretrained(str(tmp_path), device='cpu')
    assert m._w4 and not m._fp8 and m._fused
    _check_codes(m, codes)
    _, sd, _ = w4_moe_ckpt.build(name)
    assert torch.equal(m.model.layers[1].mlp.gate.weight, sd['model.layers.1.block_sparse_moe.gate.weight'])
    assert torch.equal(m.lm_head.weight, sd['lm_head.weight'])


def test_gptq_and_compressed_tensors_load_to_identical_bytes(tmp_path):
    w4_moe_ckpt.write('mixtral_ct_asym_g128_fp16', str(tmp_path / 'a'))
    w4_moe_ckpt.write('mixtral_gptq_asym_g128_fp16', str(tmp_path / 'b'))
    a, b = (_cls().from_pretrained(str(tmp_path / d), device='cpu') for d in 'ab')
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert sorted(pa) == sorted(pb)
    for k in pa:
        assert torch.equal(pa[k].view(-1).view(torch.uint8), pb[k].view(-1).view(torch.uint8)), k


def test_experts_are_interleaved_per_expert():
    """stored tile t of expert e (rows [e 2I + 128 t, +128)) holds e's gate rows [64 t, +64) then e's up rows
    [I + 64 t, +64), with their scales and zero points; interleaving the stacked [E 2I, H] matrix as a whole would pair
    rows of different experts and fails here"""
    from painlessinferenceacceleration_b200.common import ops
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import _gate_up_order
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import Int4Stack
    E, I, H = 4, 384, 256
    u, s, z = w4_ckpt.random_codes(E * 2 * I, H, 128, False, torch.bfloat16, torch.Generator().manual_seed(9))
    u, s, z = u.view(E, 2 * I, H), s.view(E, 2 * I, -1), z.view(E, 2 * I, -1)
    st = Int4Stack(u, s, z, 128, interleaved=True)
    assert st.shape == (E, 2 * I, H) and tuple(st.scale.shape) == (H // 128, E * 2 * I)
    stored = ops.untile_weight_w4(st.qweight, H)
    for e in range(E):
        for t in range(I // 64):
            r = e * 2 * I + 128 * t
            for half, src in ((0, 64 * t), (64, I + 64 * t)):
                assert torch.equal(stored[r + half:r + half + 64], u[e, src:src + 64]), (e, t, half)
                assert torch.equal(st.scale[:, r + half:r + half + 64].t(), s[e, src:src + 64]), (e, t, half)
                assert torch.equal(st.zero[:, r + half:r + half + 64].t(), z[e, src:src + 64]), (e, t, half)
    whole = _gate_up_order(u.reshape(E * 2 * I, H))
    assert not torch.equal(whole, stored)
    back = st.codes()
    assert torch.equal(back[0], u) and torch.equal(back[1], s) and torch.equal(back[2], z)
    assert torch.equal(st.dequantize()[2], ops.dequantize_w4(u[2], s[2], z[2], 128))


def test_shards_and_order_do_not_matter(tmp_path):
    """three shards split by tensor name (a layer's experts and its router in different files), and one file with the
    tensors in reverse order, load to the same bytes as one file in order"""
    from safetensors.torch import load_file, save_file
    name = 'mixtral_ct_sym_g128_bf16'
    codes = w4_moe_ckpt.write(name, str(tmp_path / 'one'))
    w4_moe_ckpt.write(name, str(tmp_path / 'three'), shards=3)
    _, sd, _ = w4_moe_ckpt.build(name)
    where = {w4_moe_ckpt.shard_of(k, 3) for k in sd if k.startswith('model.layers.0.block_sparse_moe.experts.')}
    assert len(where) == 3
    w4_moe_ckpt.write(name, str(tmp_path / 'rev'))
    f = tmp_path / 'rev' / 'model.safetensors'
    rev = load_file(str(f))
    save_file({k: rev[k] for k in reversed(list(rev))}, str(f), metadata={'format': 'pt'})
    ms = [_cls().from_pretrained(str(tmp_path / d), device='cpu') for d in ('one', 'three', 'rev')]
    _check_codes(ms[1], codes)
    ref = dict(ms[0].named_parameters())
    for m in ms[1:]:
        for k, v in m.named_parameters():
            assert torch.equal(v.view(-1).view(torch.uint8), ref[k].view(-1).view(torch.uint8)), k


def _cfg_dir(tmp_path, name, edit):
    w4_moe_ckpt.write(name, str(tmp_path))
    f = tmp_path / 'config.json'
    d = json.loads(f.read_text())
    edit(d['quantization_config'], d)
    f.write_text(json.dumps(d))
    return str(tmp_path)


def _set(key, value):
    return lambda q, d: q.__setitem__(key, value)


REFUSALS = [
    ('mixtral_ct_sym_g128_bf16', _set('ignore', ['lm_head']), 'block_sparse_moe.gate'),
    ('mixtral_ct_sym_g128_bf16', _set('ignore', ['lm_head', 'model.layers.0.block_sparse_moe.gate']),
     'layers.1.block_sparse_moe.gate'),
    ('mixtral_ct_sym_g128_bf16', _set('ignore', ['re:.*block_sparse_moe.gate']), 'lm_head'),
    ('mixtral_ct_sym_g128_bf16', lambda q, d: q['config_groups']['group_0']['weights'].update(group_size=64),
     'group_size'),
    ('mixtral_ct_sym_g128_bf16', lambda q, d: q['config_groups']['group_0']['weights'].update(num_bits=8), 'num_bits'),
    ('mixtral_ct_sym_g128_bf16', lambda q, d: q['config_groups']['group_0']['weights'].update(actorder='group'),
     'actorder'),
    ('mixtral_gptq_asym_g128_fp16', _set('desc_act', True), 'desc_act'),
    ('mixtral_gptq_asym_g128_fp16', _set('lm_head', True), 'lm_head'),
    ('mixtral_gptq_asym_g128_fp16', _set('quant_method', 'awq'), 'quant_method'),
    ('mixtral_ct_sym_g128_bf16', lambda q, d: d.update(intermediate_size=320), 'intermediate_size'),
    ('mixtral_ct_sym_g128_bf16', lambda q, d: d.update(hidden_size=320), 'hidden_size'),
]


@pytest.mark.parametrize('name,edit,field', REFUSALS, ids=[f'{r[2]}-{i}' for i, r in enumerate(REFUSALS)])
def test_refusals_name_their_field_before_any_gpu_memory(name, edit, field, tmp_path, monkeypatch):
    """config-level refusals raise ValueError naming the field before the model skeleton allocates anything"""
    cls = _cls()
    path = _cfg_dir(tmp_path, name, edit)
    touched = []
    monkeypatch.setattr(cls, '_fp8_skeleton', classmethod(lambda *a, **k: touched.append(1)))
    with pytest.raises(ValueError, match=re.escape(field)):
        cls.from_pretrained(path)
    assert not touched


def test_group_size_that_does_not_divide_the_intermediate_size_is_refused(tmp_path, monkeypatch):
    """group 256 divides hidden_size = 256 but not the I = 384 fixture's intermediate size (the down projection's K)"""
    cls = _cls()
    path = _cfg_dir(tmp_path, 'mixtral_ct_sym_g128_i384',
                    lambda q, d: q['config_groups']['group_0']['weights'].update(group_size=256))
    touched = []
    monkeypatch.setattr(cls, '_fp8_skeleton', classmethod(lambda *a, **k: touched.append(1)))
    with pytest.raises(ValueError, match='intermediate_size=384'):
        cls.from_pretrained(path)
    assert not touched


TENSOR_REFUSALS = [
    # a quantised router, embedding or lm_head tensor
    (lambda sd: sd.update({'model.layers.1.block_sparse_moe.gate.weight_packed': torch.zeros((4, 32), dtype=torch.int32)}),
     'router'),
    (lambda sd: sd.update({'model.embed_tokens.weight_packed': torch.zeros((200, 32), dtype=torch.int32)}),
     'embed_tokens'),
    (lambda sd: sd.update({'lm_head.weight_packed': torch.zeros((200, 32), dtype=torch.int32)}), 'lm_head'),
    # an expert stored in bf16 in an int4 layer
    (lambda sd: sd.update({'model.layers.0.block_sparse_moe.experts.2.w3.weight': torch.zeros((256, 256),
                                                                                             dtype=torch.bfloat16)}),
     'experts.2.w3'),
    (lambda sd: sd.update({'model.layers.1.self_attn.o_proj.weight': torch.zeros((256, 256), dtype=torch.bfloat16)}),
     'o_proj'),
    # expert 1's w3 with scales of group 256 while w1 (and the config) say 128
    (lambda sd: sd.update({'model.layers.0.block_sparse_moe.experts.1.w3.weight_scale':
                           sd['model.layers.0.block_sparse_moe.experts.1.w3.weight_scale'][:, :1].contiguous()}),
     'experts.1.w3'),
    # act-order
    (lambda sd: sd.update({'model.layers.0.block_sparse_moe.experts.0.w2.weight_g_idx': torch.zeros(256, dtype=torch.int32)}),
     'g_idx'),
]


@pytest.mark.parametrize('edit,field', TENSOR_REFUSALS, ids=[r[1] for r in TENSOR_REFUSALS])
def test_tensor_refusals_name_the_tensor(edit, field, tmp_path):
    w4_moe_ckpt.write('mixtral_ct_sym_g128_bf16', str(tmp_path), edit=edit)
    with pytest.raises(ValueError, match=re.escape(field)):
        _cls().from_pretrained(str(tmp_path), device='cpu')


def test_fp8_requests_and_knobs_are_refused(tmp_path, monkeypatch):
    """quantization='fp8' on an int4 Mixtral checkpoint and quantize_fp8() of the loaded model raise ValueError; the
    GEMM knobs that would select another path (PIA_GEMM=0, PIA_GEMM_SET, PIA_MOE_GEMM=0) are refused when the plans are
    built"""
    from types import SimpleNamespace
    cls = _cls()
    w4_moe_ckpt.write('mixtral_ct_sym_g128_bf16', str(tmp_path))
    touched = []
    with monkeypatch.context() as mp:
        mp.setattr(cls, '_fp8_skeleton', classmethod(lambda *a, **k: touched.append(1)))
        with pytest.raises(ValueError, match='already quantised'):
            cls.from_pretrained(str(tmp_path), quantization='fp8')
    assert not touched
    m = cls.from_pretrained(str(tmp_path), device='cpu')
    with pytest.raises(ValueError, match='int4'):
        m.quantize_fp8()
    layer = m.model.layers[0]
    for env in ({'PIA_GEMM': '0'}, {'PIA_GEMM_SET': 'gate_up'}, {'PIA_MOE_GEMM': '0'}):
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            b = SimpleNamespace(rows=64, y=torch.zeros((64, 256), dtype=torch.bfloat16))
            with pytest.raises(ValueError, match='int4'):
                if 'PIA_MOE_GEMM' in env:
                    m._layer_w4_plans(layer, b, 132)
                else:
                    m._w4_plans(b)


def test_int4_checkpoints_flag_is_unchanged():
    """Mixtral reads int4 through its own expert-aware loader; the Llama projection loader's flag stays off"""
    assert _cls().int4_checkpoints is False


def test_new_symbol_is_declared_and_typed():
    import os
    from painlessinferenceacceleration_b200 import _lib
    assert 'pia_gemm_plan_create_grouped_w4' in _lib.SYMBOLS
    restype, argtypes = _lib.SYMBOLS['pia_gemm_plan_create_grouped_w4']
    assert len(argtypes) == 11
    hdr = open(os.path.join(os.path.dirname(_lib.__file__), '..', 'include', 'pia_b200.h')).read()
    assert 'int pia_gemm_plan_create_grouped_w4(' in hdr
    assert hasattr(_lib.load(), 'pia_gemm_plan_create_grouped_w4')
