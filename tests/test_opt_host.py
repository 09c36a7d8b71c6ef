# -*- coding: utf-8 -*-
"""OPT, host side: the config refusals, the checkpoint key mapping for all three prefixes, the tied lm_head, the
module tree against transformers' own OPTForCausalLM, the tree-position rule of pia_learned_pos_embed restated on the
host against positions recorded from the reference's own OPTLearnedPositionalEmbedding (tests/golden/
opt_tree_positions.npz, gen_opt_golden.py), geometry(), the max_position_embeddings refusal and the new C ABI
symbols."""
import os
import re

import numpy as np
import pytest
import torch

from tests.tiny_opt import MAX_POS, hf_model, tiny_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'opt_tree_positions.npz')


def _cls(batch=False):
    if batch:
        from painlessinferenceacceleration_b200.models.opt.modeling_opt_batch import OPTForCausalLM
    else:
        from painlessinferenceacceleration_b200.models.opt.modeling_opt import OPTForCausalLM
    return OPTForCausalLM


def _cpu(shape=64, **over):
    cfg = tiny_config(shape)
    for k, v in over.items():
        setattr(cfg, k, v)
    return _cls()(cfg, device='cpu')


@pytest.mark.parametrize('field,value,exc', [
    ('activation_function', 'gelu', NotImplementedError),   # Galactica
    ('enable_bias', False, NotImplementedError),
    ('layer_norm_elementwise_affine', False, NotImplementedError),
    ('quantization_config', {'quant_method': 'gptq', 'bits': 4}, NotImplementedError),
    ('num_attention_heads', 3, ValueError),                  # 256 % 3
    ('hidden_size', 4 * 136, ValueError),                    # head dim 136 > 128
    ('model_type', 'gpt2', ValueError),
])
def test_config_refusals_name_the_field(field, value, exc):
    cfg = tiny_config(64)
    setattr(cfg, field, value)
    with pytest.raises(exc, match=field if field != 'hidden_size' else 'head dim'):
        _cls()(cfg, device='cpu')


@pytest.mark.parametrize('shape', [64, 80, 128, '350m'])
def test_module_tree_and_names_are_hf(shape):
    hf = hf_model(shape, device='cpu')
    ours = _cpu(shape)
    assert set(dict(ours.named_parameters())) == set(dict(hf.named_parameters()))
    for k, v in hf.state_dict().items():
        if k != 'lm_head.weight':
            assert tuple(ours.state_dict()[k].shape) == tuple(v.shape), k
    pre = shape != '350m'
    assert (ours.model.decoder.final_layer_norm is None) == (not pre)
    assert (ours.model.decoder.project_in is None) == pre and (ours.model.decoder.project_out is None) == pre


def test_key_mapping_for_all_three_prefixes_and_the_tied_head():
    """OPTForCausalLM (`model.decoder.`), OPTModel (`decoder.`) and OPTDecoder (no prefix) state dicts load the same
    tensors; a stored lm_head.weight is skipped by a tied model and read by an untied one"""
    hf = hf_model(64, device='cpu')
    sd = hf.state_dict()
    full = _cpu().load_hf_state_dict(sd)
    assert full.lm_head.weight is full.model.decoder.embed_tokens.weight
    model_sd = {k[len('model.'):]: v for k, v in sd.items() if k.startswith('model.')}
    dec_sd = {k[len('model.decoder.'):]: v for k, v in sd.items() if k.startswith('model.decoder.')}
    assert 'decoder.layers.0.fc1.weight' in model_sd and 'layers.0.fc1.weight' in dec_sd
    for alt in (model_sd, dec_sd):
        m = _cpu().load_hf_state_dict(alt)
        for (k, a), b in zip(full.state_dict().items(), m.state_dict().values()):
            assert torch.equal(a, b), k
    # a tied model ignores a stored head that differs from the embeddings
    odd = dict(sd)
    odd['lm_head.weight'] = torch.zeros_like(sd['lm_head.weight'])
    m = _cpu().load_hf_state_dict(odd)
    assert torch.equal(m.lm_head.weight, sd['model.decoder.embed_tokens.weight'].to(torch.bfloat16))
    # an untied one reads it, and needs it
    cfg = tiny_config(64, tie=False)
    untied = _cls()(cfg, device='cpu')
    assert untied.lm_head.weight is not untied.model.decoder.embed_tokens.weight
    untied.load_hf_state_dict(odd)
    assert not untied.lm_head.weight.any()
    with pytest.raises(RuntimeError, match='missing'):
        _cls()(cfg, device='cpu').load_hf_state_dict(dec_sd)


def test_missing_and_misshapen_tensors_raise():
    sd = hf_model(64, device='cpu').state_dict()
    part = {k: v for k, v in sd.items() if 'layers.1.fc2' not in k}
    with pytest.raises(RuntimeError, match='missing'):
        _cpu().load_hf_state_dict(part)
    bad = dict(sd)
    bad['model.decoder.layers.0.fc1.weight'] = torch.zeros(3, 3)
    with pytest.raises(ValueError, match='fc1'):
        _cpu().load_hf_state_dict(bad)


def _tree_pos(rows, P, pad, max_pos):
    """pia_learned_pos_embed's position of a row: max(P - pad, 0) + popcount(row) - 1, clamped to [0, max_pos)"""
    depth = np.array([sum(bin(int(w) & 0xFFFFFFFFFFFFFFFF).count('1') for w in r) for r in rows]) - 1
    return np.clip(max(P - pad, 0) + depth, 0, max_pos - 1)


def test_tree_positions_match_the_reference_embedding():
    """the rank-4 (lookahead) branch of the reference's OPTLearnedPositionalEmbedding reads row offset + our tree
    position for every node; the 2-D (prefill) branch reads the rows the prefill chain chunks give, except at
    left-pad rows, which the reference sends to position -1 and which no unpadded row ever attends to"""
    z = np.load(GOLDEN)
    assert int(z['offset']) == 2
    from painlessinferenceacceleration_b200.models.opt.modeling_opt import POS_OFFSET
    assert POS_OFFSET == int(z['offset'])
    k = 0
    while f'tree{k}_meta' in z:
        n, P, pad = z[f'tree{k}_meta'].tolist()
        assert np.array_equal(_tree_pos(z[f'tree{k}_rows'], P, pad, MAX_POS), z[f'tree{k}_pos']), k
        k += 1
    assert k >= 4
    k = 0
    while f'prompt{k}_meta' in z:
        T, pad = z[f'prompt{k}_meta'].tolist()
        # the prefill pass: chain rows of a chunk starting at P = 0, the first `pad` columns cleared
        full = [((1 << (i + 1)) - 1) & ~((1 << pad) - 1) for i in range(T)]
        rows = [[(r >> (64 * w)) & 0xFFFFFFFFFFFFFFFF for w in range(2)] for r in full]
        ours = _tree_pos(rows, 0, pad, MAX_POS)
        ref = z[f'prompt{k}_pos']
        assert np.array_equal(ours[pad:], ref[pad:]) and (ref[:pad] == -1).all(), k
        k += 1
    assert k >= 2


def test_geometry_pads_only_off_sizes():
    assert _cpu(64).geometry()['head_dim'] == 64
    assert _cpu(128).geometry()['head_dim'] == 128
    g = _cpu(80).geometry()
    assert g['head_dim'] == 128 and g['n_q_heads'] == g['n_kv_heads'] == 3 and g['hidden'] == 240
    assert g['inter'] == 480 and g['vocab'] == 200 and g['n_layers'] == 2


def test_max_position_embeddings_is_enforced():
    m = _cpu()
    m.check_max_length(MAX_POS)
    m._start_request(None, 10, MAX_POS)
    with pytest.raises(ValueError, match='max_position_embeddings'):
        m._start_request(None, 10, MAX_POS + 1)
    with pytest.raises(ValueError, match='max_position_embeddings'):
        m._start_request(None, MAX_POS + 1)
    b = _cls(batch=True)(tiny_config(64), device='cpu')
    with pytest.raises(ValueError, match='max_position_embeddings'):
        b.lookahead_generation(torch.zeros((2, 8), dtype=torch.long), max_length=MAX_POS + 1)
    with pytest.raises(ValueError, match='max_position_embeddings'):
        b.lookahead_generation(torch.zeros((2, 8), dtype=torch.long), decoding_kwargs={'max_length': MAX_POS + 5})


def test_quantize_fp8_refuses_shapes_off_128_before_converting():
    m = _cpu(80)
    with pytest.raises(ValueError, match='128'):
        m.quantize_fp8()
    assert not m._fp8 and not m._fused


def test_gemm_knobs_are_refused(monkeypatch):
    m = _cpu()
    for knob, val in (('PIA_ATTN_FUSED', '1'), ('PIA_GEMM', '0'), ('PIA_GEMM_SET', 'x')):
        monkeypatch.setenv(knob, val)
        with pytest.raises(ValueError, match=knob):
            m._runtime(256, 64)
        monkeypatch.delenv(knob)
    assert m._rt is None


def test_new_symbols_in_the_header_and_the_binding():
    hdr = open(os.path.join(ROOT, 'include', 'pia_b200.h')).read()
    from painlessinferenceacceleration_b200 import _lib
    for name in ('pia_kv_append_qscale', 'pia_learned_pos_embed', 'pia_gemm_plan_set_relu'):
        assert re.search(r'\bint ' + name + r'\(', hdr), name
        assert name in _lib.SYMBOLS, name
    assert '#define PIA_ABI_VERSION 3' in hdr
