# -*- coding: utf-8 -*-
"""CPU checks of the BLOOM class: config translation from a published config.json, the refusals (each naming its
field), the query_key_value regroup against transformers' own head split, checkpoint names with and without the
`transformer.` prefix, tied / untied lm_head, the knob refusals and the two new C entry points."""
import json
import os
import re

import pytest
import torch

from tests.tiny_bloom import tiny_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# bloom-560m's config.json as published (n_embed / num_attention_heads / n_layer)
BLOOM_560M = dict(apply_residual_connection_post_layernorm=False, architectures=['BloomForCausalLM'],
                  attention_dropout=0.0, attention_softmax_in_fp32=True, bias_dropout_fusion=True, bos_token_id=1,
                  eos_token_id=2, hidden_dropout=0.0, initializer_range=0.02, layer_norm_epsilon=1e-05,
                  masked_softmax_fusion=True, model_type='bloom', n_embed=1024, n_inner=None, n_layer=24,
                  num_attention_heads=16, offset_alibi=100, pad_token_id=3, pretraining_tp=1, skip_bias_add=True,
                  skip_bias_add_qkv=False, slow_but_exact=False, unk_token_id=0, use_cache=True, vocab_size=250880)


def _cls():
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import BloomForCausalLM
    return BloomForCausalLM


def _write(tmp_path, **over):
    (tmp_path / 'config.json').write_text(json.dumps(dict(BLOOM_560M, **over)))
    return str(tmp_path)


def test_config_translation(tmp_path):
    cls = _cls()
    cfg = cls._pretrained_config(_write(tmp_path))
    assert (cfg.hidden_size, cfg.n_head, cfg.n_layer, cfg.vocab_size) == (1024, 16, 24, 250880)
    assert cfg.tie_word_embeddings and cfg.layer_norm_epsilon == 1e-5
    m = cls(cfg, device='meta')
    assert m.head_dim == 64
    assert m.geometry() == dict(n_layers=24, hidden=1024, n_q_heads=16, n_kv_heads=16, head_dim=128, inter=4096,
                                vocab=250880)
    assert m.lm_head.weight is m.transformer.word_embeddings.weight
    names = {n for n, _ in m.named_parameters()}
    for n in ('transformer.word_embeddings.weight', 'transformer.word_embeddings_layernorm.bias',
              'transformer.h.23.input_layernorm.weight', 'transformer.h.0.self_attention.query_key_value.bias',
              'transformer.h.0.self_attention.dense.weight', 'transformer.h.0.post_attention_layernorm.bias',
              'transformer.h.0.mlp.dense_h_to_4h.bias', 'transformer.h.0.mlp.dense_4h_to_h.weight',
              'transformer.ln_f.weight'):
        assert n in names, n


@pytest.mark.parametrize('over,field', [
    (dict(apply_residual_connection_post_layernorm=True), 'apply_residual_connection_post_layernorm'),
    (dict(pretraining_tp=4, slow_but_exact=True), 'slow_but_exact'),
    (dict(n_embed=1000), 'hidden_size'),
    (dict(n_embed=4096), 'head dim'),
    (dict(quantization_config={'quant_method': 'gptq', 'bits': 4}), 'quantization_config'),
])
def test_config_refusals_name_the_field(tmp_path, over, field):
    cls = _cls()
    with pytest.raises((ValueError, NotImplementedError), match=field):
        cls.from_pretrained(_write(tmp_path, **over), device=torch.device('cpu'))


def test_accepted_variants(tmp_path):
    """pretraining_tp > 1 alone changes nothing in inference (HF ignores it without slow_but_exact)"""
    cls = _cls()
    cls(cls._pretrained_config(_write(tmp_path, pretraining_tp=4)), device='meta')


def test_model_type_is_checked(tmp_path):
    from transformers import GPT2Config
    cls = _cls()
    (tmp_path / 'config.json').write_text(json.dumps(dict(model_type='gpt2', n_embd=256, n_head=4, n_layer=2,
                                                          vocab_size=200)))
    with pytest.raises(ValueError, match='model_type'):
        cls.from_pretrained(str(tmp_path), device=torch.device('cpu'))
    with pytest.raises(ValueError, match='model_type'):
        cls(GPT2Config(n_embd=256, n_head=4, n_layer=2, vocab_size=200), device='meta')


@pytest.mark.parametrize('head_dim', [64, 80, 96, 128])
def test_qkv_regroup_matches_hf_head_split(head_dim):
    """the regrouped [q heads | k heads | v heads] rows of weight and bias are exactly the q / k / v of transformers'
    BloomAttention._reshape (view(H, 3, d)) of the checkpoint's rows"""
    from transformers.models.bloom.modeling_bloom import BloomAttention
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import regroup_qkv
    cfg = tiny_config(head_dim)
    H, E, d = cfg.n_head, cfg.hidden_size, head_dim
    attn = BloomAttention(cfg, layer_idx=0)
    split = attn._reshape if hasattr(attn, '_reshape') else attn._split_heads
    g = torch.Generator().manual_seed(head_dim)
    w = torch.randn((3 * E, E), generator=g)
    b = torch.randn((3 * E,), generator=g)
    q, k, v = split(w.t()[None])              # each [1, H, E, d]: row e of the fused output = column e of w^T
    want = torch.stack([q[0], k[0], v[0]])    # [3, H, E, d]
    got = regroup_qkv(w, H).view(3, H, d, E).permute(0, 1, 3, 2)
    assert torch.equal(got, want)
    q, k, v = split(b[None, None])
    assert torch.equal(regroup_qkv(b, H).view(3, H, d), torch.stack([q[0, :, 0], k[0, :, 0], v[0, :, 0]]))


def _hf_cpu(head_dim, tie=True):
    from transformers import BloomForCausalLM as HF
    torch.manual_seed(0)
    return HF(tiny_config(head_dim, tie=tie)).float()


@pytest.mark.parametrize('prefixed', [True, False])
def test_checkpoint_keys_with_and_without_prefix(prefixed):
    """a BloomForCausalLM state dict (transformer.*) and a BloomModel one (no prefix) load into the same tensors"""
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import regroup_qkv
    hf = _hf_cpu(80)
    sd = hf.state_dict() if prefixed else hf.transformer.state_dict()
    assert any(k.startswith('transformer.') for k in sd) == prefixed
    m = _cls()(hf.config, device='cpu').load_hf_state_dict(sd)
    ours = dict(m.named_parameters())
    for k, v in hf.transformer.state_dict().items():
        want = v.to(torch.bfloat16)
        if 'query_key_value' in k:
            want = regroup_qkv(want, hf.config.n_head)
        assert torch.equal(ours['transformer.' + k], want), k


def test_tied_and_untied_lm_head():
    cls = _cls()
    tied = cls(tiny_config(64), device='cpu').load_hf_state_dict(_hf_cpu(64).state_dict())
    assert tied.lm_head.weight is tied.transformer.word_embeddings.weight
    assert 'lm_head.weight' not in dict(tied.named_parameters())
    hf = _hf_cpu(64, tie=False)
    with torch.no_grad():
        hf.lm_head.weight.mul_(3.0)
    untied = cls(hf.config, device='cpu').load_hf_state_dict(hf.state_dict())
    assert untied.lm_head.weight is not untied.transformer.word_embeddings.weight
    assert torch.equal(untied.lm_head.weight, hf.lm_head.weight.to(torch.bfloat16))
    assert not torch.equal(untied.lm_head.weight, untied.transformer.word_embeddings.weight)
    sd = {k: v for k, v in hf.state_dict().items() if k != 'lm_head.weight'}
    with pytest.raises(RuntimeError, match='lm_head.weight'):
        cls(hf.config, device='cpu').load_hf_state_dict(sd)


@pytest.mark.parametrize('knob,value', [('PIA_ATTN_FUSED', '1'), ('PIA_GEMM', '1'), ('PIA_GEMM', '0'),
                                        ('PIA_GEMM_SET', 'gate_up')])
def test_knobs_are_refused_before_a_runtime_exists(monkeypatch, knob, value):
    m = _cls()(tiny_config(64), device='meta')
    monkeypatch.setenv(knob, value)
    with pytest.raises(ValueError, match=knob):
        m._runtime(256, 64)
    assert m._rt is None
    if knob != 'PIA_ATTN_FUSED':
        with pytest.raises(ValueError, match='BLOOM'):
            m._runtime(256, 64)


def test_fp8_is_refused(tmp_path):
    cls = _cls()
    with pytest.raises(NotImplementedError):
        cls(tiny_config(128), device='meta').quantize_fp8()
    with pytest.raises(NotImplementedError, match='fp8'):
        cls.from_pretrained(_write(tmp_path), quantization='fp8')


def test_init_weights_layout():
    m = _cls()(tiny_config(96), device='cpu').init_weights(seed=1)
    p = dict(m.named_parameters())
    assert torch.equal(p['transformer.h.1.input_layernorm.weight'], torch.ones(480, dtype=torch.bfloat16))
    assert float(p['transformer.ln_f.bias'].abs().sum()) == 0
    assert float(p['transformer.h.0.self_attention.query_key_value.bias'].abs().sum()) == 0
    assert float(p['transformer.h.0.mlp.dense_h_to_4h.weight'].float().std()) > 0.01


def test_new_symbols_in_header_and_ctypes_table():
    from painlessinferenceacceleration_b200 import _lib
    hdr = open(os.path.join(ROOT, 'include', 'pia_b200.h')).read()
    for name in ('pia_layernorm', 'pia_bloom_gelu'):
        assert re.search(r'\bint ' + name + r'\(', hdr), name
        assert name in _lib.SYMBOLS
    assert len(_lib.SYMBOLS['pia_layernorm'][1]) == 10
    assert len(_lib.SYMBOLS['pia_bloom_gelu'][1]) == 4
    assert '#define PIA_ABI_VERSION 3' in hdr
    assert 'bloom/modeling_bloom.py:194-203' in hdr
