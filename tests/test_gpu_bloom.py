# -*- coding: utf-8 -*-
"""BLOOM on the H100: pia_layernorm against torch's LayerNorm, pia_bloom_gelu over every bf16 bit pattern against
transformers' bloom_gelu_forward evaluated by eager torch, both kernels inside a captured graph, the lossless property
of the padded-head ALiBi verify forward at head dims 64 / 80 / 96 / 128 against transformers' own BloomForCausalLM in
fp32, and the tiny models through generate(), the oracle loop and checkpoint loading.  `big`: the BLOOM-7b1 shape
through the loop."""
import json

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from tests.test_gpu_generate import OursBackend
from tests.test_gpu_head_dim64 import _tree
from tests.tiny_bloom import hf_logits, tiny_model
from tests.tiny_models import prompts

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
DIMS = [64, 80, 96, 128]


# ---------------------------------------------------------------------------------------------------------------
# the kernels
# ---------------------------------------------------------------------------------------------------------------
def _ordered(t):
    """bf16 values -> integers in value order (adjacent bf16 values differ by 1; +0 and -0 both map to 0)"""
    i = t.contiguous().view(torch.int16).to(torch.int32)
    return torch.where(i < 0, -(i & 0x7FFF), i)


def _ln_inputs(rows, hidden, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn((rows, hidden), device=DEV, generator=g) * 2 + 0.5).to(torch.bfloat16)
    r = torch.randn((rows, hidden), device=DEV, generator=g).to(torch.bfloat16)
    w = (1 + 0.3 * torch.randn((hidden,), device=DEV, generator=g)).to(torch.bfloat16)
    b = (0.1 * torch.randn((hidden,), device=DEV, generator=g)).to(torch.bfloat16)
    return x, r, w, b


@pytest.mark.parametrize('resid', [False, True])
@pytest.mark.parametrize('hidden', [1024, 1536, 2560, 4096, 14336])
@pytest.mark.parametrize('rows', [1, 64, 256])
def test_layernorm(rows, hidden, resid):
    """residual_out bit for bit = bf16(x + r); every y within one bf16 ulp of F.layer_norm in fp32 rounded once.  The
    ulp is taken at the magnitude of the larger of the two addends x_hat * w and b: where they cancel, the result is
    far smaller than either, and an fp32 evaluation (torch's as well as ours) is only exact to the addends' fp32 ulp,
    which is many bf16 ulps of the small result.  The share of elements that differ from torch's own bf16
    F.layer_norm stays below 1 %"""
    from painlessinferenceacceleration_b200.common import ops
    eps = 1e-5
    x, r, w, b = _ln_inputs(rows, hidden, rows * hidden + resid)
    ro = torch.full_like(x, 9.0)
    y = torch.full_like(x, 9.0)
    ops.layernorm(x, r if resid else None, w, b, eps, ro, y)
    torch.cuda.synchronize()
    xs = (x.float() + r.float()).to(torch.bfloat16) if resid else x
    assert torch.equal(ro, xs)
    f = F.layer_norm(xs.float(), (hidden,), w.float(), b.float(), eps)
    ref = f.to(torch.bfloat16)
    xhat = F.layer_norm(xs.float(), (hidden,), None, None, eps)
    scale = torch.maximum(torch.maximum((xhat * w.float()).abs(), b.float().abs().expand_as(f)), f.abs())
    ulp = torch.exp2(torch.floor(torch.log2(scale.clamp_min(2.0 ** -100))) - 7)
    assert bool(((y.float() - ref.float()).abs() <= ulp).all())
    clean = f.abs() >= 0.5 * scale   # no cancellation: one ulp of the result itself
    assert int((_ordered(y) - _ordered(ref)).abs()[clean].max()) <= 1
    share = (y != F.layer_norm(xs, (hidden,), w, b, eps)).float().mean().item()
    print(f'rows={rows} hidden={hidden} resid={resid}: {100 * share:.3f} % of elements differ from torch bf16')
    assert share < 0.01


def test_layernorm_in_place_and_without_residual_out():
    from painlessinferenceacceleration_b200.common import ops
    x, _, w, b = _ln_inputs(64, 4096, 5)
    want = torch.empty_like(x)
    ops.layernorm(x, None, w, b, 1e-5, None, want)
    y = x.clone()
    ops.layernorm(y, None, w, b, 1e-5, None, y)
    torch.cuda.synchronize()
    assert torch.equal(y, want)


def test_bloom_gelu_every_bf16_bit_pattern():
    """all 65 536 bf16 values at once, bit for bit against transformers' bloom_gelu_forward run by eager torch on the
    same GPU; NaNs match as NaNs; in place gives the same bits"""
    from transformers.models.bloom.modeling_bloom import bloom_gelu_forward
    from painlessinferenceacceleration_b200.common import ops
    x = torch.arange(-32768, 32768, dtype=torch.int32, device=DEV).to(torch.int16).view(torch.bfloat16)
    want = bloom_gelu_forward(x)
    got = ops.bloom_gelu(x, out=torch.empty_like(x))
    inplace = ops.bloom_gelu(x.clone())
    torch.cuda.synchronize()
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan) and torch.equal(inplace.isnan(), nan)
    bad = (got.view(torch.int16) != want.view(torch.int16)) & ~nan
    assert int(bad.sum()) == 0, (x[bad][:8].tolist(), got[bad][:8].tolist(), want[bad][:8].tolist())
    assert torch.equal(inplace.view(torch.int16)[~nan], got.view(torch.int16)[~nan])


def test_kernels_in_a_captured_graph_and_refusals():
    """both kernels replay inside a CUDA graph with the eager results; an invalid hidden / length raises and launches
    nothing"""
    from painlessinferenceacceleration_b200.common import ops
    x, r, w, b = _ln_inputs(64, 4096, 7)
    act = (torch.randn((64, 16384), device=DEV) * 3).to(torch.bfloat16)
    ro, y, g_out = torch.empty_like(x), torch.empty_like(x), torch.empty_like(act)
    ops.layernorm(x, r, w, b, 1e-5, ro, y)
    ops.bloom_gelu(act, out=g_out)
    want = (ro.clone(), y.clone(), g_out.clone())
    for t in (ro, y, g_out):
        t.zero_()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.layernorm(x, r, w, b, 1e-5, ro, y)
        ops.bloom_gelu(act, out=g_out)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(ro, want[0]) and torch.equal(y, want[1]) and torch.equal(g_out, want[2])
    l0 = ops.launch_count()
    for hidden in (12, 16392):
        z = torch.zeros((4, hidden), dtype=torch.bfloat16, device=DEV)
        wz = torch.ones((hidden,), dtype=torch.bfloat16, device=DEV)
        with pytest.raises(AssertionError, match='layernorm'):
            ops.layernorm(z, None, wz, wz, 1e-5, None, z)
    with pytest.raises(AssertionError, match='bloom_gelu'):
        ops.bloom_gelu(torch.zeros((12,), dtype=torch.bfloat16, device=DEV))
    assert ops.launch_count() == l0


# ---------------------------------------------------------------------------------------------------------------
# lossless: the verify logits of every draft node = a causal forward over prefix + root-to-node path
# ---------------------------------------------------------------------------------------------------------------
def _check(got, truth, eager):
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)


@pytest.mark.parametrize('head_dim', DIMS)
def test_tree_verify_logits_are_lossless(head_dim):
    """a prompt (two chain chunks), then one random 64-node tree: each node's verify-logit row vs transformers'
    BloomForCausalLM in fp32 over prompt + its root-to-node path, within 2 x the bf16 eager model's own error + 0.02"""
    model, hf = tiny_model(head_dim, seed=3)
    torch.manual_seed(4)
    T0, n = 100, 64
    prompt = torch.randint(3, 200, (1, T0), device=DEV)
    rows = _tree(np.random.default_rng(5), n, max_depth=10)
    ids = torch.randint(3, 200, (1, n), device=DEV)
    be = OursBackend(model, max_seq=512)
    m01 = torch.tril(torch.ones((1, 1, T0, T0), dtype=torch.long, device=DEV))
    be.forward(prompt, m01, None)
    tm = torch.zeros((1, 1, n, T0 + n), dtype=torch.long, device=DEV)
    tm[..., :T0] = 1
    for i, r in enumerate(rows):
        for j in range(n):
            if (r >> j) & 1:
                tm[0, 0, i, T0 + j] = 1
    got = be.forward(ids, tm, None)[0].float()
    for i in list(range(0, n, 7)) + [n - 1]:
        path = [j for j in range(n) if (rows[i] >> j) & 1]
        seq = torch.cat([prompt[0], ids[0, path]])
        _check(got[i], hf_logits(hf, seq)[-1], hf_logits(hf, seq, torch.bfloat16)[-1])


@pytest.mark.parametrize('head_dim', [64, 128])
def test_prefill_with_left_padding_is_lossless(head_dim):
    """the prefill pass of a left-padded prompt: its last-row logits vs the HF forward of the unpadded prompt"""
    model, hf = tiny_model(head_dim, seed=6)
    torch.manual_seed(7)
    pad, T = 13, 150
    p = torch.randint(3, 200, (T,), device=DEV)
    rt = model._runtime(512, 64)
    rt.set_request(0, pad, 1 << 30)
    rt.seq[0, :pad] = 0
    rt.seq[0, pad:pad + T] = p.to(torch.int32)
    model._prefill_logits(rt, pad + T)
    _check(rt.logits[0].float(), hf_logits(hf, p)[-1], hf_logits(hf, p, torch.bfloat16)[-1])


# ---------------------------------------------------------------------------------------------------------------
# the tiny models
# ---------------------------------------------------------------------------------------------------------------
def _cache(model):
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    model.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    return model


@pytest.mark.parametrize('head_dim,penalty', [(64, 1.0), (64, 1.1), (80, 1.0), (96, 1.1), (128, 1.0), (128, 1.1)])
def test_generate_equals_plain_greedy(head_dim, penalty):
    """lookahead generate() (prefill + tree drafts) gives the tokens of plain greedy decoding with the same kernels,
    and a second pass over the same prompts accepts drafts"""
    model = _cache(tiny_model(head_dim, seed=1)[0])
    edls = []
    for rep in range(2):
        for p in prompts(21, 2, 40, 200):
            p = p.to(DEV)
            g = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               decoding_kwargs={'use_lookahead': False})
            o = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               return_dict_in_generate=True,
                               decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
            assert o.sequences[0].tolist() == g[0].tolist(), (head_dim, rep)
            edls += o.kwargs['edls'][1:]
    assert max(edls) > 2


def test_do_sample():
    """an untied lm_head (initialised at std 0.06, unlike the tied 0.5-std embeddings) keeps the logits soft enough
    for sampling to leave the greedy path"""
    model = _cache(tiny_model(96, seed=2, tie=False)[0])
    torch.manual_seed(11)
    differs = 0
    for p in prompts(9, 3, 24, 200):
        p = p.to(DEV)
        g = model.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
        o = model.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, do_sample=True, return_dict_in_generate=True,
                           decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
        seq = o.sequences[0].tolist()
        assert seq[:24] == p[0].tolist() and len(seq) <= 24 + 40 and sum(o.kwargs['edls']) == len(seq) - 24
        assert all(0 <= t < 200 for t in seq)
        differs += seq != g[0].tolist()
    assert differs >= 1


@pytest.mark.parametrize('head_dim,penalty', [(64, 1.1), (80, 1.0), (128, 1.0)])
def test_loop_is_exact_given_the_same_logits(head_dim, penalty):
    """the oracle loop drives one copy of our model, the fused device loop another: tokens, dls, edls identical"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    a = _cache(tiny_model(head_dim, seed=6)[0])
    b = tiny_model(head_dim, seed=6)[0]
    otrie = OracleLookaheadCache(eos_ids=[2])
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 3, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=56, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=56, eos_token_id=[2], repetition_penalty=penalty,
                                     decoding_length=64,
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=90 + 56 + 129))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (head_dim, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (head_dim, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def _verify_logits(model, p):
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    return OursBackend(model).forward(p, m01, None)[0].float()


@pytest.mark.parametrize('head_dim,tie', [(64, True), (128, False)])
def test_from_pretrained(tmp_path, head_dim, tie):
    """an HF save_pretrained directory (transformer.* names) and an unprefixed BloomModel-style one load into the
    logits of the same weights handed over directly"""
    from safetensors.torch import save_file
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import BloomForCausalLM
    direct, hf = tiny_model(head_dim, seed=10, tie=tie)
    hf.save_pretrained(str(tmp_path / 'hf'))
    plain = tmp_path / 'plain'
    plain.mkdir()
    (plain / 'config.json').write_text(json.dumps(hf.config.to_dict()))
    sd = {k: v.detach().cpu().contiguous() for k, v in hf.transformer.state_dict().items()}
    if not tie:
        sd['lm_head.weight'] = hf.lm_head.weight.detach().cpu().contiguous()
    keys = sorted(sd)
    save_file({k: sd[k] for k in keys[:len(keys) // 2]}, str(plain / 'model-00001-of-00002.safetensors'))
    save_file({k: sd[k] for k in keys[len(keys) // 2:]}, str(plain / 'model-00002-of-00002.safetensors'))
    p = prompts(79, 1, 70, 200)[0].to(DEV)
    want = _verify_logits(direct, p)
    for d in ('hf', 'plain'):
        loaded = BloomForCausalLM.from_pretrained(str(tmp_path / d), device=torch.device(DEV))
        assert (loaded.lm_head.weight is loaded.transformer.word_embeddings.weight) == tie
        assert torch.equal(_verify_logits(loaded, p), want), d


def test_fused_attention_and_fp8_are_refused(monkeypatch, tmp_path):
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import BloomForCausalLM
    model, hf = tiny_model(64, seed=4)
    monkeypatch.setenv('PIA_ATTN_FUSED', '1')
    with pytest.raises(ValueError, match='PIA_ATTN_FUSED'):
        model.generate(input_ids=prompts(6, 1, 16, 200)[0].to(DEV), max_new_tokens=8, eos_token_id=2,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert model._rt is None
    monkeypatch.delenv('PIA_ATTN_FUSED')
    with pytest.raises(NotImplementedError):
        model.quantize_fp8()
    hf.save_pretrained(str(tmp_path))
    with pytest.raises(NotImplementedError, match='fp8'):
        BloomForCausalLM.from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')


# ---------------------------------------------------------------------------------------------------------------
# the real shape: BLOOM-7b1 (30 layers, 4096, 32 heads of 128, V = 250 880)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.big
def test_bloom_7b1_shape_loop_is_exact():
    """the benchmark's synthetic weights, the oracle loop drives one copy, the fused device loop the other; 64-token /
    8-branch drafts, 256-token phrase-bank prompts, two passes: tokens, dls, edls identical"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from scripts.bench_bloom import bloom_7b1_config, synth_fill_bloom
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import BloomForCausalLM
    cfg = bloom_7b1_config()
    a = synth_fill_bloom(BloomForCausalLM(cfg, device=torch.device(DEV)))
    b = BloomForCausalLM(cfg, device=torch.device(DEV))
    b.load_state_dict(a.state_dict(), strict=True)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=cfg.vocab_size)
    otrie = OracleLookaheadCache(eos_ids=[2])
    new = 96
    edl_all = []
    for rep in range(2):
        for p in bench.phrase_bank_prompts(2, cfg.vocab_size):
            p = torch.tensor([p], device=DEV)
            out = a.generate(input_ids=p, max_new_tokens=new, eos_token_id=2,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=new, eos_token_id=[2],
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=256 + new + 65))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), rep
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], rep
            if rep == 1:
                edl_all += ref['edls'][1:]
    assert max(edl_all) > 2
