# -*- coding: utf-8 -*-
"""GLM-family models on the H100: k_rope_kv_append's interleaved (GLM) instance bit for bit against a torch bf16
restatement of transformers' glm apply_rotary_pos_emb, and the tiny GLM / GLM-4-0414 models (tests/tiny_glm.py)
through the verify forward, the loop, sampling, checkpoint loading in the three formats (glm, glm4, THUDM chatglm) and
fp8 weights.  `big`: the ChatGLM3-6B and GLM-4-9B shapes through the loop."""
import json

import numpy as np
import pytest
import torch

from tests.test_gpu_fp8 import OursBackend128, _same_bytes
from tests.test_gpu_generate import OursBackend
from tests.test_gpu_head_dim64 import _mask, _tree
from tests.test_gpu_kernels import _slots
from tests.tiny_glm import glm_hf_model, glm_model_class, thudm_config, thudm_state_dict
from tests.tiny_models import prompts

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


# ---------------------------------------------------------------------------------------------------------------
# the kernel: pia_rope_interleaved_kv_append
# ---------------------------------------------------------------------------------------------------------------
def _tables(max_pos, rd, theta=10000.0):
    inv = 1.0 / (theta ** (torch.arange(0, rd, 2, device=DEV).float() / rd))
    ang = torch.arange(max_pos, device=DEV).float()[:, None] * inv[None]
    return ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()


def _hf_rope(x, cos, sin, pos, rd):
    """transformers' glm apply_rotary_pos_emb in bf16: x [n, H, D], tables [max_pos, rd / 2], positions [n]"""
    c = cos[pos].repeat_interleave(2, dim=-1)[:, None, :]
    s = sin[pos].repeat_interleave(2, dim=-1)[:, None, :]
    xr, xp = x[..., :rd], x[..., rd:]
    rot = torch.stack((-xr[..., 1::2], xr[..., 0::2]), dim=-1).flatten(-2)
    return torch.cat([(xr * c) + (rot * s), xp], dim=-1)


def _run_and_check(Hq, Hkv, D, rd, rps, cases, stride_slots, max_pos=None, seed=0):
    """cases: per table slot (tree rows | n, P, pad); stride_slots: one cache per slot (True) or all slots appending
    into one cache (prefill chunks).  Checks q, the appended K / V rows and that nothing else was written"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(seed)
    B = len(cases)
    R = rps * B
    W = max(1, rps // 64)
    max_seq = max(P + len(rows) for rows, P, _ in cases) + 40
    max_pos = max_pos or max_seq + 8
    n_slots = B if stride_slots else 1
    kc = torch.full((n_slots, Hkv, max_seq, D), 7.0, dtype=torch.bfloat16, device=DEV)
    vc = torch.full_like(kc, 7.0)
    qkv = (torch.randn((R, (Hq + 2 * Hkv) * D), device=DEV) * 2).to(torch.bfloat16)
    q = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    cos, sin = _tables(max_pos, rd)
    mask = _mask([rows for rows, _, _ in cases], 64 * W, rps)
    sl = _slots([len(r) for r, _, _ in cases], [P for _, P, _ in cases], [pad for _, _, pad in cases], rps,
                stride=Hkv * max_seq * D if stride_slots else 0)
    ops.rope_kv_append(qkv, mask, sl, Hq, Hkv, D, cos, sin, q, kc[0], vc[0], max_seq, rotary_dim=rd)
    torch.cuda.synchronize()
    k_want, v_want = torch.full_like(kc, 7.0), torch.full_like(vc, 7.0)
    q_want = torch.full_like(q, 9.0)
    for s_, (rows, P, pad) in enumerate(cases):
        n = len(rows)
        if not n:
            continue
        r0 = s_ * rps
        depth = torch.tensor([bin(r).count('1') - 1 for r in rows], device=DEV)
        pos = (max(P - pad, 0) + depth).clamp(0, max_pos - 1)
        x = qkv[r0:r0 + n].view(n, Hq + 2 * Hkv, D)
        q_want[r0:r0 + n] = _hf_rope(x[:, :Hq], cos, sin, pos, rd)
        c = s_ if stride_slots else 0
        k_want[c, :, P:P + n] = _hf_rope(x[:, Hq:Hq + Hkv], cos, sin, pos, rd).transpose(0, 1)
        v_want[c, :, P:P + n] = x[:, Hq + Hkv:].transpose(0, 1)
        # the dims past rotary_dim are the projection's values, untouched
        assert torch.equal(q[r0:r0 + n, :, rd:], x[:, :Hq, rd:])
    assert torch.equal(q, q_want)
    assert torch.equal(kc, k_want) and torch.equal(vc, v_want)


@pytest.mark.parametrize('Hq,Hkv,D,rd', [(32, 2, 128, 64), (16, 2, 128, 64), (6, 2, 64, 32), (48, 8, 128, 64),
                                         (8, 2, 128, 128), (8, 2, 128, 8), (4, 4, 64, 64)])
@pytest.mark.parametrize('n,P,pad', [(64, 384, 0), (33, 1000, 5), (1, 0, 0), (17, 3, 9)])
def test_rope_interleaved_bit_exact(Hq, Hkv, D, rd, n, P, pad):
    """one slot, a random tree: q and the appended K rows equal HF's apply_rotary_pos_emb in bf16 bit for bit at
    positions rowsum(mask) - 1 (left padding taken off the prefix); V rows are copied"""
    rng = np.random.default_rng(n + P + Hq + rd)
    _run_and_check(Hq, Hkv, D, rd, 64, [(_tree(rng, n), P, pad)], True, seed=n + P)


@pytest.mark.parametrize('D,rd', [(128, 64), (64, 32)])
def test_rope_interleaved_128_node_drafts(D, rd):
    """mask_words 2: 128-node drafts, depth counted over both words"""
    rng = np.random.default_rng(D)
    _run_and_check(16, 2, D, rd, 128, [(_tree(rng, 128, max_depth=100), 700, 0)], True, seed=3)
    _run_and_check(6, 2, D, rd, 128, [(_tree(rng, 97, max_depth=12), 33, 4)], True, seed=4)


@pytest.mark.parametrize('D,rd', [(128, 64), (64, 32)])
def test_rope_interleaved_several_slots(D, rd):
    """one launch over request slots with their own caches, ragged drafts and one empty slot"""
    rng = np.random.default_rng(D + 1)
    cases = [(_tree(rng, 16), 100, 0), (_tree(rng, 5), 0, 0), ([], 7, 0), (_tree(rng, 9), 257, 3)]
    _run_and_check(16, 2, D, rd, 16, cases, True, seed=5)


@pytest.mark.parametrize('D,rd', [(128, 64), (64, 32)])
def test_rope_interleaved_prefill_chunks_share_one_cache(D, rd):
    """a prefill pass: 64-row chain chunks, one table slot each, appending into one cache one after the other"""
    chain = [(1 << (i + 1)) - 1 for i in range(64)]
    base = 40
    cases = [(chain, base, 0), (chain, base + 64, 0), (chain[:23], base + 128, 0)]
    _run_and_check(16, 2, D, rd, 64, cases, False, seed=6)


def test_rope_interleaved_position_clamp():
    """positions past the table are clamped to its last row, as the half-split instance does"""
    rng = np.random.default_rng(8)
    _run_and_check(6, 2, 64, 32, 64, [(_tree(rng, 40), 300, 0)], True, max_pos=310, seed=8)


@pytest.mark.parametrize('rd', [0, 12, 136, -8, 4])
def test_bad_rotary_dim_refused_without_launch(rd):
    from painlessinferenceacceleration_b200.common import ops
    D, Hq, Hkv = 128, 4, 2
    qkv = torch.zeros((64, (Hq + 2 * Hkv) * D), dtype=torch.bfloat16, device=DEV)
    q = torch.zeros((64, Hq, D), dtype=torch.bfloat16, device=DEV)
    kc = torch.zeros((Hkv, 256, D), dtype=torch.bfloat16, device=DEV)
    mask = torch.ones((64, 1), dtype=torch.int64, device=DEV)
    cos, sin = _tables(256, 64)
    l0 = ops.launch_count()
    with pytest.raises(AssertionError, match='rotary_dim'):
        ops.rope_kv_append(qkv, mask, _slots([1], [0], [0], 64), Hq, Hkv, D, cos, sin, q, kc, kc.clone(), 256,
                           rotary_dim=rd)
    assert ops.launch_count() == l0


def test_half_split_entry_point_unchanged_by_rotary_dim_none():
    """rotary_dim=None keeps pia_rope_kv_append: Llama RoPE over the whole head"""
    from painlessinferenceacceleration_b200.common import ops
    D, Hq, Hkv, n, P = 128, 4, 2, 10, 50
    torch.manual_seed(9)
    qkv = torch.randn((64, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    q = torch.zeros((64, Hq, D), dtype=torch.bfloat16, device=DEV)
    kc = torch.zeros((Hkv, 256, D), dtype=torch.bfloat16, device=DEV)
    vc = kc.clone()
    cos, sin = _tables(256, D)
    rows = [(1 << (i + 1)) - 1 for i in range(n)]
    ops.rope_kv_append(qkv, _mask([rows], 64, 64), _slots([n], [P], [0], 64), Hq, Hkv, D, cos, sin, q, kc, vc, 256)
    torch.cuda.synchronize()
    pos = P + torch.arange(n, device=DEV)
    x = qkv[:n].view(n, -1, D)[:, :Hq]
    c = torch.cat([cos[pos], cos[pos]], -1)[:, None]
    s = torch.cat([sin[pos], sin[pos]], -1)[:, None]
    want = (x * c) + (torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1) * s)
    assert torch.equal(q[:n], want)


# ---------------------------------------------------------------------------------------------------------------
# the tiny models
# ---------------------------------------------------------------------------------------------------------------
MODELS = [('glm', 128), ('glm', 64), ('glm4', 128)]


def _pair(kind, hd, seed, **over):
    hf = glm_hf_model(kind, hd, seed=seed, dtype=torch.bfloat16, device=DEV, vocab=200, **over)
    return hf, _ours(kind, hf)


def _ours(kind, hf):
    m = glm_model_class(kind)(hf.config, device=torch.device(DEV))
    res = m.load_state_dict(hf.state_dict(), strict=False)
    assert not res.missing_keys, res
    return m


def _verify_logits(model, p):
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    return OursBackend(model).forward(p, m01, None)[0].float()


def _check_against_fp32(kind, hd, seed, hf, got, p, sd=None):
    """max |error| <= 2 x the eager bf16 HF model's own error + 0.02, same greedy tokens where the fp32 margin is clear.
    sd: evaluate these fp32 weights instead of hf's (the dequantised fp8 weights)"""
    sd = sd if sd is not None else {k: v.float() for k, v in hf.state_dict().items()}
    hf32 = glm_hf_model(kind, hd, seed=seed, dtype=torch.float32, device=DEV, vocab=200)
    hf32.load_state_dict(sd)
    eager_m = glm_hf_model(kind, hd, seed=seed, dtype=torch.bfloat16, device=DEV, vocab=200)
    eager_m.load_state_dict({k: v.to(torch.bfloat16) for k, v in sd.items()})
    with torch.no_grad():
        truth = hf32(input_ids=p).logits[0].float()
        eager = eager_m(input_ids=p).logits[0].float()
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)
    top = torch.topk(truth, 2, dim=-1).values
    sure = (top[:, 0] - top[:, 1]) > 2 * e_ours
    assert torch.equal(got.argmax(-1)[sure], truth.argmax(-1)[sure])


@pytest.mark.parametrize('kind,hd', MODELS)
def test_glm_verify_logits_within_tolerance(kind, hd):
    hf, ours = _pair(kind, hd, seed=8)
    assert float(hf.model.layers[0].self_attn.k_proj.bias.detach().float().abs().max()) > 1.0
    p = prompts(77, 1, 100, 200)[0].to(DEV)
    _check_against_fp32(kind, hd, 8, hf, _verify_logits(ours, p), p)


def test_glm4_sandwich_norms_matter_and_work_on_split_k_slices(monkeypatch):
    """the glm4 model without its post norms is far off; with the o / down projections on the weight-streaming GEMM
    returning fp32 split-K slices (the post norms then read the slices) the logits stay within tolerance"""
    hf, ours = _pair('glm4', 128, seed=12)
    p = prompts(78, 1, 60, 200)[0].to(DEV)
    base = _verify_logits(ours, p)
    _check_against_fp32('glm4', 128, 12, hf, base, p)
    plain = glm_model_class('glm')(hf.config, device=torch.device(DEV))
    plain.load_state_dict(hf.state_dict(), strict=False)
    assert (_verify_logits(plain, p) - base).abs().max().item() > 1.0
    monkeypatch.setenv('PIA_GEMM_SET', 'gate_up,o,down')
    monkeypatch.setenv('PIA_GEMM_SPLIT', '4')
    split = _ours('glm4', hf)
    got = _verify_logits(split, p)
    lp = split._rt.gemm_plans['layers'][0]
    assert lp['o'].splits == 4 and lp['down'].splits == 4
    _check_against_fp32('glm4', 128, 12, hf, got, p)


@pytest.mark.parametrize('kind,hd,penalty,dl', [('glm', 128, 1.0, 64), ('glm', 128, 1.1, 128), ('glm', 64, 1.1, 64),
                                                ('glm', 64, 1.0, 128), ('glm4', 128, 1.1, 64), ('glm4', 128, 1.0, 128)])
def test_glm_loop_is_exact_given_the_same_logits(kind, hd, penalty, dl):
    """the oracle loop drives one copy of our model through the backend interface, the fused device loop another copy
    with the same weights: tokens, dls and edls identical for every request, tries carried across requests"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, a = _pair(kind, hd, seed=6)
    b = _ours(kind, hf)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    backend = OursBackend128 if dl == 128 else OursBackend
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 3, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=56, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': dl, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=56, eos_token_id=[2], repetition_penalty=penalty,
                                     decoding_length=dl,
                                     backend=backend(b, prefill_like_generate=True, max_seq=90 + 56 + 2 * dl + 1))
            assert a._rt.max_nodes == dl
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (kind, hd, dl, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (kind, hd, dl, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


@pytest.mark.parametrize('kind,hd', [('glm', 64), ('glm4', 128)])
def test_glm_do_sample(kind, hd):
    """multinomial accept: well-formed output, and sampling really departs from greedy decoding somewhere"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, ours = _pair(kind, hd, seed=3)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    torch.manual_seed(11)
    differs = 0
    for p in prompts(9, 3, 24, 200):
        p = p.to(DEV)
        g = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
        o = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, do_sample=True, return_dict_in_generate=True,
                          decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
        seq = o.sequences[0].tolist()
        assert seq[:24] == p[0].tolist() and len(seq) <= 24 + 40
        assert sum(o.kwargs['edls']) == len(seq) - 24
        assert all(0 <= t < 200 for t in seq)
        differs += seq != g[0].tolist()
    assert differs >= 1


def _write_thudm(hf, path, per_head_dim=None, **cfg_over):
    from safetensors.torch import save_file
    path.mkdir(parents=True, exist_ok=True)
    (path / 'config.json').write_text(json.dumps(thudm_config(hf.config, **cfg_over)))
    sd = {k: v.detach().cpu().contiguous()
          for k, v in thudm_state_dict(hf.state_dict(), per_head_dim=per_head_dim).items()}
    half = len(sd) // 2   # two shards
    keys = sorted(sd)
    save_file({k: sd[k] for k in keys[:half]}, str(path / 'model-00001-of-00002.safetensors'))
    save_file({k: sd[k] for k in keys[half:]}, str(path / 'model-00002-of-00002.safetensors'))


@pytest.mark.parametrize('kind,hd', MODELS)
def test_glm_from_pretrained(tmp_path, kind, hd):
    """a save_pretrained directory loads into the logits of the weights handed over directly; for `glm`, a THUDM-layout
    directory of the same weights (model_type chatglm, fused query_key_value, an inv_freq tensor) gives identical
    logits through ChatGLMForConditionalGeneration; then generate() runs on the loaded model"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    hf, direct = _pair(kind, hd, seed=10)
    hf.save_pretrained(str(tmp_path / 'hf'))
    loaded = glm_model_class(kind).from_pretrained(str(tmp_path / 'hf'), device=torch.device(DEV))
    p = prompts(79, 1, 70, 200)[0].to(DEV)
    want = _verify_logits(direct, p)
    assert torch.equal(_verify_logits(loaded, p), want)
    if kind == 'glm':
        _write_thudm(hf, tmp_path / 'thudm')
        cg = ChatGLMForConditionalGeneration.from_pretrained(str(tmp_path / 'thudm'), device=torch.device(DEV))
        assert cg.geometry() == loaded.geometry()
        assert torch.equal(cg.rope_tables(512)[0], loaded.rope_tables(512)[0])
        assert torch.equal(_verify_logits(cg, p), want)
        loaded = cg
    loaded.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    out = loaded.generate(input_ids=p, max_new_tokens=24, eos_token_id=2, return_dict_in_generate=True,
                          decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert sum(out.kwargs['edls']) == out.sequences.shape[1] - 70


def test_chatglm_without_multi_query_from_pretrained(tmp_path):
    """multi_query_attention=False (every head its own K / V, query_key_value rows per head [q_h; k_h; v_h]): the
    THUDM directory gives logits identical to the HF-format load of the same weights"""
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    hf, direct = _pair('glm', 64, seed=13, num_key_value_heads=6)
    _write_thudm(hf, tmp_path, per_head_dim=64, multi_query_attention=False)
    cg = ChatGLMForConditionalGeneration.from_pretrained(str(tmp_path), device=torch.device(DEV))
    assert cg.geometry()['n_kv_heads'] == 6
    p = prompts(82, 1, 70, 200)[0].to(DEV)
    assert torch.equal(_verify_logits(cg, p), _verify_logits(direct, p))


@pytest.mark.parametrize('kind,hd,dl', [('glm', 128, 64), ('glm', 64, 128), ('glm4', 128, 64)])
def test_glm_fp8_loop_is_exact_given_the_same_logits(kind, hd, dl):
    """quantize_fp8() (the q/k/v bias through the fp8 GEMM's bias epilogue, the fused gate_up_proj as the SiLU*up
    operand); the oracle loop drives one fp8 copy, the fused device loop another with identical bytes: tokens, dls and
    edls identical"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, a = _pair(kind, hd, seed=6)
    a.quantize_fp8()
    b = _ours(kind, hf).quantize_fp8()
    _same_bytes(a, b)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    backend = OursBackend128 if dl == 128 else OursBackend
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 3, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=48, eos_token_id=2,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': dl, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=48, eos_token_id=[2], decoding_length=dl,
                                     backend=backend(b, prefill_like_generate=True, max_seq=90 + 48 + 2 * dl + 1))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (kind, dl, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (kind, dl, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def _dequantised_state(hf, ours):
    """HF state dict whose projections are ours' dequantised fp8 weights (fp32)"""
    sd = {k: v.float() for k, v in hf.state_dict().items()}
    for i, layer in enumerate(ours.model.layers):
        pre = f'model.layers.{i}.'
        for n in ('q_proj', 'k_proj', 'v_proj', 'o_proj'):
            sd[pre + f'self_attn.{n}.weight'] = getattr(layer.self_attn, n).dequantize()
        for n in ('gate_up_proj', 'down_proj'):
            sd[pre + f'mlp.{n}.weight'] = getattr(layer.mlp, n).dequantize()
    return sd


@pytest.mark.parametrize('kind,hd', MODELS)
def test_glm_fp8_verify_logits_within_tolerance(kind, hd):
    """fp8 verify logits (bias epilogue, fused gate_up_proj as the SiLU*up operand) vs an fp32 evaluation of the
    dequantised weights, with the rule of the bf16 test"""
    hf, ours = _pair(kind, hd, seed=8)
    ours.quantize_fp8()
    assert type(ours.model.layers[0].mlp.gate_up_proj).__name__ == 'Fp8Rows'
    p = prompts(77, 1, 100, 200)[0].to(DEV)
    _check_against_fp32(kind, hd, 8, hf, _verify_logits(ours, p), p, sd=_dequantised_state(hf, ours))


@pytest.mark.parametrize('fmt', ['glm', 'glm4', 'chatglm'])
def test_glm_fp8_from_pretrained(tmp_path, fmt):
    """from_pretrained(..., quantization='fp8') gives quantize_fp8()'s bytes in all three formats and runs generate()"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    kind = 'glm4' if fmt == 'glm4' else 'glm'
    hf, ref = _pair(kind, 128, seed=12)
    ref.quantize_fp8()
    if fmt == 'chatglm':
        _write_thudm(hf, tmp_path)
        got = ChatGLMForConditionalGeneration.from_pretrained(str(tmp_path), device=torch.device(DEV),
                                                              quantization='fp8')
    else:
        hf.save_pretrained(str(tmp_path))
        got = glm_model_class(kind).from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')
    _same_bytes(ref, got)
    got.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    p = prompts(80, 1, 40, 200)[0].to(DEV)
    out = got.generate(input_ids=p, max_new_tokens=24, eos_token_id=2, return_dict_in_generate=True,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert sum(out.kwargs['edls']) == out.sequences.shape[1] - 40


def test_glm_fused_attention_knob_is_refused(monkeypatch):
    """PIA_ATTN_FUSED=1: ValueError before a runtime or graph exists, no silent two-kernel path"""
    hf, ours = _pair('glm', 64, seed=4)
    monkeypatch.setenv('PIA_ATTN_FUSED', '1')
    with pytest.raises(ValueError, match='PIA_ATTN_FUSED'):
        ours.generate(input_ids=prompts(6, 1, 16, 200)[0].to(DEV), max_new_tokens=8, eos_token_id=2,
                      decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert ours._rt is None


# ---------------------------------------------------------------------------------------------------------------
# the real shapes: ChatGLM3-6B (28 layers, 4096 / 13696, 32 / 2 heads, V = 65024) and GLM-4-9B (40 layers, V = 151552)
# ---------------------------------------------------------------------------------------------------------------
def chatglm3_6b_shape():
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    return ChatGLMForConditionalGeneration, ChatGLMForConditionalGeneration.chatglm_config(dict(
        model_type='chatglm', add_bias_linear=False, add_qkv_bias=True, apply_query_key_layer_scaling=True,
        apply_residual_connection_post_layernorm=False, ffn_hidden_size=13696, hidden_size=4096, kv_channels=128,
        layernorm_epsilon=1e-05, multi_query_attention=True, multi_query_group_num=2, num_attention_heads=32,
        num_layers=28, original_rope=True, padded_vocab_size=65024, post_layer_norm=True, rmsnorm=True,
        seq_length=8192, eos_token_id=2, pad_token_id=0))


def glm4_9b_shape():
    from transformers import GlmConfig
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    return GlmForCausalLM, GlmConfig(vocab_size=151552, hidden_size=4096, intermediate_size=13696, num_hidden_layers=40,
                                     num_attention_heads=32, num_key_value_heads=2, head_dim=128,
                                     max_position_embeddings=8192, rms_norm_eps=1.5625e-07, attention_bias=True,
                                     tie_word_embeddings=False, bos_token_id=1, eos_token_id=2, pad_token_id=0)


@pytest.mark.big
@pytest.mark.parametrize('shape', ['chatglm3-6b', 'glm-4-9b'])
def test_glm_shapes_loop_is_exact(shape):
    """as test_head_dim64_shapes_loop_is_exact: bench.synth_fill weights, the oracle loop drives one copy, the fused
    device loop the other; 64-token / 8-branch drafts, 256-token phrase-bank prompts, two passes.  Tokens, dls and
    edls identical, and the second pass accepts drafts longer than 2"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    cls, cfg = chatglm3_6b_shape() if shape.startswith('chatglm') else glm4_9b_shape()
    a = bench.synth_fill(cls(cfg, device=torch.device(DEV)), cfg)
    b = cls(cfg, device=torch.device(DEV))
    b.load_state_dict(a.state_dict(), strict=True)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=cfg.vocab_size)
    otrie = OracleLookaheadCache(eos_ids=[2])
    new = 96
    edl_all = []
    for rep in range(2):
        for p in bench.phrase_bank_prompts(3, cfg.vocab_size):
            p = torch.tensor([p], device=DEV)
            out = a.generate(input_ids=p, max_new_tokens=new, eos_token_id=2, repetition_penalty=1.0,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=new, eos_token_id=[2],
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=256 + new + 65))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), rep
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], rep
            if rep == 1:
                edl_all += ref['edls'][1:]
    assert max(edl_all) > 2, 'the second pass never accepted a draft: the test did not exercise the accept path'
