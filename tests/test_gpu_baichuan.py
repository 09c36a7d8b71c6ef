# -*- coding: utf-8 -*-
"""Baichuan family on the H100: k_tree_attn's ALiBi instance against an fp32 restatement with explicit tree positions,
k_rope_kv_append's fp32 instance bit for bit against torch's Baichuan2 formula, the lossless property of the ALiBi /
fp32-RoPE verify forward (every draft node's logits = a causal forward over prefix + root-to-node path), and the tiny
models (tests/tiny_baichuan.py) through generate(), the oracle loop, checkpoint loading and fp8.  `big`: the
Baichuan-13B and Baichuan2-7B shapes through the loop."""
import json

import numpy as np
import pytest
import torch
from torch.nn import functional as F

from tests import attn_ref
from tests.test_gpu_fp8 import _same_bytes
from tests.test_gpu_generate import OursBackend
from tests.test_gpu_head_dim64 import _mask, _tree
from tests.test_gpu_kernels import _slots
from tests.tiny_baichuan import causal_logits, model_class, ref_forward, slopes_f64, tiny_config, tiny_model, \
    w_pack_state_dict
from tests.tiny_models import prompts

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
D = 128


# ---------------------------------------------------------------------------------------------------------------
# the kernel: pia_tree_attn_alibi_fwd
# ---------------------------------------------------------------------------------------------------------------
def _ref_alibi(q, kc, vc, rows, n, P, pad, G, slopes):
    """exact (fp64) restatement: row i (tree depth t_i = popc(rows[i]) - 1) at qpos = max(P - pad, 0) + t_i; cached
    key j in [pad, P) at kpos = j - pad, draft key k (an ancestor of i, or i) at max(P - pad, 0) + t_k; score =
    q.k / sqrt(D) + slope_h * (kpos - qpos) (tests/attn_ref.py)"""
    return attn_ref.reference(q, kc, vc, rows, n, P, pad, G, slopes=slopes)


def _slopes(H):
    return torch.tensor(slopes_f64(H), dtype=torch.float64).to(torch.float32).to(DEV)


def _cases():
    out = [(hq, hkv, P, n, 64) for hq, hkv in ((40, 40), (5, 5), (8, 2), (6, 1)) for P in (0, 129, 1000, 3968)
           for n in (1, 33, 64)]
    out += [(hq, hkv, P, n, 128) for hq, hkv in ((5, 5), (8, 2)) for P in (0, 200, 3968) for n in (65, 128)]
    return out


@pytest.mark.parametrize('Hq,Hkv,P,n,R', _cases())
def test_alibi_tree_attention(Hq, Hkv, P, n, R):
    """one slot, a random tree, left padding (P % 7 columns): against the fp32 restatement with the tolerance of the
    other attention tests; rows beyond the draft untouched; the plain instance on the same plan is unchanged"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(P + n + Hq + R)
    torch.manual_seed(P * 7 + n + Hq)
    pad = P % 7 if P > 8 else 0
    max_seq = P + n + 70
    kc = (torch.randn((2, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((2, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    q = (torch.randn((R, Hq, D), device=DEV) * 0.7).to(torch.bfloat16)
    rows = _tree(rng, n, max_depth=12)
    mask = _mask([rows], R, R)
    plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
    slopes = _slopes(Hq)
    out = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    for layer in (1, 0):
        out.fill_(9.0)
        plan.forward(layer, q, mask, _slots([n], [P], [pad], R), out, alibi_slopes=slopes)
        torch.cuda.synchronize()
        ref = _ref_alibi(q, kc[layer], vc[layer], rows, n, P, pad, Hq // Hkv, slopes)
        err = (out[:n].float() - ref).abs().max().item()
        attn_ref.assert_close(out[:n].float(), ref, f'layer {layer} max abs err {err}')
        assert float((out[n:].float() - 9.0).abs().sum()) == 0


def test_alibi_bias_is_not_a_no_op():
    """steep slopes: the ALiBi output is far from the plain instance's, and close to the restatement"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(1)
    Hq, P, n, R = 4, 300, 40, 64
    kc = (torch.randn((1, Hq, P + n + 8, D), device=DEV)).to(torch.bfloat16)
    vc = (torch.randn((1, Hq, P + n + 8, D), device=DEV)).to(torch.bfloat16)
    q = (torch.randn((R, Hq, D), device=DEV)).to(torch.bfloat16)
    rows = _tree(np.random.default_rng(2), n)
    mask = _mask([rows], R, R)
    plan = ops.AttnPlan(kc, vc, Hq, Hq, D, R)
    slopes = torch.tensor([0.5, 0.25, 0.125, 0.0], device=DEV)
    a, b = torch.zeros((R, Hq, D), dtype=torch.bfloat16, device=DEV), torch.zeros((R, Hq, D), dtype=torch.bfloat16,
                                                                                   device=DEV)
    plan.forward(0, q, mask, _slots([n], [P], [0], R), a, alibi_slopes=slopes)
    plan.forward(0, q, mask, _slots([n], [P], [0], R), b)
    torch.cuda.synchronize()
    assert (a[:n, 0].float() - b[:n, 0].float()).abs().max().item() > 0.3
    assert torch.equal(a[:n, 3], b[:n, 3])   # slope 0: the plain arithmetic
    ref = _ref_alibi(q, kc[0], vc[0], rows, n, P, 0, 1, slopes)
    attn_ref.assert_close(a[:n].float(), ref)


@pytest.mark.parametrize('R,rps', [(64, 16), (128, 32)])
def test_alibi_several_slots(R, rps):
    """one launch over request slots with their own caches: ragged drafts, left padding, one idle slot"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(R)
    rng = np.random.default_rng(R)
    Hq, Hkv = 8, 2
    cases = [(_tree(rng, rps), 700, 3), (_tree(rng, 5), 0, 0), ([], 7, 0), (_tree(rng, 9), 2100, 0)]
    B = len(cases)
    max_seq = 2100 + rps + 40
    kc = (torch.randn((B, 1, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((B, 1, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    q = (torch.randn((B * rps, Hq, D), device=DEV) * 0.7).to(torch.bfloat16)
    mask = _mask([r for r, _, _ in cases], R, rps)
    plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
    sl = _slots([len(r) for r, _, _ in cases], [P for _, P, _ in cases], [p for _, _, p in cases], rps,
                stride=plan.slot_stride)
    slopes = _slopes(Hq)
    out = torch.full((B * rps, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    plan.forward(0, q, mask, sl, out, alibi_slopes=slopes)
    torch.cuda.synchronize()
    for s_, (rows, P, pad) in enumerate(cases):
        n, r0 = len(rows), s_ * rps
        assert float((out[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0
        if n:
            ref = _ref_alibi(q[r0:], kc[s_, 0], vc[s_, 0], rows, n, P, pad, Hq // Hkv, slopes)
            attn_ref.assert_close(out[r0:r0 + n].float(), ref, s_)


def test_alibi_head_dim64_is_unsupported():
    from painlessinferenceacceleration_b200 import _lib
    from painlessinferenceacceleration_b200.common import ops
    kc = torch.zeros((1, 2, 256, 64), dtype=torch.bfloat16, device=DEV)
    plan = ops.AttnPlan(kc, kc.clone(), 2, 2, 64, 64)
    q = torch.zeros((64, 2, 64), dtype=torch.bfloat16, device=DEV)
    mask = torch.ones((64, 1), dtype=torch.int64, device=DEV)
    l0 = ops.launch_count()
    with pytest.raises(_lib.PiaError, match='-5'):
        plan.forward(0, q, mask, _slots([1], [10], [0], 64), q.clone(), alibi_slopes=_slopes(2))
    assert ops.launch_count() == l0


# ---------------------------------------------------------------------------------------------------------------
# the kernel: pia_rope_f32_kv_append
# ---------------------------------------------------------------------------------------------------------------
def _f32_tables(max_pos):
    inv = 1.0 / (10000 ** (torch.arange(0, D, 2).float() / D))
    ang = torch.outer(torch.arange(max_pos, dtype=torch.float32), inv)
    return ang.cos().to(DEV).contiguous(), ang.sin().to(DEV).contiguous()


def _baichuan2_rope(x, cos, sin, pos):
    """baichuan2_7b apply_rotary_pos_emb: x.float() * cos + rotate_half(x.float()) * sin, then one cast to bf16"""
    c = torch.cat([cos[pos], cos[pos]], -1)[:, None, :]
    s = torch.cat([sin[pos], sin[pos]], -1)[:, None, :]
    xf = x.float()
    rot = torch.cat([-xf[..., D // 2:], xf[..., :D // 2]], -1)
    return ((xf * c) + (rot * s)).to(torch.bfloat16)


@pytest.mark.parametrize('Hq,Hkv,n,P,pad,R', [(32, 32, 64, 384, 0, 64), (4, 4, 33, 1000, 5, 64), (8, 2, 1, 0, 0, 64),
                                              (4, 4, 128, 700, 3, 128), (40, 40, 17, 3, 9, 64)])
def test_rope_f32_bit_exact(Hq, Hkv, n, P, pad, R):
    """q and the appended K rows bit for bit against torch's Baichuan2 formula at the tree positions; V copied; only
    the new cache rows written"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(n + P)
    torch.manual_seed(n + P)
    rows = _tree(rng, n, max_depth=30)
    max_seq = P + n + 40
    cos, sin = _f32_tables(max_seq + 8)
    kc = torch.full((Hkv, max_seq, D), 7.0, dtype=torch.bfloat16, device=DEV)
    vc = torch.full_like(kc, 7.0)
    qkv = (torch.randn((R, (Hq + 2 * Hkv) * D), device=DEV) * 2).to(torch.bfloat16)
    q = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    ops.rope_kv_append(qkv, _mask([rows], R, R), _slots([n], [P], [pad], R), Hq, Hkv, D, cos, sin, q, kc, vc, max_seq)
    torch.cuda.synchronize()
    depth = torch.tensor([bin(r).count('1') - 1 for r in rows], device=DEV)
    pos = max(P - pad, 0) + depth
    x = qkv[:n].view(n, Hq + 2 * Hkv, D)
    q_want = torch.full_like(q, 9.0)
    q_want[:n] = _baichuan2_rope(x[:, :Hq], cos, sin, pos)
    k_want, v_want = torch.full_like(kc, 7.0), torch.full_like(vc, 7.0)
    k_want[:, P:P + n] = _baichuan2_rope(x[:, Hq:Hq + Hkv], cos, sin, pos).transpose(0, 1)
    v_want[:, P:P + n] = x[:, Hq + Hkv:].transpose(0, 1)
    assert torch.equal(q, q_want)
    assert torch.equal(kc, k_want) and torch.equal(vc, v_want)
    if int(pos.max()) == 0:   # cos 1, sin 0: every arithmetic gives x
        return
    # and it is not the bf16 instance's arithmetic
    q2 = torch.full_like(q, 9.0)
    ops.rope_kv_append(qkv, _mask([rows], R, R), _slots([n], [P], [pad], R), Hq, Hkv, D, cos.to(torch.bfloat16),
                       sin.to(torch.bfloat16), q2, kc.clone(), vc.clone(), max_seq)
    torch.cuda.synchronize()
    assert not torch.equal(q2[:n], q[:n])


# ---------------------------------------------------------------------------------------------------------------
# lossless: the verify logits of every draft node = a causal forward over prefix + root-to-node path
# ---------------------------------------------------------------------------------------------------------------
def _sd(model):
    return {k: v.detach().float() for k, v in model.state_dict().items()}


def _check(got, truth, eager):
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)


@pytest.mark.parametrize('kind', ['13b', '2_13b', '2_7b', '7b'])
def test_tree_verify_logits_are_lossless(kind):
    """a prompt (two chain chunks), then one random 64-node tree: each node's verify-logit row vs the fp32 causal
    forward over prompt + its root-to-node path, within 2 x the bf16 eager restatement's own error + 0.02"""
    model = tiny_model(kind, seed=3)
    cfg = tiny_config(kind)
    sd = _sd(model)
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
        truth = causal_logits(sd, cfg, kind, seq)[-1]
        eager = causal_logits(sd, cfg, kind, seq, dtype=torch.bfloat16)[-1]
        _check(got[i], truth, eager)


@pytest.mark.parametrize('kind', ['13b', '2_7b'])
def test_prefill_with_left_padding_is_lossless(kind):
    """the prefill pass of a left-padded prompt: its last-row logits vs the fp32 causal forward of the unpadded
    prompt (pad columns invisible, positions counted from the first real token)"""
    model = tiny_model(kind, seed=6)
    cfg = tiny_config(kind)
    sd = _sd(model)
    torch.manual_seed(7)
    pad, T = 13, 150
    p = torch.randint(3, 200, (T,), device=DEV)
    rt = model._runtime(512, 64)
    rt.set_request(0, pad, 1 << 30)
    rt.seq[0, :pad] = 0
    rt.seq[0, pad:pad + T] = p.to(torch.int32)
    model._prefill_logits(rt, pad + T)
    got = rt.logits[0].float()
    _check(got, causal_logits(sd, cfg, kind, p)[-1], causal_logits(sd, cfg, kind, p, dtype=torch.bfloat16)[-1])


# ---------------------------------------------------------------------------------------------------------------
# the tiny models
# ---------------------------------------------------------------------------------------------------------------
def _cache(model):
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    model.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    return model


@pytest.mark.parametrize('kind,penalty', [('13b', 1.0), ('13b', 1.1), ('2_7b', 1.0), ('2_7b', 1.1), ('2_13b', 1.0),
                                          ('7b', 1.0)])
def test_generate_equals_plain_greedy(kind, penalty):
    """lookahead generate() (prefill + tree drafts) gives the tokens of plain greedy decoding with the same kernels,
    and a second pass over the same prompts accepts drafts"""
    model = _cache(tiny_model(kind, seed=1))
    edls = []
    for rep in range(2):
        for p in prompts(21, 2, 40, 200):
            p = p.to(DEV)
            g = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               decoding_kwargs={'use_lookahead': False})
            o = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               return_dict_in_generate=True,
                               decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
            assert o.sequences[0].tolist() == g[0].tolist(), (kind, rep)
            edls += o.kwargs['edls'][1:]
    assert max(edls) > 2


@pytest.mark.parametrize('kind', ['13b', '2_7b'])
def test_do_sample(kind):
    model = _cache(tiny_model(kind, seed=2))
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


@pytest.mark.parametrize('kind', ['2_7b', '13b'])
def test_batched_generate_equals_per_request(kind):
    """the batched loop class over a batch of 3 prompts gives the per-request greedy tokens, up to a near-tie of the
    logits (the batched step splits the KV range differently, which moves the fp32 summation order)"""
    single = _cache(tiny_model(kind, seed=5))
    batch = _cache(tiny_model(kind, seed=5, batch=True))
    ps = torch.cat([p for p in prompts(31, 3, 32, 200)]).to(DEV)
    dk = {'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8}
    out = batch.generate(input_ids=ps, max_new_tokens=32, eos_token_id=2, decoding_kwargs=dict(dk))
    out = out.sequences if hasattr(out, 'sequences') else out
    same = 0
    for b in range(3):
        s = single.generate(input_ids=ps[b:b + 1], max_new_tokens=32, eos_token_id=2, decoding_kwargs=dict(dk))[0]
        s = s.tolist()
        bt = out[b].tolist()[:len(s)]
        if bt == s:
            same += 1
            continue
        k = next(j for j in range(min(len(bt), len(s))) if bt[j] != s[j])
        m01 = torch.tril(torch.ones((1, 1, k, k), dtype=torch.long, device=DEV))
        lg = single.forward(torch.tensor([s[:k]], device=DEV), m01)[0][0, -1].float()
        top = torch.topk(lg, 2).values
        assert (top[0] - top[1]).item() < 0.1, (b, k)
    assert same >= 2


@pytest.mark.parametrize('kind,penalty', [('13b', 1.1), ('2_7b', 1.0), ('2_13b', 1.0)])
def test_loop_is_exact_given_the_same_logits(kind, penalty):
    """the oracle loop drives one copy of our model, the fused device loop another: tokens, dls, edls identical"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    a = _cache(tiny_model(kind, seed=6))
    b = tiny_model(kind, seed=6)
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
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (kind, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (kind, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def _write_checkpoint(model, kind, path, unnormalised_head=None):
    """a Baichuan-format directory: config.json (model_max_length / max_position_embeddings as published), W_pack,
    two safetensors shards"""
    from safetensors.torch import save_file
    path.mkdir(parents=True, exist_ok=True)
    (path / 'config.json').write_text(json.dumps(dict(tiny_config(kind), architectures=['BaichuanForCausalLM'])))
    sd = {k: v.detach().cpu().contiguous() for k, v in w_pack_state_dict(model.state_dict()).items()}
    if unnormalised_head is not None:
        sd['lm_head.weight'] = unnormalised_head.cpu().contiguous()
    keys = sorted(sd)
    save_file({k: sd[k] for k in keys[:len(keys) // 2]}, str(path / 'model-00001-of-00002.safetensors'))
    save_file({k: sd[k] for k in keys[len(keys) // 2:]}, str(path / 'model-00002-of-00002.safetensors'))


def _verify_logits(model, p):
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    return OursBackend(model).forward(p, m01, None)[0].float()


@pytest.mark.parametrize('kind', ['13b', '2_7b', '2_13b', '7b'])
def test_from_pretrained_bf16_and_fp8(tmp_path, kind):
    """a Baichuan-format checkpoint loads into the logits of the same weights handed over directly (NormHead applied
    on load to a raw head); quantization='fp8' gives quantize_fp8()'s bytes with a bf16 lm_head, and generate() runs"""
    direct = tiny_model(kind, seed=10)
    raw = direct.lm_head.weight.detach().clone()
    if direct.norm_head:   # the checkpoint holds the un-normalised head (NormHead normalises on the first forward)
        torch.manual_seed(3)
        raw = (torch.randn_like(raw.float()) * 0.3).to(torch.bfloat16)
        with torch.no_grad():
            direct.lm_head.weight.copy_(F.normalize(raw))
    _write_checkpoint(direct, kind, tmp_path, unnormalised_head=raw)
    cls = model_class(kind)
    loaded = cls.from_pretrained(str(tmp_path), device=torch.device(DEV))
    assert torch.equal(loaded.lm_head.weight, direct.lm_head.weight)
    p = prompts(79, 1, 70, 200)[0].to(DEV)
    assert torch.equal(_verify_logits(loaded, p), _verify_logits(direct, p))
    ref = tiny_model(kind, seed=10)
    ref.load_state_dict(direct.state_dict())
    ref.quantize_fp8()
    got = cls.from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')
    _same_bytes(ref, got)
    assert got.lm_head.weight.dtype == torch.bfloat16 and torch.equal(got.lm_head.weight, direct.lm_head.weight)
    _cache(got)
    out = got.generate(input_ids=p, max_new_tokens=24, eos_token_id=2, return_dict_in_generate=True,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert sum(out.kwargs['edls']) == out.sequences.shape[1] - 70


def test_norm_head_rows_are_unit_and_equal_f_normalize():
    """Baichuan2: lm_head rows are unit-norm in bf16 and equal F.normalize of the raw rows, in init_weights and in
    build_fp8; Baichuan-13B keeps its raw head"""
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    m = tiny_model('2_13b', seed=4)
    raw = model_class('13b')(baichuan_config(tiny_config('13b')), device=torch.device(DEV)).init_weights(seed=4,
                                                                                                         std=0.08)
    w = m.lm_head.weight
    assert w.dtype == torch.bfloat16
    assert torch.allclose(w.float().norm(dim=1), torch.ones(w.shape[0], device=DEV), atol=1e-2)
    assert torch.equal(w, F.normalize(raw.lm_head.weight))
    assert not torch.equal(raw.lm_head.weight, w)
    cfg = baichuan_config(tiny_config('2_7b'))
    gen = torch.Generator(device=DEV).manual_seed(0)

    def fill_rest(model):
        for name, p in model.named_parameters():
            if p.device.type != 'meta':
                p.normal_(0.0, 0.08, generator=gen)

    def fill_weight(name, t):
        t.normal_(0.0, 0.08, generator=gen)

    f = model_class('2_7b').build_fp8(cfg, fill_rest, fill_weight, device=torch.device(DEV))
    assert torch.allclose(f.lm_head.weight.float().norm(dim=1), torch.ones(cfg.vocab_size, device=DEV), atol=1e-2)


@pytest.mark.parametrize('kind', ['13b', '2_7b'])
def test_fused_attention_knob_is_refused(monkeypatch, kind):
    model = tiny_model(kind, seed=4)
    monkeypatch.setenv('PIA_ATTN_FUSED', '1')
    with pytest.raises(ValueError, match='PIA_ATTN_FUSED'):
        model.generate(input_ids=prompts(6, 1, 16, 200)[0].to(DEV), max_new_tokens=8, eos_token_id=2,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert model._rt is None


def test_fp8_verify_logits_within_tolerance():
    """fp8 weights (ALiBi model): verify logits vs an fp32 forward of the dequantised weights, the bf16 rule"""
    model = tiny_model('13b', seed=8)
    cfg = tiny_config('13b')
    sd = _sd(model)
    model.quantize_fp8()
    for i, layer in enumerate(model.model.layers):
        pre = f'model.layers.{i}.'
        for n in ('q_proj', 'k_proj', 'v_proj', 'o_proj'):
            sd[pre + f'self_attn.{n}.weight'] = getattr(layer.self_attn, n).dequantize()
        for n in ('gate_proj', 'up_proj', 'down_proj'):
            sd[pre + f'mlp.{n}.weight'] = getattr(layer.mlp, n).dequantize()
    p = prompts(77, 1, 100, 200)[0].to(DEV)
    got = _verify_logits(model, p)
    truth = causal_logits(sd, cfg, '13b', p[0])
    eager = causal_logits(sd, cfg, '13b', p[0], dtype=torch.bfloat16)
    _check(got, truth, eager)


# ---------------------------------------------------------------------------------------------------------------
# the real shapes: Baichuan-13B (40 layers, 5120 / 13696, 40 heads, V = 64000) and Baichuan2-7B (32 layers,
# 4096 / 11008, 32 heads, V = 125696, NormHead)
# ---------------------------------------------------------------------------------------------------------------
def baichuan_13b_config():
    return dict(model_type='baichuan', vocab_size=64000, hidden_size=5120, intermediate_size=13696,
                num_hidden_layers=40, num_attention_heads=40, hidden_act='silu', model_max_length=4096,
                rms_norm_eps=1e-6, bos_token_id=1, eos_token_id=2, pad_token_id=0, tie_word_embeddings=False)


def baichuan2_7b_config():
    return dict(model_type='baichuan', vocab_size=125696, hidden_size=4096, intermediate_size=11008,
                num_hidden_layers=32, num_attention_heads=32, hidden_act='silu', max_position_embeddings=4096,
                model_max_length=4096, rms_norm_eps=1e-6, bos_token_id=1, eos_token_id=2, pad_token_id=0,
                tie_word_embeddings=False)


@pytest.mark.big
@pytest.mark.parametrize('shape', ['baichuan-13b', 'baichuan2-7b'])
def test_baichuan_shapes_loop_is_exact(shape):
    """bench.synth_fill weights (NormHead applied), the oracle loop drives one copy, the fused device loop the other;
    64-token / 8-branch drafts, 256-token phrase-bank prompts, two passes: tokens, dls, edls identical"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    kind = '13b' if shape == 'baichuan-13b' else '2_7b'
    cfg = baichuan_config(baichuan_13b_config() if kind == '13b' else baichuan2_7b_config())
    cls = model_class(kind)
    a = bench.synth_fill(cls(cfg, device=torch.device(DEV)), cfg).normalize_lm_head()
    b = cls(cfg, device=torch.device(DEV))
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
