# -*- coding: utf-8 -*-
"""OPT on the H100: pia_kv_append_qscale bit for bit against eager CUDA torch (`q_proj(h) * scaling` after the bias
add, the zero-padded K / V planes), pia_learned_pos_embed against `wte[ids] + wpe[pos + 2]`, the fp8 GEMM's ReLU
epilogue against the bias epilogue's output through relu at split 1 and at 2-, 4- and 8-CTA clusters, all three in a
captured graph; then the lossless property of the verify forward against transformers' own OPTForCausalLM in fp32 at
head dims 64 / 80 / 128 and for the post-LN OPT-350m shape, and the tiny models through generate(), the oracle loop,
the batched loop, checkpoint loading and fp8.  `big`: the OPT-6.7B shape through the loop in bf16 and fp8."""
import json

import numpy as np
import pytest
import torch

from tests.test_gpu_baichuan import _check
from tests.test_gpu_generate import OursBackend
from tests.test_gpu_head_dim64 import _mask, _tree
from tests.test_gpu_kernels import _slots
from tests.tiny_models import prompts
from tests.tiny_opt import MAX_POS, hf_logits, tiny_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _deep_tree(rng, n):
    """ancestor rows of a tree of n nodes whose first 3n/4 form one chain, the rest hanging off random chain nodes"""
    m = max(1, 3 * n // 4)
    parent = [i - 1 for i in range(m)] + [int(rng.integers(0, m)) for _ in range(m, n)]
    rows = []
    for i in range(n):
        r, j = 0, i
        while j >= 0:
            r |= 1 << j
            j = parent[j]
        rows.append(r)
    return rows


# ---------------------------------------------------------------------------------------------------------------
# (a) pia_kv_append_qscale
# ---------------------------------------------------------------------------------------------------------------
# (H, d_src, D, R, slots [(n, P, pad)])
APPEND_CASES = [(12, 64, 64, 64, [(64, 40, 0)]), (4, 64, 64, 128, [(128, 30, 3)]),
                (32, 80, 128, 64, [(50, 300, 5)]), (3, 80, 128, 128, [(40, 10, 0), (20, 70, 2)]),
                (32, 128, 128, 64, [(16, 50, 2), (5, 0, 0), (0, 7, 0), (9, 300, 0)]),
                (2, 128, 128, 128, [(128, 0, 0)])]


def _append(qkv, mask, sl, H, d, D, max_seq, B, q_mul):
    from painlessinferenceacceleration_b200.common import ops
    R = qkv.shape[0]
    kc = torch.full((B, H, max_seq, D), 7.0, dtype=torch.bfloat16, device=DEV)
    vc = torch.full_like(kc, 7.0)
    q = torch.full((R, H, D), 9.0, dtype=torch.bfloat16, device=DEV)
    ops.kv_append(qkv, mask, sl, H, H, d, D, q_mul, q, kc[0], vc[0], max_seq)
    return q, kc, vc


@pytest.mark.parametrize('H,d,D,R,cases', APPEND_CASES)
def test_kv_append_qscale_bit_exact(H, d, D, R, cases):
    """q = eager CUDA `(addmm(b, y, W^T)) * d ** -0.5` (the Python float taken as fp32 by torch), zero-padded to D; K
    / V the projection's planes, zero-padded, at cache rows P + node of their slot; nothing else written"""
    rng = np.random.default_rng(H + d + R)
    torch.manual_seed(H * d + R)
    B = len(cases)
    rps = R // B if B > 1 else R
    trees = [_deep_tree(rng, n) for n, _, _ in cases]
    max_seq = max(P + n for n, P, _ in cases) + 40
    E = H * d
    y = torch.randn((B * rps, E), device=DEV).to(torch.bfloat16)
    w = (torch.randn((3 * E, E), device=DEV) * E ** -0.5).to(torch.bfloat16)
    bias = (torch.randn((3 * E,), device=DEV) * 0.5).to(torch.bfloat16)
    qkv = torch.addmm(bias, y, w.t())
    scaling = d ** -0.5
    mask = _mask(trees, R, rps)
    sl = _slots([n for n, _, _ in cases], [P for _, P, _ in cases], [p for _, _, p in cases], rps,
                stride=H * max_seq * D)
    q, kc, vc = _append(qkv, mask, sl, H, d, D, max_seq, B, scaling)
    torch.cuda.synchronize()
    x = qkv.view(B * rps, 3, H, d)
    q_want = torch.zeros((B * rps, H, D), dtype=torch.bfloat16, device=DEV)
    q_want[..., :d] = x[:, 0] * scaling                    # HF: q_proj(hidden_states) * self.scaling
    kv_want = torch.zeros((B * rps, 2, H, D), dtype=torch.bfloat16, device=DEV)
    kv_want[..., :d] = x[:, 1:]
    for s_, (n, P, pad) in enumerate(cases):
        r0 = s_ * rps
        assert torch.equal(q[r0:r0 + n], q_want[r0:r0 + n]), s_
        assert (q[r0 + n:r0 + rps] == 9.0).all()
        assert torch.equal(kc[s_, :, P:P + n], kv_want[r0:r0 + n, 0].transpose(0, 1)), s_
        assert torch.equal(vc[s_, :, P:P + n], kv_want[r0:r0 + n, 1].transpose(0, 1)), s_
        assert (kc[s_, :, :P] == 7.0).all() and (kc[s_, :, P + n:] == 7.0).all()
        assert (vc[s_, :, :P] == 7.0).all() and (vc[s_, :, P + n:] == 7.0).all()


def test_kv_append_qscale_refusals():
    from painlessinferenceacceleration_b200.common import ops
    qkv = torch.zeros((64, 3 * 2 * 80), dtype=torch.bfloat16, device=DEV)
    kc = torch.zeros((2, 100, 128), dtype=torch.bfloat16, device=DEV)
    q = torch.zeros((64, 2, 128), dtype=torch.bfloat16, device=DEV)
    mask, sl = _mask([[1]], 64, 64), _slots([1], [0], [0], 64)
    l0 = ops.launch_count()
    with pytest.raises(AssertionError, match='source head width'):
        ops.kv_append(qkv, mask, sl, 2, 2, 80, 64, 0.1, q, kc, kc.clone(), 100)    # d_src > D
    qkv_odd = torch.zeros((64, 3 * 2 * 76), dtype=torch.bfloat16, device=DEV)
    with pytest.raises(AssertionError, match='source head width'):
        ops.kv_append(qkv_odd, mask, sl, 2, 2, 76, 128, 0.1, q, kc, kc.clone(), 100)
    assert ops.launch_count() == l0


# ---------------------------------------------------------------------------------------------------------------
# (b) pia_learned_pos_embed
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('with_table', [True, False])
@pytest.mark.parametrize('R,hidden,cases', [(64, 768, [(64, 40, 0)]), (128, 2560, [(100, 480, 7)]),
                                            (64, 512, [(16, 50, 2), (5, 0, 0), (0, 7, 0), (9, 300, 0)]),
                                            (128, 9216, [(32, 60, 0), (20, 200, 4)])])
def test_learned_pos_embed_bit_exact(R, hidden, cases, with_table):
    """out = eager bf16 `wte[ids] + wpe[pos + 2]` at the tree positions (with the token table), or `out + wpe[pos + 2]`
    in place (without: OPT-350m after project_in); rows past their slot's n are zero"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(R + hidden)
    torch.manual_seed(R + hidden + with_table)
    B = len(cases)
    rps = R // B if B > 1 else R
    trees = [_deep_tree(rng, n) for n, _, _ in cases]
    n_pos = 1024
    wte = torch.randn((300, hidden), device=DEV).to(torch.bfloat16)
    wpe = torch.randn((n_pos + 2, hidden), device=DEV).to(torch.bfloat16)
    ids = torch.randint(0, 300, (B * rps,), dtype=torch.int32, device=DEV)
    mask = _mask(trees, R, rps)
    sl = _slots([n for n, _, _ in cases], [P for _, P, _ in cases], [p for _, _, p in cases], rps)
    a = torch.randn((B * rps, hidden), device=DEV).to(torch.bfloat16)
    out = a.clone() if not with_table else torch.full_like(a, 9.0)
    ops.learned_pos_embed(wte if with_table else None, ids, wpe, 2, mask, sl, out)
    torch.cuda.synchronize()
    for s_, ((n, P, pad), rows) in enumerate(zip(cases, trees)):
        r0 = s_ * rps
        assert (out[r0 + n:r0 + rps] == 0).all()
        if not n:
            continue
        pos = max(P - pad, 0) + torch.tensor([bin(r).count('1') - 1 for r in rows], device=DEV)
        base = wte[ids[r0:r0 + n].long()] if with_table else a[r0:r0 + n]
        assert torch.equal(out[r0:r0 + n], base + wpe[pos + 2]), s_


def test_learned_pos_embed_clamps_to_the_table():
    """a position past the table's last row reads the last row (a request never gets there: max_length is checked)"""
    from painlessinferenceacceleration_b200.common import ops
    wpe = torch.randn((10 + 2, 64), device=DEV).to(torch.bfloat16)
    wte = torch.randn((5, 64), device=DEV).to(torch.bfloat16)
    rows = _deep_tree(np.random.default_rng(1), 8)
    out = torch.empty((64, 64), dtype=torch.bfloat16, device=DEV)
    ids = torch.zeros((64,), dtype=torch.int32, device=DEV)
    ops.learned_pos_embed(wte, ids, wpe, 2, _mask([rows], 64, 64), _slots([8], [6], [0], 64), out)
    torch.cuda.synchronize()
    pos = (6 + torch.tensor([bin(r).count('1') - 1 for r in rows], device=DEV)).clamp(max=9)
    assert torch.equal(out[:8], wte[0] + wpe[pos + 2])


# ---------------------------------------------------------------------------------------------------------------
# (c) the fp8 ReLU epilogue
# ---------------------------------------------------------------------------------------------------------------
def _fp8_weights(N, K, seed):
    from painlessinferenceacceleration_b200.common import ops
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn((N, K), device=DEV, generator=g) * K ** -0.5
    q, s = ops.quantize_fp8(w)
    x = torch.randn((128, K), device=DEV, generator=g).to(torch.bfloat16)
    bias = torch.randn((N,), device=DEV, generator=g) * 0.3
    return ops.tile_weight_fp8(q), s, x, bias


@pytest.mark.parametrize('split', [1, -2, -4, -8])
@pytest.mark.parametrize('rows', [1, 37, 64, 128])
def test_fp8_relu_epilogue_bit_exact(split, rows):
    """set_relu: every output = relu of the same plan's bias-epilogue output, bit for bit, and roughly half of them
    were negative (the flag has something to do)"""
    from painlessinferenceacceleration_b200.common import ops
    qw, s, x, bias = _fp8_weights(512, 1024, 3 + split)
    plain = ops.Gemm.fp8(qw, s, x, bias=bias, split_k=split)
    relu = ops.Gemm.fp8(qw, s, x, bias=bias, split_k=split).set_relu()
    assert plain.splits == 1 and relu.splits == 1   # cluster splits write bf16
    a, b = plain.run(rows).clone(), relu.run(rows).clone()
    torch.cuda.synchronize()
    assert torch.equal(b[:rows], torch.relu(a[:rows]))
    neg = (a[:rows] < 0).float().mean().item()
    assert 0.3 < neg < 0.7, neg
    relu.set_relu(False)
    assert torch.equal(relu.run(rows)[:rows], a[:rows])


def test_fp8_relu_refusals():
    """no ReLU on plans that write fp32 split-K slices, on SiLU plans, or on bf16-weight plans; no SiLU on a ReLU
    plan"""
    from painlessinferenceacceleration_b200.common import ops
    qw, s, x, bias = _fp8_weights(256, 1024, 9)
    with pytest.raises(AssertionError, match='ReLU'):
        ops.Gemm.fp8(qw, s, x, split_k=2).set_relu()
    with pytest.raises(AssertionError, match='activation'):
        ops.Gemm.fp8(qw, s, x).set_silu().set_relu()
    with pytest.raises(AssertionError, match='activation'):
        ops.Gemm.fp8(qw, s, x).set_relu().set_silu()
    wb = torch.zeros((256, 1024), dtype=torch.bfloat16, device=DEV)
    with pytest.raises(AssertionError, match='fp8'):
        ops.Gemm(wb, x).set_relu()


def test_new_kernels_in_a_captured_graph():
    """the three kernels replay inside one CUDA graph with their eager results"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(5)
    rows = _deep_tree(np.random.default_rng(2), 64)
    mask, sl = _mask([rows], 64, 64), _slots([64], [33], [2], 64)
    H, d, D = 4, 80, 128
    qkv = torch.randn((64, 3 * H * d), device=DEV).to(torch.bfloat16)
    kc = torch.zeros((H, 200, D), dtype=torch.bfloat16, device=DEV)
    vc, q = torch.zeros_like(kc), torch.zeros((64, H, D), dtype=torch.bfloat16, device=DEV)
    wte = torch.randn((50, 512), device=DEV).to(torch.bfloat16)
    wpe = torch.randn((300, 512), device=DEV).to(torch.bfloat16)
    ids = torch.randint(0, 50, (64,), dtype=torch.int32, device=DEV)
    emb = torch.zeros((64, 512), dtype=torch.bfloat16, device=DEV)
    qw, s, x, bias = _fp8_weights(512, 1024, 11)
    gm = ops.Gemm.fp8(qw, s, x, bias=bias, split_k=-4).set_relu()

    def run():
        ops.kv_append(qkv, mask, sl, H, H, d, D, d ** -0.5, q, kc, vc, 200)
        ops.learned_pos_embed(wte, ids, wpe, 2, mask, sl, emb)
        gm.run(64)

    out = gm.out[:64]   # the plan's buffer holds x's 128 rows; run(64) writes the first 64
    run()
    want = [t.clone() for t in (q, kc, vc, emb, out)]
    for t in (q, kc, vc, emb, out):
        t.zero_()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip((q, kc, vc, emb, out), want):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------
# lossless: the verify logits of every draft node = a causal forward over prefix + root-to-node path
# ---------------------------------------------------------------------------------------------------------------
SHAPES = [64, 80, 128, '350m']


@pytest.mark.parametrize('shape', SHAPES)
def test_tree_verify_logits_are_lossless(shape):
    """a prompt (two chain chunks), then one random 64-node tree: each node's verify-logit row vs transformers'
    OPTForCausalLM in fp32 over prompt + its root-to-node path, within 2 x the bf16 eager model's own error + 0.02"""
    model, hf = tiny_model(shape, seed=3)
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


@pytest.mark.parametrize('shape', [64, 80, '350m'])
def test_prefill_with_left_padding_is_lossless(shape):
    """the prefill pass of a left-padded prompt: its last-row logits vs the HF forward of the unpadded prompt"""
    model, hf = tiny_model(shape, seed=6)
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


@pytest.mark.parametrize('shape,penalty', [(64, 1.0), (80, 1.1), (128, 1.0), ('350m', 1.1)])
def test_generate_equals_plain_greedy(shape, penalty):
    """lookahead generate() (prefill + tree drafts) gives the tokens of plain greedy decoding with the same kernels,
    and a second pass over the same prompts accepts drafts"""
    model = _cache(tiny_model(shape, seed=1)[0])
    edls = []
    for rep in range(2):
        for p in prompts(21, 2, 40, 200):
            p = p.to(DEV)
            g = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               decoding_kwargs={'use_lookahead': False})
            o = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               return_dict_in_generate=True,
                               decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
            assert o.sequences[0].tolist() == g[0].tolist(), (shape, rep)
            edls += o.kwargs['edls'][1:]
    assert max(edls) > 2


def test_do_sample():
    """an untied lm_head keeps the logits soft enough for sampling to leave the greedy path"""
    model = _cache(tiny_model(80, seed=2, tie=False)[0])
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


@pytest.mark.parametrize('shape,penalty', [(64, 1.1), (80, 1.0), ('350m', 1.0)])
def test_loop_is_exact_given_the_same_logits(shape, penalty):
    """the oracle loop drives one copy of our model, the fused device loop another: tokens, dls, edls identical"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    a = _cache(tiny_model(shape, seed=6)[0])
    b = tiny_model(shape, seed=6)[0]
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
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (shape, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (shape, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def test_batched_generate_equals_per_request():
    """the batched loop class over a batch of 3 prompts gives the per-request greedy tokens, up to a near-tie of the
    logits (the batched step splits the KV range differently, which moves the fp32 summation order)"""
    single = _cache(tiny_model(64, seed=5)[0])
    batch = _cache(tiny_model(64, seed=5, batch=True)[0])
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


def test_max_length_past_the_position_table_is_refused():
    """refused before a runtime or a graph exists, in the per-request and the batched loop"""
    model = _cache(tiny_model(64, seed=2)[0])
    p = prompts(3, 1, 16, 200)[0].to(DEV)
    with pytest.raises(ValueError, match='max_position_embeddings'):
        model.generate(input_ids=p, max_length=MAX_POS + 1, eos_token_id=2,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert not model._rt.graphs
    batch = _cache(tiny_model(64, seed=2, batch=True)[0])
    with pytest.raises(ValueError, match='max_position_embeddings'):
        batch.generate(input_ids=torch.cat([p, p]), max_length=MAX_POS + 1, eos_token_id=2,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert batch._rt is None
    o = model.generate(input_ids=p, max_length=MAX_POS, eos_token_id=2,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert o.shape[1] <= MAX_POS


def test_fused_attention_knob_is_refused(monkeypatch):
    model = _cache(tiny_model(64, seed=4)[0])
    monkeypatch.setenv('PIA_ATTN_FUSED', '1')
    with pytest.raises(ValueError, match='PIA_ATTN_FUSED'):
        model.generate(input_ids=prompts(6, 1, 16, 200)[0].to(DEV), max_new_tokens=8, eos_token_id=2,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert model._rt is None


# ---------------------------------------------------------------------------------------------------------------
# checkpoints and fp8
# ---------------------------------------------------------------------------------------------------------------
def _verify_logits(model, p):
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    return OursBackend(model).forward(p, m01, None)[0].float()


@pytest.mark.parametrize('shape', [64, '350m'])
def test_from_pretrained_bf16_and_fp8(tmp_path, shape):
    """a save_pretrained directory (`model.decoder.` names) and an unprefixed OPTDecoder-style sharded one load into
    the logits of the same weights handed over directly; quantization='fp8' loads, one layer at a time, into the bytes
    and logits of quantize_fp8() on that model"""
    from safetensors.torch import save_file
    from painlessinferenceacceleration_b200.models.opt.modeling_opt import OPTForCausalLM
    direct, hf = tiny_model(shape, seed=10)
    hf.save_pretrained(str(tmp_path / 'hf'))
    plain = tmp_path / 'plain'
    plain.mkdir()
    (plain / 'config.json').write_text(json.dumps(hf.config.to_dict()))
    sd = {k: v.detach().cpu().contiguous() for k, v in hf.model.decoder.state_dict().items()}
    keys = sorted(sd)
    save_file({k: sd[k] for k in keys[:len(keys) // 2]}, str(plain / 'model-00001-of-00002.safetensors'))
    save_file({k: sd[k] for k in keys[len(keys) // 2:]}, str(plain / 'model-00002-of-00002.safetensors'))
    p = prompts(79, 1, 70, 200)[0].to(DEV)
    want = _verify_logits(direct, p)
    for d in ('hf', 'plain'):
        loaded = OPTForCausalLM.from_pretrained(str(tmp_path / d), device=torch.device(DEV))
        assert loaded.lm_head.weight is loaded.model.decoder.embed_tokens.weight
        assert torch.equal(_verify_logits(loaded, p), want), d
    direct.quantize_fp8()
    want8 = _verify_logits(direct, p)
    for d in ('hf', 'plain'):
        f8 = OPTForCausalLM.from_pretrained(str(tmp_path / d), device=torch.device(DEV), quantization='fp8')
        for (k, a), (k2, b) in zip(sorted(direct.state_dict().items()), sorted(f8.state_dict().items())):
            assert k == k2 and torch.equal(a, b), (d, k)
        assert torch.equal(_verify_logits(f8, p), want8), d


def _dequantised_hf_state(hf, ours):
    """the HF state dict with every fp8 projection replaced by its dequantised weight (fp32)"""
    sd = {k: v.float().clone() for k, v in hf.state_dict().items()}
    for li, layer in enumerate(ours.model.decoder.layers):
        pre = f'model.decoder.layers.{li}.'
        a = layer.self_attn
        for n in ('q_proj', 'k_proj', 'v_proj', 'out_proj'):
            sd[pre + f'self_attn.{n}.weight'] = getattr(a, n).dequantize()
        for n in ('fc1', 'fc2'):
            sd[pre + f'{n}.weight'] = getattr(layer, n).dequantize()
    return sd


@pytest.mark.parametrize('shape', [64, 128, '350m'])
def test_fp8_verify_logits_within_tolerance(shape):
    """fp8 verify logits vs an fp32 evaluation of the dequantised weights: max |error| <= 2 x the eager bf16 error of
    the same weights + 0.02 (the Llama fp8 tests' tolerance)"""
    import copy
    ours, hf = tiny_model(shape, seed=8)
    ours.quantize_fp8()
    deq = _dequantised_hf_state(hf, ours)
    p = prompts(77, 1, 100, 200)[0].to(DEV)
    hf32 = copy.deepcopy(hf)
    with torch.no_grad():
        hf32.load_state_dict(deq)
        truth = hf32(input_ids=p).logits[0].float()
        eager_m = copy.deepcopy(hf32).to(torch.bfloat16)
        eager = eager_m(input_ids=p).logits[0].float()
    got = _verify_logits(ours, p)
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    print(f'fp8 verify logits opt {shape}: err vs dequantised fp32 {e_ours:.4f}, eager bf16 {e_eager:.4f}')
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)


def test_fp8_lookahead_equals_own_greedy():
    model = _cache(tiny_model(128, seed=4)[0].quantize_fp8())
    for p in prompts(33, 2, 24, 200):
        p = p.to(DEV)
        g = model.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
        for _ in range(2):
            o = model.generate(input_ids=p, max_new_tokens=40, eos_token_id=2,
                               decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
        assert o[0].tolist() == g[0].tolist()


# ---------------------------------------------------------------------------------------------------------------
# the real shape: OPT-6.7B (32 layers, 4096, 32 heads of 128, ffn 16384, V = 50 272)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.big
@pytest.mark.parametrize('fp8', [False, True])
def test_opt_6_7b_shape_loop_is_exact(fp8):
    """the benchmark's synthetic weights, the oracle loop drives one copy, the fused device loop the other; 64-token /
    8-branch drafts, 256-token phrase-bank prompts, two passes: tokens, dls, edls identical"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from scripts.bench_opt import opt_config, synth_opt
    cfg = opt_config('6.7b')
    a = synth_opt(cfg, fp8)
    b = synth_opt(cfg, fp8)
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
