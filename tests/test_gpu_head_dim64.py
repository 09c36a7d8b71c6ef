# -*- coding: utf-8 -*-
"""Head dim 64 on the H100: k_tree_attn<64> (plain and fused RoPE / KV append, 64- and 128-node drafts, several slots,
prefill chunks sharing one cache), the plan's grid and refusals, and two tiny models - a Llama with llama3 RoPE and a
Qwen2 with G = 7 and q/k/v biases - through the verify forward, the loop, the batched loop, sampling, checkpoint
loading and fp8 weights.  `big`: the Llama-3.2-1B and Qwen2.5-0.5B shapes through the loop."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import attn_ref
from tests.test_gpu_fp8 import OursBackend128, _same_bytes
from tests.test_gpu_generate import EPS, OursBackend
from tests.test_gpu_kernels import _ref_attention, _slots
from tests.tiny_models import prompts
from tests.tiny_qwen2 import qwen2_hf_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
D = 64
HEADS = [(4, 4), (32, 8), (14, 2), (7, 1), (3, 1)]


# ---------------------------------------------------------------------------------------------------------------
# k_tree_attn at head dim 64
# ---------------------------------------------------------------------------------------------------------------
def _tree(rng, n, max_depth=8):
    """ancestor rows (python ints, bit j = draft node j) of a random DFS-pre-order tree of n <= 128 nodes"""
    parent, depth = [-1], [0]
    for i in range(1, n):
        path = [i - 1]
        while parent[path[-1]] >= 0:
            path.append(parent[path[-1]])
        cands = [p for p in path if depth[p] < max_depth]
        p = cands[int(rng.integers(0, len(cands)))] if cands else 0
        parent.append(p)
        depth.append(depth[p] + 1)
    rows = []
    for i in range(n):
        r, j = 0, i
        while j >= 0:
            r |= 1 << j
            j = parent[j]
        rows.append(r)
    return rows


def _mask(rows_per_slot, R, rps):
    """[len(rows_per_slot) * rps, R // 64] int64 mask words of the slots' trees"""
    W = R // 64
    m = np.zeros((len(rows_per_slot) * rps, W), dtype=np.uint64)
    for s_, rows in enumerate(rows_per_slot):
        for i, r in enumerate(rows):
            for w in range(W):
                m[s_ * rps + i, w] = np.uint64((r >> (64 * w)) & 0xFFFFFFFFFFFFFFFF)
    return torch.from_numpy(m.view(np.int64)).to(DEV)


def _rope(max_pos, theta=500000.0):
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, device=DEV).float() / D))
    ang = torch.arange(max_pos, device=DEV).float()[:, None] * inv[None]
    return ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()


def _cases():
    out = [(hq, hkv, P, n, 64) for hq, hkv in HEADS for P in (0, 127, 128, 129, 1000, 3968) for n in (1, 33, 64)]
    out += [(hq, hkv, P, n, 128) for hq, hkv in HEADS for P in (0, 129, 3968) for n in (65, 128)]
    return out


@pytest.mark.parametrize('Hq,Hkv,P,n,R', _cases())
def test_tree_attention_d64(Hq, Hkv, P, n, R):
    """pia_tree_attn_fwd at D = 64 against the fp32 restatement, left padding (P % 7 columns) included; rows beyond the
    draft stay untouched"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(P + n + Hq + R)
    torch.manual_seed(P * 7 + n + Hq)
    pad = P % 7 if P > 8 else 0
    n_layers, max_seq = 2, P + n + 70
    kc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    q = (torch.randn((R, Hq, D), device=DEV) * 0.7).to(torch.bfloat16)
    rows = _tree(rng, n)
    mask = _mask([rows], R, R)
    plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
    out = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    for layer in (1, 0):
        out.fill_(9.0)
        plan.forward(layer, q, mask, _slots([n], [P], [pad], R), out)
        torch.cuda.synchronize()
        ref = _ref_attention(q, kc[layer], vc[layer], rows, n, P, pad, Hq // Hkv)
        err = (out[:n].float() - ref).abs().max().item()
        attn_ref.assert_close(out[:n].float(), ref, f'layer {layer} max abs err {err}')
        assert float((out[n:].float() - 9.0).abs().sum()) == 0


@pytest.mark.parametrize('Hq,Hkv,R,rps,cases', [
    (32, 8, 64, 64, [(64, 384, 0)]),
    (14, 2, 64, 64, [(33, 0, 0)]),                                 # empty cache: the draft tile is the only tile
    (7, 1, 64, 64, [(47, 1000, 5)]),                               # ragged draft, left padding
    (3, 1, 64, 64, [(1, 130, 0)]),                                 # a root-only draft right after a tile boundary
    (4, 4, 64, 64, [(64, 3968, 0)]),
    (14, 2, 128, 128, [(128, 700, 3)]),                            # 128-node draft
    (7, 1, 128, 128, [(90, 129, 0)]),
    (14, 2, 64, 8, [(8, 300, 0), (3, 290, 0), (8, 310, 2), (1, 5, 0), (7, 128, 0), (8, 64, 0), (2, 500, 0), (6, 301, 0)]),
    (32, 8, 64, 16, [(16, 100, 0), (5, 0, 0), (0, 7, 0), (9, 257, 3)])])
def test_fused_and_two_kernel_paths_d64(Hq, Hkv, R, rps, cases):
    """fused RoPE / KV append / attention against pia_rope_kv_append + pia_tree_attn_fwd on the same inputs, one cache
    per slot: the appended cache rows are bit identical, both outputs agree with the fp32 reference"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(Hq + rps + R)
    torch.manual_seed(Hq * 3 + rps + R)
    n_layers, B = 2, len(cases)
    max_seq = max(P + n for n, P, _ in cases) + 70
    kc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    rows_all = B * rps
    qkv = torch.randn((rows_all, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    cos, sin = _rope(max_seq + 8)
    trees = [_tree(rng, n) for n, _, _ in cases]
    mask = _mask(trees, R, rps)
    ns, Ps, pads = [c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases]
    layer = 1
    k2, v2 = kc.clone(), vc.clone()
    plan, plan2 = ops.AttnPlan(kc, vc, Hq, Hkv, D, R), ops.AttnPlan(k2, v2, Hq, Hkv, D, R)
    sl = _slots(ns, Ps, pads, rps, stride=plan.slot_stride if B > 1 else 0)
    q = torch.zeros((rows_all, Hq, D), dtype=torch.bfloat16, device=DEV)
    o1 = torch.full((rows_all, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    o2 = torch.full((rows_all, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    ops.rope_kv_append(qkv, mask, sl, Hq, Hkv, D, cos, sin, q, kc[0, layer], vc[0, layer], max_seq)
    plan.forward(layer, q, mask, sl, o1)
    plan2.forward_fused(layer, qkv, mask, sl, cos, sin, o2)
    torch.cuda.synchronize()
    assert torch.equal(k2, kc) and torch.equal(v2, vc)
    for s_, (n, P, pad) in enumerate(cases):
        r0 = s_ * rps
        if n:
            ref = _ref_attention(q[r0:], kc[s_, layer], vc[s_, layer], trees[s_], n, P, pad, Hq // Hkv)
            attn_ref.assert_close(o1[r0:r0 + n].float(), ref, s_)
            attn_ref.assert_close(o2[r0:r0 + n].float(), ref, s_)
            assert torch.allclose(o2[r0:r0 + n].float(), o1[r0:r0 + n].float(), atol=4e-3, rtol=2e-2), s_
        assert float((o2[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0
        assert float((o1[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0


@pytest.mark.parametrize('Hq,Hkv', [(14, 2), (8, 2)])
def test_prefill_chunks_share_one_cache_d64(Hq, Hkv):
    """a prefill pass at D = 64: one table slot per 64-row chain chunk over the same cache (kv_slot_stride 0) equals
    feeding the chunks one after the other, and the fp32 reference"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(5 + Hq)
    R, Cn, n_layers, lens, max_seq, base = 64, 3, 1, [64, 64, 23], 400, 40
    chain = [(1 << (i + 1)) - 1 for i in range(R)]
    mask = _mask([chain] * Cn, R, R)
    qkv = torch.randn((Cn * R, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    cos, sin = _rope(max_seq)
    outs = []
    for batched in (True, False):
        kc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV, generator=torch.Generator(DEV).manual_seed(1)) * 0.7).to(torch.bfloat16)
        vc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV, generator=torch.Generator(DEV).manual_seed(2)) * 0.7).to(torch.bfloat16)
        plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
        q = torch.zeros((Cn * R, Hq, D), dtype=torch.bfloat16, device=DEV)
        o = torch.zeros((Cn * R, Hq, D), dtype=torch.bfloat16, device=DEV)
        if batched:
            sl = _slots(lens, [base + R * c for c in range(Cn)], [0] * Cn, R)
            ops.rope_kv_append(qkv, mask, sl, Hq, Hkv, D, cos, sin, q, kc[0], vc[0], max_seq)
            plan.forward(0, q, mask, sl, o)
        else:
            for c in range(Cn):
                sl = _slots([lens[c]], [base + R * c], [0], R)
                ops.rope_kv_append(qkv[R * c:], mask[R * c:], sl, Hq, Hkv, D, cos, sin, q[R * c:], kc[0], vc[0], max_seq)
            for c in range(Cn):
                plan.forward(0, q[R * c:], mask[R * c:], _slots([lens[c]], [base + R * c], [0], R), o[R * c:])
        torch.cuda.synchronize()
        outs.append((q.clone(), o.clone(), kc.clone(), vc.clone()))
    (q_a, o_a, k_a, v_a), (q_b, o_b, k_b, v_b) = outs
    assert torch.equal(q_a, q_b) and torch.equal(k_a, k_b) and torch.equal(v_a, v_b)
    assert torch.allclose(o_a.float(), o_b.float(), atol=4e-3, rtol=2e-2)
    for c in range(Cn):
        ref = _ref_attention(q_a[R * c:], k_a[0], v_a[0], chain, lens[c], base + R * c, 0, Hq // Hkv)
        attn_ref.assert_close(o_a[R * c:R * c + lens[c]].float(), ref, c)


def _plan_rc(Hq, Hkv, hd, max_nodes):
    from painlessinferenceacceleration_b200 import _lib as L
    kc = torch.zeros((1, Hkv, 4096, hd), dtype=torch.bfloat16, device=DEV)
    vc = kc.clone()
    cfg = L.AttnConfig(Hq, Hkv, hd, 4096, max_nodes, 1, 0, 1)
    h = L.vp()
    lib = L.load()
    rc = lib.pia_attn_plan_create(C.byref(cfg), C.c_void_p(kc.data_ptr()), C.c_void_p(vc.data_ptr()), C.byref(h))
    grid = None
    if rc == 0:
        ns, ng = C.c_int(0), C.c_int(0)
        assert lib.pia_attn_plan_grid(h, C.byref(ns), C.byref(ng)) == 0
        grid = (ns.value, ng.value)
        lib.pia_attn_plan_destroy(h)
    return rc, grid


@pytest.mark.parametrize('Hq,Hkv,max_nodes', [(32, 8, 64), (14, 2, 64), (7, 1, 64), (4, 4, 64), (3, 1, 64),
                                               (32, 8, 128), (14, 2, 128)])
def test_attention_grid_d64_equals_d128(Hq, Hkv, max_nodes):
    """the head packing and the KV split do not depend on the head dim"""
    rc64, g64 = _plan_rc(Hq, Hkv, 64, max_nodes)
    rc128, g128 = _plan_rc(Hq, Hkv, 128, max_nodes)
    assert rc64 == 0 and rc128 == 0 and g64 == g128


@pytest.mark.parametrize('hd', [96, 256, 32])
def test_other_head_dims_are_refused(hd):
    from painlessinferenceacceleration_b200 import _lib as L
    rc, _ = _plan_rc(8, 2, hd, 64)
    assert rc == L.PIA_ERR_UNSUPPORTED
    assert f'head_dim {hd}' in L.load().pia_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------
# tiny models at head dim 64
# ---------------------------------------------------------------------------------------------------------------
def llama64_config(vocab=200, **over):
    """Llama, head dim 64, llama3 RoPE whose smoothing band falls inside the test lengths; every projection dimension
    a multiple of 128 (fp8)"""
    from transformers import LlamaConfig
    kw = dict(vocab_size=vocab, hidden_size=512, intermediate_size=512, num_hidden_layers=2, num_attention_heads=8,
              num_key_value_heads=2, max_position_embeddings=1024, rms_norm_eps=1e-6, bos_token_id=1, eos_token_id=2,
              pad_token_id=0, tie_word_embeddings=False, rope_theta=10000.0,
              rope_scaling={'rope_type': 'llama3', 'factor': 8.0, 'low_freq_factor': 1.0, 'high_freq_factor': 4.0,
                            'original_max_position_embeddings': 256})
    kw.update(over)
    cfg = LlamaConfig(**kw)
    cfg._attn_implementation = 'eager'
    return cfg


def llama64_hf_model(seed=0, dtype=torch.float32, device='cpu', vocab=200, **over):
    """seeded and initialised like tests/tiny_models.py"""
    from transformers import AutoModelForCausalLM
    torch.manual_seed(seed)
    model = AutoModelForCausalLM.from_config(llama64_config(vocab=vocab, **over), attn_implementation='eager')
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() >= 2:
                p.normal_(0.0, 0.08)
    return model.to(device=device, dtype=dtype).eval()


def qwen64_hf_model(seed=0, dtype=torch.float32, device='cpu', vocab=200, **over):
    """tests/tiny_qwen2.py's model at head dim 64: hidden 448, 7 query heads over 1 KV head, q/k/v biases"""
    return qwen2_hf_model(seed=seed, dtype=dtype, device=device, vocab=vocab, hidden_size=448, **over)


def _hf(family, seed, dtype, **over):
    return (llama64_hf_model if family == 'llama' else qwen64_hf_model)(seed=seed, dtype=dtype, device=DEV, **over)


def _cls(family):
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    return LlamaForCausalLM if family == 'llama' else Qwen2ForCausalLM


def _ours(family, hf):
    m = _cls(family)(hf.config, device=torch.device(DEV))
    res = m.load_state_dict(hf.state_dict(), strict=False)
    assert not res.missing_keys, res
    return m


def _verify_logits(model, p):
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    return OursBackend(model).forward(p, m01, None)[0].float()


@pytest.mark.parametrize('family', ['llama', 'qwen2'])
def test_d64_verify_logits_within_tolerance(family):
    """our bf16 verify forward vs an fp32 evaluation of the same weights (HF eager, llama3 RoPE for the Llama): max
    |error| <= 2 x the eager bf16 HF model's own error + 0.02, same greedy tokens wherever the fp32 margin is clear"""
    hf = _hf(family, 8, torch.bfloat16)
    ours = _ours(family, hf)
    assert ours.geometry()['head_dim'] == 64
    hf32 = _hf(family, 8, torch.float32)
    hf32.load_state_dict({k: v.float() for k, v in hf.state_dict().items()})
    p = prompts(77, 1, 100, 200)[0].to(DEV)
    with torch.no_grad():
        truth = hf32(input_ids=p).logits[0].float()
        eager = hf(input_ids=p).logits[0].float()
    got = _verify_logits(ours, p)
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)
    top = torch.topk(truth, 2, dim=-1).values
    sure = (top[:, 0] - top[:, 1]) > 2 * e_ours
    assert torch.equal(got.argmax(-1)[sure], truth.argmax(-1)[sure])


@pytest.mark.parametrize('family,penalty,dl', [('llama', 1.0, 64), ('llama', 1.1, 64), ('llama', 1.0, 128),
                                               ('qwen2', 1.0, 64), ('qwen2', 1.1, 128)])
def test_d64_loop_is_exact_given_the_same_logits(family, penalty, dl):
    """the oracle loop drives one copy of our model through the backend interface, the fused device loop another copy
    with the same weights: tokens, dls and edls identical for every request, tries carried across requests"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf = _hf(family, 6, torch.bfloat16)
    a, b = _ours(family, hf), _ours(family, hf)
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
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (family, dl, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (family, dl, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def test_d64_batched_loop_matches_single_request_loop():
    """the batched Llama class (bs = 3) at head dim 64: every request equals the single-request loop, except where they
    part on a near-tie of the model's own logits"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.llama.modeling_llama_batch import LlamaForCausalLM as Batched
    hf = _hf('llama', 14, torch.bfloat16)
    single = _ours('llama', hf)
    batched = Batched(hf.config, device=torch.device(DEV))
    assert not batched.load_state_dict(hf.state_dict(), strict=False).missing_keys
    ps = torch.cat([p for p in prompts(61, 3, 20, 200)], dim=0).to(DEV)
    dk = {'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8}
    batched.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    single.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    outb = batched.generate(input_ids=ps, max_new_tokens=32, eos_token_id=2, decoding_kwargs=dict(dk))
    outb = outb.sequences if hasattr(outb, 'sequences') else outb
    same = 0
    for i in range(3):
        s = single.generate(input_ids=ps[i:i + 1], max_new_tokens=32, eos_token_id=2, decoding_kwargs=dict(dk))[0].tolist()
        bt = outb[i].tolist()[:len(s)]
        if bt == s:
            same += 1
            continue
        k = next(j for j in range(min(len(bt), len(s))) if bt[j] != s[j])
        m01 = torch.tril(torch.ones((1, 1, k, k), dtype=torch.long, device=DEV))
        lg = single.forward(torch.tensor([s[:k]], device=DEV), m01)[0][0, -1].float()
        top = torch.topk(lg, 2).values
        assert (top[0] - top[1]).item() < EPS, (i, k)
    assert same >= 1


@pytest.mark.parametrize('family,dl', [('llama', 64), ('qwen2', 128)])
def test_d64_do_sample(family, dl):
    """multinomial accept at head dim 64: well-formed output (lengths, accepted lengths summing to the new tokens,
    ids inside the vocabulary), and sampling really departs from greedy decoding somewhere"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf = _hf(family, 3, torch.bfloat16)
    ours = _ours(family, hf)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    torch.manual_seed(11)
    differs = 0
    for p in prompts(9, 3, 24, 200):
        p = p.to(DEV)
        g = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
        o = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, do_sample=True, return_dict_in_generate=True,
                          decoding_kwargs={'use_lookahead': True, 'decoding_length': dl, 'branch_length': 8})
        seq = o.sequences[0].tolist()
        assert seq[:24] == p[0].tolist() and len(seq) <= 24 + 40
        assert sum(o.kwargs['edls']) == len(seq) - 24
        assert all(0 <= t < 200 for t in seq)
        differs += seq != g[0].tolist()
    assert differs >= 1


@pytest.mark.parametrize('family,tied', [('llama', False), ('llama', True), ('qwen2', False), ('qwen2', True)])
def test_d64_from_pretrained(tmp_path, family, tied):
    """a save_pretrained directory loads into the logits of the weights handed over directly, tied and untied; then
    generate() with lookahead runs on the loaded model"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf = _hf(family, 10, torch.bfloat16, tie_word_embeddings=tied)
    direct = _ours(family, hf)
    hf.save_pretrained(str(tmp_path))
    loaded = _cls(family).from_pretrained(str(tmp_path), device=torch.device(DEV))
    assert loaded.config.rope_parameters == hf.config.rope_parameters
    if tied:
        assert torch.equal(loaded.lm_head.weight, loaded.model.embed_tokens.weight)
    p = prompts(79, 1, 70, 200)[0].to(DEV)
    assert torch.equal(_verify_logits(loaded, p), _verify_logits(direct, p))
    loaded.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    out = loaded.generate(input_ids=p, max_new_tokens=24, eos_token_id=2, return_dict_in_generate=True,
                          decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert sum(out.kwargs['edls']) == out.sequences.shape[1] - 70


@pytest.mark.parametrize('dl', [64, 128])
def test_d64_fp8_loop_is_exact_given_the_same_logits(dl):
    """quantize_fp8() on the head-dim-64 Llama (every projection dimension a multiple of 128); the oracle loop drives
    one fp8 copy, the fused device loop another with identical bytes: tokens, dls and edls identical; the fp8 model
    from from_pretrained(..., quantization='fp8') runs as well"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf = _hf('llama', 6, torch.bfloat16)
    a, b = _ours('llama', hf).quantize_fp8(), _ours('llama', hf).quantize_fp8()
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
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (dl, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (dl, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def test_d64_fp8_from_pretrained(tmp_path):
    """from_pretrained(..., quantization='fp8') of a head-dim-64 llama3 checkpoint gives quantize_fp8()'s bytes and runs
    generate() with lookahead"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf = _hf('llama', 12, torch.bfloat16, tie_word_embeddings=True)
    hf.save_pretrained(str(tmp_path))
    ref = _ours('llama', hf).quantize_fp8()
    got = _cls('llama').from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')
    _same_bytes(ref, got)
    got.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    p = prompts(80, 1, 40, 200)[0].to(DEV)
    out = got.generate(input_ids=p, max_new_tokens=24, eos_token_id=2, return_dict_in_generate=True,
                       decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    assert sum(out.kwargs['edls']) == out.sequences.shape[1] - 40


# ---------------------------------------------------------------------------------------------------------------
# the real shapes: Llama-3.2-1B and Qwen2.5-0.5B
# ---------------------------------------------------------------------------------------------------------------
def llama32_1b_shape():
    from transformers import LlamaConfig
    return LlamaConfig(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16,
                       num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=4096, rms_norm_eps=1e-5,
                       rope_theta=500000.0, tie_word_embeddings=False, bos_token_id=1, eos_token_id=2, pad_token_id=0,
                       rope_scaling={'rope_type': 'llama3', 'factor': 32.0, 'low_freq_factor': 1.0,
                                     'high_freq_factor': 4.0, 'original_max_position_embeddings': 8192})


def qwen25_05b_shape():
    from transformers import Qwen2Config
    return Qwen2Config(vocab_size=151936, hidden_size=896, intermediate_size=4864, num_hidden_layers=24,
                       num_attention_heads=14, num_key_value_heads=2, max_position_embeddings=4096, rms_norm_eps=1e-6,
                       rope_theta=1000000.0, use_sliding_window=False, tie_word_embeddings=False,
                       bos_token_id=1, eos_token_id=2, pad_token_id=0)


@pytest.mark.big
@pytest.mark.parametrize('shape', ['llama3.2-1b', 'qwen2.5-0.5b'])
def test_head_dim64_shapes_loop_is_exact(shape):
    """as test_qwen2_7b_loop_is_exact: bench.synth_fill weights, the oracle loop drives one copy, the fused device loop
    the other; 64-token / 8-branch drafts, 256-token phrase-bank prompts, two passes.  Tokens, dls and edls identical,
    and the second pass accepts drafts longer than 2"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    family = 'llama' if shape.startswith('llama') else 'qwen2'
    cfg = llama32_1b_shape() if family == 'llama' else qwen25_05b_shape()
    a = bench.synth_fill(_cls(family)(cfg, device=torch.device(DEV)), cfg)
    b = _cls(family)(cfg, device=torch.device(DEV))
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
