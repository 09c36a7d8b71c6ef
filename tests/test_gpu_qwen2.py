# -*- coding: utf-8 -*-
"""Qwen2 on the H100: tree attention at odd GQA groups (two query heads of one KV head per 128-row tile, the last
tile of each KV head holding one), the biased QKV projection through the verify forward and the loop, checkpoint
loading, the sliding-window warning and the refusal of a GEMM set that would drop the QKV bias."""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from tests import attn_ref
from tests.test_gpu_generate import OursBackend, _legit_divergence
from tests.test_gpu_kernels import _mask_tensor, _random_tree, _ref_attention, _slots
from tests.tiny_models import prompts
from tests.tiny_qwen2 import qwen2_config, qwen2_hf_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
# fp32 logit margin below which a bf16 implementation may pick the other candidate, for the tiny Qwen2 below: its
# logits spread wider than the tiny Llama's (std ~2.6 vs ~1.3 with 896 vs 256 hidden) and the eager bf16 HF model's own
# max logit error is ~0.3 (median over greedy positions, CPU) against ~0.07 for the tiny Llama (EPS = 0.35 there)
EPS_QWEN2 = 1.0


# ---------------------------------------------------------------------------------------------------------------
# tree attention at odd G = Hq / Hkv
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('Hq,Hkv,P,n,pad', [(28, 4, 384, 64, 0), (28, 4, 3900, 64, 0), (28, 4, 129, 1, 0),
                                             (7, 1, 0, 64, 0), (7, 1, 1000, 33, 5), (7, 1, 2500, 64, 0),
                                             (40, 8, 2500, 64, 0), (40, 8, 127, 33, 0), (3, 1, 37, 33, 0),
                                             (3, 1, 3968, 64, 7), (3, 1, 300, 1, 0)])
def test_tree_attention_odd_gqa(Hq, Hkv, P, n, pad):
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(P + n + Hq)
    torch.manual_seed(P * 7 + n + Hq)
    D, R, n_layers = 128, 64, 2
    max_seq = P + n + 70
    kc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    q = (torch.randn((R, Hq, D), device=DEV) * 0.7).to(torch.bfloat16)
    _, _, rows = _random_tree(rng, n)
    mask = _mask_tensor(rows, R)
    plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
    out = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    for layer in (1, 0):
        out.fill_(9.0)
        plan.forward(layer, q, mask, _slots([n], [P], [pad], R), out)
        torch.cuda.synchronize()
        ref = _ref_attention(q, kc[layer], vc[layer], rows, n, P, pad, Hq // Hkv)
        err = (out[:n].float() - ref).abs().max().item()
        attn_ref.assert_close(out[:n].float(), ref, f'layer {layer} max abs err {err}')
        assert float((out[n:].float() - 9.0).abs().sum()) == 0   # rows beyond the draft: untouched


@pytest.mark.parametrize('Hq,Hkv,rps,cases', [
    (28, 4, 64, [(64, 384, 0)]),
    (7, 1, 64, [(33, 0, 0)]),                                      # empty cache: the draft tile is the only tile
    (40, 8, 64, [(47, 1000, 5)]),                                  # ragged draft, left padding
    (3, 1, 64, [(1, 130, 0)]),                                     # a root-only draft right after a tile boundary
    (7, 1, 64, [(64, 3900, 0)]),
    (28, 4, 8, [(8, 300, 0), (3, 290, 0), (8, 310, 2), (1, 5, 0), (7, 128, 0), (8, 64, 0), (2, 500, 0), (6, 301, 0)])])
def test_fused_and_two_kernel_paths_odd_gqa(Hq, Hkv, rps, cases):
    """fused RoPE / KV-append / attention against pia_rope_kv_append + pia_tree_attn_fwd on the same inputs at odd G:
    the appended cache rows are bit identical (one writer per KV head), both outputs agree with the fp32 reference"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(Hq + rps)
    torch.manual_seed(Hq * 3 + rps)
    D, R, n_layers, B = 128, 64, 2, len(cases)
    max_seq = max(P + n for n, P, _ in cases) + 70
    kc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    qkv = torch.randn((R, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    inv = 1.0 / (1000000.0 ** (torch.arange(0, D, 2, device=DEV).float() / D))
    ang = torch.arange(max_seq + 8, device=DEV).float()[:, None] * inv[None]
    cos, sin = ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()
    mask = torch.zeros((R, 1), dtype=torch.int64, device=DEV)
    trees = []
    for s_, (n, P, pad) in enumerate(cases):
        rows = _random_tree(rng, n)[2]
        trees.append(rows)
        mask[s_ * rps:s_ * rps + n, 0] = torch.from_numpy(rows.view(np.int64)).to(DEV)
    ns, Ps, pads = [c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases]
    layer = 1
    k2, v2 = kc.clone(), vc.clone()
    plan, plan2 = ops.AttnPlan(kc, vc, Hq, Hkv, D, R), ops.AttnPlan(k2, v2, Hq, Hkv, D, R)
    sl = _slots(ns, Ps, pads, rps, stride=plan.slot_stride if B > 1 else 0)
    q = torch.zeros((R, Hq, D), dtype=torch.bfloat16, device=DEV)
    o1 = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    o2 = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    ops.rope_kv_append(qkv, mask, sl, Hq, Hkv, D, cos, sin, q, kc[0, layer], vc[0, layer], max_seq)
    plan.forward(layer, q, mask, sl, o1)
    plan2.forward_fused(layer, qkv, mask, sl, cos, sin, o2)
    torch.cuda.synchronize()
    assert torch.equal(k2, kc) and torch.equal(v2, vc)
    for s_, (n, P, pad) in enumerate(cases):
        r0 = s_ * rps
        ref = _ref_attention(q[r0:], kc[s_, layer], vc[s_, layer], trees[s_], n, P, pad, Hq // Hkv)
        attn_ref.assert_close(o1[r0:r0 + n].float(), ref, s_)
        attn_ref.assert_close(o2[r0:r0 + n].float(), ref, s_)
        assert torch.allclose(o2[r0:r0 + n].float(), o1[r0:r0 + n].float(), atol=4e-3, rtol=2e-2), s_
        assert float((o2[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0
        assert float((o1[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0


@pytest.mark.parametrize('Hq,Hkv,rps,cases', [
    (7, 1, 16, [(16, 100, 0), (5, 0, 0), (0, 7, 0), (9, 257, 3)]),
    (40, 8, 8, [(8, 300, 0), (3, 290, 0), (8, 310, 2), (1, 5, 0), (7, 128, 0), (8, 64, 0), (2, 500, 0), (6, 301, 0)])])
def test_batched_slots_odd_gqa(Hq, Hkv, rps, cases):
    """one launch over all request slots equals the per-slot launches (to the fp32 summation order of the KV splits)
    and the fp32 reference, at odd G"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(rps + Hq)
    torch.manual_seed(rps + Hq)
    D, R, n_layers, B = 128, 64, 2, len(cases)
    max_seq = max(P + n for n, P, _ in cases) + 70
    kc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    q = (torch.randn((R, Hq, D), device=DEV) * 0.7).to(torch.bfloat16)
    mask = torch.zeros((R, 1), dtype=torch.int64, device=DEV)
    trees = []
    for s_, (n, P, pad) in enumerate(cases):
        rows = _random_tree(rng, n)[2] if n else np.zeros((0,), dtype=np.uint64)
        trees.append(rows)
        if n:
            mask[s_ * rps:s_ * rps + n, 0] = torch.from_numpy(rows.view(np.int64)).to(DEV)
    ns, Ps, pads = [c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases]
    plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
    layer = 1
    ob = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    plan.forward(layer, q, mask, _slots(ns, Ps, pads, rps, stride=plan.slot_stride), ob)
    for s_, (n, P, pad) in enumerate(cases):
        r0 = s_ * rps
        o1 = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
        plan.forward(layer, q[r0:], mask[r0:], _slots([n], [P], [pad], rps, first=s_), o1)
        torch.cuda.synchronize()
        assert torch.allclose(ob[r0:r0 + n].float(), o1[:n].float(), atol=4e-3, rtol=2e-2)
        assert float((ob[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0
        if n:
            ref = _ref_attention(q[r0:], kc[s_, layer], vc[s_, layer], trees[s_], n, P, pad, Hq // Hkv)
            attn_ref.assert_close(ob[r0:r0 + n].float(), ref)


def _grid(Hq, Hkv, max_nodes):
    from painlessinferenceacceleration_b200.common import ops
    kc = torch.zeros((1, Hkv, 4096, 128), dtype=torch.bfloat16, device=DEV)
    plan = ops.AttnPlan(kc, kc.clone(), Hq, Hkv, 128, max_nodes)
    ns, ng = C.c_int(0), C.c_int(0)
    assert plan.lib.pia_attn_plan_grid(plan.h, C.byref(ns), C.byref(ng)) == 0
    return ns.value, ng.value


@pytest.mark.parametrize('Hq,Hkv,max_nodes,groups', [
    (28, 4, 64, 16), (7, 1, 64, 4), (40, 8, 64, 24), (3, 1, 64, 2),   # odd G: Hkv * ceil(G / 2)
    (32, 32, 64, 32), (32, 8, 64, 16), (4, 2, 64, 2),                 # MHA and even G: as before
    (32, 8, 128, 32), (28, 4, 128, 28), (7, 1, 128, 7)])              # 128 draft rows: one head per CTA
def test_attention_grid_packs_odd_groups(Hq, Hkv, max_nodes, groups):
    ns, ng = _grid(Hq, Hkv, max_nodes)
    assert ng == groups
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert ns == max(1, min(8, n_sm // groups))   # one wave of clusters (4096 / 128 = 32 tiles never limit it)


# ---------------------------------------------------------------------------------------------------------------
# the model: tiny Qwen2 with G = 7 and non-zero q/k/v biases
# ---------------------------------------------------------------------------------------------------------------
def _qwen2_pair(seed, **over):
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    hf = qwen2_hf_model(seed=seed, dtype=torch.bfloat16, device=DEV, vocab=200, **over)
    hf.fp32_twin = None
    ours = Qwen2ForCausalLM(hf.config, device=torch.device(DEV))
    res = ours.load_state_dict(hf.state_dict(), strict=False)
    assert not res.missing_keys, res
    return hf, ours


def _verify_logits(model, p):
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    return OursBackend(model).forward(p, m01, None)[0].float()


def test_qwen2_verify_logits_within_tolerance():
    """our bf16 forward (biased QKV addmm, G = 7 attention) vs an fp32 evaluation of the same weights: max |error| <=
    2 x the eager bf16 HF model's own error + 0.02, and the same greedy tokens wherever the fp32 margin is clear"""
    hf, ours = _qwen2_pair(seed=8)
    assert float(hf.model.layers[0].self_attn.k_proj.bias.detach().float().abs().max()) > 1.0   # the biases are really there
    hf32 = qwen2_hf_model(seed=8, dtype=torch.float32, device=DEV, vocab=200)
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


@pytest.mark.parametrize('penalty', [1.0, 1.1])
def test_qwen2_generate_matches_oracle(penalty):
    """generate() vs oracle/loop.py over the HF Qwen2: every divergence sits on a bf16 near-tie of the fp32 logits.
    Near-ties are about twice as frequent as on the tiny Llama (see EPS_QWEN2), so only a tenth of the tokens is
    required to precede the first one; equal text must come with equal drafts and accepted lengths"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, ours = _qwen2_pair(seed=2)
    # the fp32 evaluation _legit_divergence compares against (it builds one itself only for the tiny_models families)
    twin = qwen2_hf_model(seed=2, dtype=torch.float32, device=DEV, vocab=200)
    twin.load_state_dict({k: v.float() for k, v in hf.state_dict().items()})
    hf.fp32_twin = twin   # (attached after hf.state_dict() is read: it becomes a submodule of hf)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    exact = total = agree_tok = all_tok = 0
    for rep in range(2):
        for p in prompts(21, 4, 24, 200):
            p = p.to(DEV)
            out = ours.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                                decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                                return_dict_in_generate=True)
            ref = lookahead_generate(hf, otrie, p, max_new_tokens=48, eos_token_id=[2], repetition_penalty=penalty)
            a, b = out.sequences[0].tolist(), ref['sequences'][0].tolist()
            total += 1
            all_tok += len(b) - p.shape[1]
            if a == b:
                exact += 1
                agree_tok += len(b) - p.shape[1]
                assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls']
            else:
                k = next(i for i in range(min(len(a), len(b))) if a[i] != b[i])
                agree_tok += k - p.shape[1]
                ok, gap, noise = _legit_divergence('qwen2', hf, ref['sequences'][:, :k], a[k], b[k], penalty)
                assert ok, f'diverged at {k}: fp32 gap {gap:.3f} vs bf16 noise {noise:.3f}'
                assert gap < EPS_QWEN2, f'diverged at {k} although the fp32 top-2 margin is {gap:.3f} >= {EPS_QWEN2}'
                ours.lookahead_cache.fresh()
                otrie.fresh()
    assert agree_tok >= 0.1 * all_tok, f'only {agree_tok}/{all_tok} tokens precede the first bf16 near-tie ({exact}/{total} exact)'


@pytest.mark.parametrize('penalty', [1.0, 1.1])
def test_qwen2_loop_is_exact_given_the_same_logits(penalty):
    """the oracle loop drives one copy of our Qwen2 through the backend interface, the fused device loop the other:
    tokens, dls and edls identical for every request, tries carried across requests"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    hf, a = _qwen2_pair(seed=6)
    b = Qwen2ForCausalLM(hf.config, device=torch.device(DEV))
    b.load_state_dict(hf.state_dict(), strict=False)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 4, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=56, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=56, eos_token_id=[2], repetition_penalty=penalty,
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=90 + 56 + 65))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist()
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls']
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


@pytest.mark.parametrize('tied', [False, True])
def test_qwen2_from_pretrained(tmp_path, tied):
    """a save_pretrained directory (safetensors) loads into the same logits as the weights handed over directly; a
    tie_word_embeddings=True checkpoint ships no lm_head.weight and gets the embedding as its head"""
    from safetensors.torch import load_file
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    hf, direct = _qwen2_pair(seed=10, tie_word_embeddings=tied)
    hf.save_pretrained(str(tmp_path))
    saved = {}
    for f in tmp_path.glob('*.safetensors'):
        saved.update(load_file(str(f)))
    assert ('lm_head.weight' in saved) != tied
    assert 'model.layers.0.self_attn.k_proj.bias' in saved
    loaded = Qwen2ForCausalLM.from_pretrained(str(tmp_path), device=torch.device(DEV))
    assert torch.equal(loaded.lm_head.weight, hf.lm_head.weight)
    if tied:
        assert torch.equal(loaded.lm_head.weight, loaded.model.embed_tokens.weight)
    p = prompts(79, 1, 70, 200)[0].to(DEV)
    got, want = _verify_logits(loaded, p), _verify_logits(direct, p)
    assert torch.equal(got, want)
    # and the HF model's logits: within the tolerance of test_qwen2_verify_logits_within_tolerance of an fp32 evaluation
    hf32 = qwen2_hf_model(seed=10, dtype=torch.float32, device=DEV, vocab=200, tie_word_embeddings=tied)
    hf32.load_state_dict({k: v.float() for k, v in hf.state_dict().items()})
    with torch.no_grad():
        truth = hf32(input_ids=p).logits[0].float()
        eager = hf(input_ids=p).logits[0].float()
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)


def test_qwen2_sliding_window_warns_only_when_enabled():
    """use_sliding_window=True: the window is ignored on the lookahead path (as in the reference) and says so; a config
    that merely carries a sliding_window value (every Qwen2 config.json does) stays silent; the tokens are the same"""
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    hf = qwen2_hf_model(seed=3, dtype=torch.bfloat16, device=DEV, vocab=200)
    ids = prompts(5, 1, 24, 200)[0].to(DEV)
    kw = dict(input_ids=ids, max_new_tokens=12, eos_token_id=2,
              decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
    outs = []
    for use in (False, True):
        cfg = qwen2_config(vocab=200, use_sliding_window=use, sliding_window=16)
        ours = Qwen2ForCausalLM(cfg, device=torch.device(DEV))
        assert not ours.load_state_dict(hf.state_dict(), strict=False).missing_keys
        if use:
            with pytest.warns(UserWarning, match='sliding_window=16 is ignored'):
                outs.append(ours.generate(**kw))
        else:
            with warnings.catch_warnings(record=True) as rec:
                warnings.simplefilter('always')
                outs.append(ours.generate(**kw))
            assert not [w for w in rec if 'sliding_window' in str(w.message)]
    assert torch.equal(outs[0], outs[1])


def test_qwen2_gemm_set_qkv_raises(monkeypatch):
    """the weight-streaming GEMM has no bias epilogue: PIA_GEMM_SET=qkv must not silently drop the QKV bias"""
    hf, ours = _qwen2_pair(seed=4)
    monkeypatch.setenv('PIA_GEMM_SET', 'gate_up,qkv')
    with pytest.raises(ValueError, match='bias'):
        ours.generate(input_ids=prompts(6, 1, 16, 200)[0].to(DEV), max_new_tokens=8, eos_token_id=2,
                      decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})


# ---------------------------------------------------------------------------------------------------------------
# the real shape: Qwen2-7B (3584 hidden, 18944 inter, 28 / 4 heads, V = 152064, rope_theta 1e6)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.big
def test_qwen2_7b_loop_is_exact():
    """as test_loop_is_exact_at_baseline_shapes: the oracle loop drives one copy (all 28 layers), the fused device loop
    the other; 64-token / 8-branch drafts, 256-token phrase-bank prompts, two passes.  Tokens, dls and edls identical,
    and the second pass accepts drafts longer than 2"""
    import bench
    from transformers import Qwen2Config
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cfg = Qwen2Config(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                      num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=4096, rms_norm_eps=1e-6,
                      rope_theta=1000000.0, use_sliding_window=False, tie_word_embeddings=False,
                      bos_token_id=1, eos_token_id=2, pad_token_id=0)
    a = bench.synth_fill(Qwen2ForCausalLM(cfg, device=torch.device(DEV)), cfg)
    b = Qwen2ForCausalLM(cfg, device=torch.device(DEV))
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
