# -*- coding: utf-8 -*-
"""Qwen (v1) on the H100: pia_rope_f32_logn_kv_append bit for bit against a torch restatement, the lossless property of
the verify forward with dynamic NTK and log-n live (every draft node's logits = a causal forward over prefix +
root-to-node path at the request's alpha), and the tiny model (tests/tiny_qwen.py, seq_length 64) through generate(),
request-to-request alpha switches, forward(), checkpoint loading and fp8.  `big`: the Qwen-7B shape through the loop."""
import json

import numpy as np
import pytest
import torch

from tests.test_gpu_baichuan import _check, _sd
from tests.test_gpu_fp8 import _same_bytes
from tests.test_gpu_generate import OursBackend
from tests.test_gpu_head_dim64 import _mask, _tree
from tests.test_gpu_kernels import _slots
from tests.tiny_models import prompts
from tests.tiny_qwen import SEQ_LENGTH, causal_logits, model_class, ntk_alpha_ref, qwen_state_dict, tiny_config, \
    tiny_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


# ---------------------------------------------------------------------------------------------------------------
# the kernel: pia_rope_f32_logn_kv_append
# ---------------------------------------------------------------------------------------------------------------
def _tables(D, max_pos, S, alpha=1):
    from painlessinferenceacceleration_b200.models.qwen.modeling_qwen import logn_table, rope_tables_f32
    cos, sin = rope_tables_f32(D, 10000, alpha, max_pos)
    return cos.to(DEV), sin.to(DEV), logn_table(S, max_pos).to(DEV)


def _rope_logn(x, cos, sin, scale, pos, D):
    """apply_rotary_pos_emb (fp32, one cast to bf16, modeling_qwen.py:1231-1237), then query * logn_tensor in bf16"""
    c = torch.cat([cos[pos], cos[pos]], -1)[:, None, :]
    s = torch.cat([sin[pos], sin[pos]], -1)[:, None, :]
    xf = x.float()
    rot = torch.cat([-xf[..., D // 2:], xf[..., :D // 2]], -1)
    r = ((xf * c) + (rot * s)).to(torch.bfloat16)
    return r if scale is None else r * scale[pos][:, None, None]


def _run(qkv, mask, sl, Hq, Hkv, D, cos, sin, max_seq, B, scale):
    from painlessinferenceacceleration_b200.common import ops
    R = qkv.shape[0]
    kc = torch.full((B, Hkv, max_seq, D), 7.0, dtype=torch.bfloat16, device=DEV)
    vc = torch.full_like(kc, 7.0)
    q = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    ops.rope_kv_append(qkv, mask, sl, Hq, Hkv, D, cos, sin, q, kc[0], vc[0], max_seq, q_scale=scale)
    torch.cuda.synchronize()
    return q, kc, vc


def _deep_tree(rng, n):
    """ancestor rows of a tree of n nodes whose first 3n/4 form one chain, the rest hanging off random chain nodes,
    so that its depths span most of 0 .. n - 1"""
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


# (Hq, Hkv, D, R, S, slots [(n, P, pad)]): drafts straddling seq_length, left padding, several slots
KERNEL_CASES = [(32, 32, 128, 64, 64, [(64, 40, 0)]), (8, 2, 128, 64, 2048, [(64, 2080, 5)]),
                (4, 4, 64, 64, 64, [(64, 40, 3)]), (8, 2, 64, 128, 64, [(128, 30, 0)]),
                (4, 4, 128, 128, 512, [(100, 480, 7)]), (6, 2, 128, 64, 64, [(16, 50, 2), (5, 0, 0), (0, 7, 0), (9, 300, 0)]),
                (4, 1, 64, 128, 64, [(32, 60, 0), (20, 200, 4), (32, 10, 0), (1, 70, 0)])]


@pytest.mark.parametrize('Hq,Hkv,D,R,S,cases', KERNEL_CASES)
def test_rope_logn_bit_exact(Hq, Hkv, D, R, S, cases):
    """q bit for bit against the restatement at the tree positions; K / V equal pia_rope_f32_kv_append's; q rows before
    seq_length equal the plain entry's, rows whose scale is not 1 differ"""
    rng = np.random.default_rng(Hq + D + R + S)
    torch.manual_seed(Hq * D + R + S)
    B = len(cases)
    rps = R // B if B > 1 else R
    trees = [_deep_tree(rng, n) for n, _, _ in cases]
    max_seq = max(P + n for n, P, _ in cases) + 40
    cos, sin, scale = _tables(D, max_seq + 8, S, alpha=3)
    qkv = (torch.randn((B * rps, (Hq + 2 * Hkv) * D), device=DEV) * 2).to(torch.bfloat16)
    mask = _mask(trees, R, rps)
    stride = Hkv * max_seq * D
    sl = _slots([n for n, _, _ in cases], [P for _, P, _ in cases], [p for _, _, p in cases], rps, stride=stride)
    q, kc, vc = _run(qkv, mask, sl, Hq, Hkv, D, cos, sin, max_seq, B, scale)
    q0, kc0, vc0 = _run(qkv, mask, sl, Hq, Hkv, D, cos, sin, max_seq, B, None)
    assert torch.equal(kc, kc0) and torch.equal(vc, vc0)
    seen_scaled = seen_plain = 0
    for s_, ((n, P, pad), rows) in enumerate(zip(cases, trees)):
        r0 = s_ * rps
        assert (q[r0 + n:r0 + rps].float() == 9.0).all()
        if not n:
            continue
        depth = torch.tensor([bin(r).count('1') - 1 for r in rows], device=DEV)
        pos = max(P - pad, 0) + depth
        x = qkv[r0:r0 + n].view(n, Hq + 2 * Hkv, D)
        assert torch.equal(q[r0:r0 + n], _rope_logn(x[:, :Hq], cos, sin, scale, pos, D))
        assert torch.equal(q0[r0:r0 + n], _rope_logn(x[:, :Hq], cos, sin, None, pos, D))
        k_want = _rope_logn(x[:, Hq:Hq + Hkv], cos, sin, None, pos, D).transpose(0, 1)
        assert torch.equal(kc[s_, :, P:P + n], k_want) and torch.equal(vc[s_, :, P:P + n],
                                                                       x[:, Hq + Hkv:].transpose(0, 1))
        one = scale[pos] == 1
        assert torch.equal(q[r0:r0 + n][one], q0[r0:r0 + n][one])
        for i in torch.nonzero(~one).flatten().tolist():
            assert not torch.equal(q[r0 + i], q0[r0 + i]), (s_, i)
        seen_scaled += int((~one).sum())
        seen_plain += int(one.sum())
    assert seen_scaled > 0 and seen_plain > 0   # rows on both sides of seq_length


def test_rope_logn_argument_checks():
    from painlessinferenceacceleration_b200.common import ops
    D, R = 128, 64
    cos, sin, scale = _tables(D, 200, 64)
    qkv = torch.zeros((R, 3 * D), dtype=torch.bfloat16, device=DEV)
    kc = torch.zeros((1, 192, D), dtype=torch.bfloat16, device=DEV)
    q = torch.zeros((R, 1, D), dtype=torch.bfloat16, device=DEV)
    args = (qkv, _mask([[1]], R, R), _slots([1], [0], [0], R), 1, 1, D)
    with pytest.raises(ValueError, match='q_scale'):
        ops.rope_kv_append(*args, cos, sin, q, kc, kc.clone(), 192, q_scale=scale[:100])
    with pytest.raises(ValueError, match='fp32'):
        ops.rope_kv_append(*args, cos.to(torch.bfloat16), sin.to(torch.bfloat16), q, kc, kc.clone(), 192,
                           q_scale=scale)


# ---------------------------------------------------------------------------------------------------------------
# lossless: the verify logits of every draft node = a causal forward over prefix + root-to-node path
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('T0', [40, 100, 300])
def test_tree_verify_logits_are_lossless(T0):
    """prompt of T0 tokens (below seq_length: alpha 1; above: alpha 3 / 7, log-n live on every row), then one random
    64-node tree; each node's verify-logit row vs the fp32 causal forward over prompt + its root-to-node path, within
    2 x the bf16 eager restatement's own error + 0.02"""
    model = tiny_model(seed=3)
    cfg = tiny_config()
    sd = _sd(model)
    alpha = ntk_alpha_ref(T0, SEQ_LENGTH)
    torch.manual_seed(4 + T0)
    n = 64
    prompt = torch.randint(3, 200, (1, T0), device=DEV)
    rows = _tree(np.random.default_rng(5), n, max_depth=10)
    ids = torch.randint(3, 200, (1, n), device=DEV)
    rt = model._runtime(T0 + n + 70, 64)
    model._start_request(rt, T0)
    assert rt.ntk_alpha == alpha
    be = OursBackend(model, prefill_like_generate=True, max_seq=T0 + n + 70)
    be.forward(prompt, None, None)
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
        truth = causal_logits(sd, cfg, seq, alpha)[-1]
        eager = causal_logits(sd, cfg, seq, alpha, dtype=torch.bfloat16)[-1]
        _check(got[i], truth, eager)
    if alpha > 1:   # the alpha matters: alpha 1's forward is further from the truth than ours
        wrong = causal_logits(sd, cfg, torch.cat([prompt[0], ids[0, :1]]), 1)[-1]
        truth = causal_logits(sd, cfg, torch.cat([prompt[0], ids[0, :1]]), alpha)[-1]
        assert (wrong - truth).abs().max().item() > 2 * (got[0] - truth).abs().max().item()


def test_forward_without_past_sets_alpha():
    """forward() with no past is a prefill: it fixes alpha from its input length, and the logits are the causal
    forward's at that alpha"""
    model = tiny_model(seed=6)
    sd, cfg = _sd(model), tiny_config()
    for T, alpha in ((100, 3), (30, 1), (65, 3), (64, 1)):
        p = prompts(T, 1, T, 200)[0].to(DEV)
        m01 = torch.tril(torch.ones((1, 1, T, T), dtype=torch.long, device=DEV))
        lg, past = model.forward(p, m01)
        assert model._rt.ntk_alpha == alpha and past == T
        truth = causal_logits(sd, cfg, p[0], alpha)[-1]
        eager = causal_logits(sd, cfg, p[0], alpha, dtype=torch.bfloat16)[-1]
        _check(lg[0, -1].float(), truth, eager)


# ---------------------------------------------------------------------------------------------------------------
# the tiny model through generate()
# ---------------------------------------------------------------------------------------------------------------
def _cache(model):
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    model.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    return model


DK = {'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8}


@pytest.mark.parametrize('penalty', [1.0, 1.1])
def test_generate_equals_plain_greedy(penalty):
    """lookahead generate() gives the tokens of plain greedy decoding with the same kernels, for prompts below and
    above seq_length, and a second pass accepts drafts"""
    model = _cache(tiny_model(seed=1))
    edls = []
    for rep in range(2):
        for T in (40, 90, 200):
            p = prompts(21 + T, 1, T, 200)[0].to(DEV)
            g = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               decoding_kwargs={'use_lookahead': False})
            o = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                               return_dict_in_generate=True, decoding_kwargs=dict(DK))
            assert o.sequences[0].tolist() == g[0].tolist(), (T, rep)
            assert model._rt.ntk_alpha == ntk_alpha_ref(T, SEQ_LENGTH)
            edls += o.kwargs['edls'][1:]
    assert max(edls) > 2


def test_short_long_short_requests_match_fresh_models():
    """one model and runtime serve short -> long -> short -> long prompts (alpha 1, 7, 1, 3): every output equals that
    of a fresh model given the request alone, so no captured graph keeps a stale table"""
    shared = _cache(tiny_model(seed=9))
    rt = shared._runtime(1024, 64)
    for T in (30, 150, 20, 100):
        p = prompts(T, 1, T, 200)[0].to(DEV)
        got = shared.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs=dict(DK))
        assert shared._rt is rt and rt.ntk_alpha == ntk_alpha_ref(T, SEQ_LENGTH)
        fresh = _cache(tiny_model(seed=9))
        fresh._runtime(1024, 64)
        want = fresh.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs=dict(DK))
        assert got[0].tolist() == want[0].tolist(), T
        del fresh
    assert len(rt.graphs) >= 1 and len(rt.prefill_graphs) >= 1   # the captured graphs were reused across requests


def test_max_length_past_the_logn_table_is_refused():
    model = tiny_model(seed=2)
    p = prompts(3, 1, 10, 200)[0].to(DEV)
    with pytest.raises(ValueError, match='32767'):
        model.generate(input_ids=p, max_length=32768, eos_token_id=2, decoding_kwargs=dict(DK))


class _QwenBackend(OursBackend):
    """the oracle loop's backend with the request start generate() makes: the prompt fixes the NTK alpha"""

    def forward(self, ids_in, m01, pos):
        if self.P == 0:
            self.m._start_request(self.m._runtime(self.max_seq, 64), ids_in.shape[1])
        return super().forward(ids_in, m01, pos)


@pytest.mark.parametrize('penalty', [1.0, 1.1])
def test_loop_is_exact_given_the_same_logits(penalty):
    """the oracle loop drives one copy of our model, the fused device loop another: tokens, dls, edls identical"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    a = _cache(tiny_model(seed=6))
    b = tiny_model(seed=6)
    otrie = OracleLookaheadCache(eos_ids=[2])
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 3, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=56, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs=dict(DK), return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=56, eos_token_id=[2], repetition_penalty=penalty,
                                     decoding_length=64,
                                     backend=_QwenBackend(b, prefill_like_generate=True, max_seq=90 + 56 + 129))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), rep
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], rep
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def _write_checkpoint(model, path):
    """a Qwen-format directory: config.json, transformer.h.* names with c_attn weight and bias, two safetensors
    shards"""
    from safetensors.torch import save_file
    path.mkdir(parents=True, exist_ok=True)
    (path / 'config.json').write_text(json.dumps(tiny_config()))
    sd = {k: v.detach().cpu().contiguous() for k, v in qwen_state_dict(model.state_dict()).items()}
    sd['transformer.rotary_emb.inv_freq'] = torch.ones(64)
    keys = sorted(sd)
    save_file({k: sd[k] for k in keys[:len(keys) // 2]}, str(path / 'model-00001-of-00002.safetensors'))
    save_file({k: sd[k] for k in keys[len(keys) // 2:]}, str(path / 'model-00002-of-00002.safetensors'))


def _verify_logits(model, p):
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    return model.forward(p, m01)[0][0].float()


def test_from_pretrained_bf16_and_fp8(tmp_path):
    """a Qwen-format checkpoint loads into the logits of the same weights handed over directly; quantization='fp8'
    gives quantize_fp8()'s bytes with bf16 QKV biases, its logits are within the bf16 rule of an fp32 forward of the
    dequantised weights, and generate() runs"""
    direct = tiny_model(seed=10)
    _write_checkpoint(direct, tmp_path)
    cls = model_class()
    loaded = cls.from_pretrained(str(tmp_path), device=torch.device(DEV))
    p = prompts(79, 1, 100, 200)[0].to(DEV)
    assert torch.equal(_verify_logits(loaded, p), _verify_logits(direct, p))
    ref = tiny_model(seed=10)
    ref.quantize_fp8()
    got = cls.from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')
    _same_bytes(ref, got)
    a = got.model.layers[0].self_attn
    assert a.qkv_bias.dtype == torch.bfloat16 and torch.equal(a.qkv_bias, ref.model.layers[0].self_attn.qkv_bias)
    sd, cfg = _sd(direct), tiny_config()
    for i, layer in enumerate(got.model.layers):
        pre = f'model.layers.{i}.'
        for n in ('q_proj', 'k_proj', 'v_proj', 'o_proj'):
            sd[pre + f'self_attn.{n}.weight'] = getattr(layer.self_attn, n).dequantize()
        for n in ('gate_proj', 'up_proj', 'down_proj'):
            sd[pre + f'mlp.{n}.weight'] = getattr(layer.mlp, n).dequantize()
    alpha = ntk_alpha_ref(100, SEQ_LENGTH)
    _check(_verify_logits(got, p)[-1], causal_logits(sd, cfg, p[0], alpha)[-1],
           causal_logits(sd, cfg, p[0], alpha, dtype=torch.bfloat16)[-1])
    _cache(got)
    out = got.generate(input_ids=p, max_new_tokens=24, eos_token_id=2, return_dict_in_generate=True,
                       decoding_kwargs=dict(DK))
    assert sum(out.kwargs['edls']) == out.sequences.shape[1] - 100


def test_fused_attention_knob_is_refused(monkeypatch):
    model = tiny_model(seed=4)
    monkeypatch.setenv('PIA_ATTN_FUSED', '1')
    with pytest.raises(ValueError, match='PIA_ATTN_FUSED'):
        model.generate(input_ids=prompts(6, 1, 16, 200)[0].to(DEV), max_new_tokens=8, eos_token_id=2,
                       decoding_kwargs=dict(DK))
    assert model._rt is None


# ---------------------------------------------------------------------------------------------------------------
# the real shape: Qwen-7B (32 layers, 4096, 32 x 128 MHA, 11008 per branch, V = 151936, c_attn bias)
# ---------------------------------------------------------------------------------------------------------------
def qwen_7b_config(seq_length=8192):
    return dict(model_type='qwen', vocab_size=151936, hidden_size=4096, intermediate_size=22016,
                num_hidden_layers=32, num_attention_heads=32, kv_channels=128, layer_norm_epsilon=1e-6,
                rotary_emb_base=10000, rotary_pct=1.0, seq_length=seq_length, max_position_embeddings=32768,
                use_dynamic_ntk=True, use_logn_attn=True, no_bias=True, tie_word_embeddings=False)


@pytest.mark.big
def test_qwen_7b_loop_is_exact():
    """bench.synth_fill weights, seq_length 128 below the 256-token phrase-bank prompts (alpha 3, log-n live): the
    oracle loop drives one copy, the fused device loop the other; tokens, dls, edls identical over two passes"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.qwen.modeling_qwen import qwen_config
    cfg = qwen_config(qwen_7b_config(seq_length=128))
    cls = model_class()
    a = bench.synth_fill(cls(cfg, device=torch.device(DEV)), cfg)
    b = cls(cfg, device=torch.device(DEV))
    b.load_state_dict(a.state_dict(), strict=True)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=cfg.vocab_size)
    otrie = OracleLookaheadCache(eos_ids=[2])
    new = 96
    edl_all = []
    for rep in range(2):
        for p in bench.phrase_bank_prompts(2, cfg.vocab_size):
            p = torch.tensor([p], device=DEV)
            out = a.generate(input_ids=p, max_new_tokens=new, eos_token_id=2, decoding_kwargs=dict(DK),
                             return_dict_in_generate=True)
            assert a._rt.ntk_alpha == ntk_alpha_ref(p.shape[1], 128) > 1
            ref = lookahead_generate(None, otrie, p, max_new_tokens=new, eos_token_id=[2],
                                     backend=_QwenBackend(b, prefill_like_generate=True, max_seq=256 + new + 65))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), rep
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], rep
            if rep == 1:
                edl_all += ref['edls'][1:]
    assert max(edl_all) > 2
