# -*- coding: utf-8 -*-
"""Int4 (GPTQ / compressed-tensors W4A16) weights on the H100: the int4 weight-streaming GEMM (k_gemm_w4) against the
dequantisation formula bit for bit, an fp64 reference and k_gemm_ws on the dequantised weight, and the int4 checkpoints
of tests/w4_ckpt.py end to end - verify logits against the eager transformers model of each checkpoint
(tests/golden/w4_logits.npz), loop exactness against the oracle loop, the lossless property, the batched loop, and
GPTQ against compressed-tensors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import gemm_ref, w4_ckpt
from tests.test_gpu_generate import EPS, OursBackend
from tests.tiny_models import prompts

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'w4_logits.npz'))


def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


def _plan(u, s, z, gs, x, **kw):
    ops = _ops()
    return ops.Gemm.w4(ops.tile_weight_w4(u), s.t().contiguous(), z.t().contiguous(), gs, x, **kw)


# ------------------------------------------------------------------------------------------------ the GEMM
@pytest.mark.parametrize('sdt', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('K', [512, 384])
def test_w4_exact_dequantisation(sdt, K):
    """every (u, z) pair (u 0..15, z 0..16) under power-of-two and ordinary scales, X one-hot rows: each output is one
    weight, which must equal bf16(dtype_s(s * (u - z))) bit for bit (zeros by value: the accumulator starts at +0).
    K = 384 ends in a half (128-k) chunk."""
    ops = _ops()
    N, gs = 256, 128
    G = K // gs
    n, k = torch.arange(N)[:, None], torch.arange(K)[None, :]
    u = ((k + n // 17) % 16).to(torch.uint8)
    z = ((torch.arange(N)[:, None] + 5 * torch.arange(G)[None, :]) % 17).to(torch.uint8)
    gen = torch.Generator().manual_seed(K)
    pow2 = torch.pow(2.0, (torch.arange(N * G) % 9 - 6).float()).view(N, G)
    ordinary = 1e-3 + 0.05 * torch.rand((N, G), generator=gen)
    s = torch.where(torch.arange(N)[:, None] % 2 == 0, pow2, ordinary).to(sdt)
    want = ops.dequantize_w4(u, s, z, gs)
    ref = (u.to(sdt) - z.repeat_interleave(gs, 1).to(sdt)) * s.repeat_interleave(gs, 1)
    assert torch.equal(want, ref.to(torch.bfloat16))
    x = torch.eye(K, dtype=torch.bfloat16, device=DEV)
    out = _plan(u.to(DEV), s.to(DEV), z.to(DEV), gs, x).run(K).cpu()   # out[k, n] = W[n, k]
    w = want.t()
    nz = w != 0
    assert torch.equal(out.view(torch.int16)[nz], w.view(torch.int16)[nz])
    assert (out[~nz] == 0).all()


def _codes(N, K, gs, seed, sdt=torch.bfloat16, sym=False):
    return w4_ckpt.random_codes(N, K, gs, sym, sdt, torch.Generator().manual_seed(seed))


# (name, N, K, group, bias, split modes): Llama-2-7B, Llama-3-8B, Qwen2-7B (biased qkv), Qwen2.5-0.5B (K = 896 ends in a
# half chunk)
SHAPES = [('llama2_qkv', 12288, 4096, 128, False, (1, -2)), ('llama2_o', 4096, 4096, 128, False, (1, -4, 4)),
          ('llama2_gate_up', 22016, 4096, 128, False, (1,)), ('llama2_down', 4096, 11008, 128, False, (1, -4, 4)),
          ('llama3_qkv', 6144, 4096, 128, False, (1, -2)), ('llama3_gate_up', 28672, 4096, 128, False, (1,)),
          ('llama3_down', 4096, 14336, 128, False, (-4, 8)),
          ('qwen2_qkv', 4608, 3584, 128, True, (1, -4)), ('qwen2_down', 3584, 18944, 128, False, (-4, -8)),
          ('qwen25_qkv', 1152, 896, 128, True, (1, -2)), ('qwen25_down', 896, 4864, 128, False, (1, -4))]
ROWS = (1, 5, 64, 128, 256)


@pytest.mark.parametrize('name,N,K,gs,biased,splits', SHAPES)
def test_w4_gemm_against_fp64(name, N, K, gs, biased, splits):
    """out = bf16(X @ W^T (+ bias)) of the dequantised weight against fp64 with tests/gemm_ref.py's comparator, for
    1..256 rows and every split mode; two runs bit-identical; rows beyond `rows` untouched"""
    u, s, z = _codes(N, K, gs, seed=N + K)
    w = _ops().dequantize_w4(u, s, z, gs).to(DEV)
    u, s, z = u.to(DEV), s.to(DEV), z.to(DEV)
    x = torch.randn((256, K), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV).to(torch.bfloat16)
    bias = (torch.randn(N, device=DEV) * 2).to(torch.bfloat16).float() if biased else None
    ref, mass = gemm_ref.reference(x, w, None, bias)
    for sk in splits:
        g = _plan(u, s, z, gs, x, bias=bias, split_k=sk)
        for rows in ROWS:
            g.out.fill_(7.0)
            o1 = g.run(rows).clone()
            o2 = g.run(rows).clone()
            assert torch.equal(o1, o2), (name, sk, rows)
            if g.splits > 1:
                assert (o1[:, rows:] == 7.0).all()
                got = o1[0, :rows].clone()
                for i in range(1, g.splits):
                    got += o1[i, :rows]
                got = got.to(torch.bfloat16)
            else:
                assert (o1[rows:] == 7.0).all(), (name, sk, rows)
                got = o1[:rows]
            gemm_ref.assert_close(got, ref[:rows], mass[:rows], K, g.splits if sk > 0 else -sk,
                                  f'{name} split {sk} rows {rows}')


@pytest.mark.parametrize('N,K,sdt', [(4096, 4096, torch.bfloat16), (1152, 896, torch.float16),
                                     (11008, 4096, torch.float16)])
def test_w4_equals_k_gemm_ws_on_the_dequantised_weight(N, K, sdt):
    """split 1: k_gemm_w4 == k_gemm_ws on the dequantised bf16 weight, bit for bit (same bf16 operands, same wgmma
    shape, same k order); a wrong A fragment shows here first"""
    ops = _ops()
    u, s, z = _codes(N, K, 128, seed=3, sdt=sdt)
    w = ops.dequantize_w4(u, s, z, 128).to(DEV)
    x = torch.randn((64, K), generator=torch.Generator(device=DEV).manual_seed(2), device=DEV).to(torch.bfloat16)
    ws = ops.Gemm(ops.tile_weight(w), x, tiled=True)
    w4 = _plan(u.to(DEV), s.to(DEV), z.to(DEV), 128, x)
    for rows in (1, 17, 64):
        assert torch.equal(w4.run(rows)[:rows], ws.run(rows)[:rows]), rows


@pytest.mark.parametrize('rows', [5, 64, 200])
def test_w4_silu_epilogue_equals_gate_up_then_silu_mul(rows):
    """the fused SiLU*up epilogue on the interleaved int4 gate/up weight == the plain int4 GEMM + pia_silu_mul"""
    ops = _ops()
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import _gate_up_order
    H, I = 4096, 11008
    u, s, z = (_gate_up_order(t) for t in _codes(2 * I, H, 128, seed=5))
    u, s, z = u.to(DEV), s.to(DEV), z.to(DEV)
    x = torch.randn((256, H), generator=torch.Generator(device=DEV).manual_seed(5), device=DEV).to(torch.bfloat16)
    act = torch.full((256, I), 7.0, dtype=torch.bfloat16, device=DEV)
    _plan(u, s, z, 128, x, out=act).set_silu().run(rows)
    assert (act[rows:] == 7.0).all()
    gu_int = _plan(u, s, z, 128, x).run(rows)[:rows]
    gu = _gate_up_order(gu_int.t(), inverse=True).t().contiguous()
    ref = torch.empty((rows, I), dtype=torch.bfloat16, device=DEV)
    ops.silu_mul(gu, ref)
    assert torch.equal(act[:rows], ref)


def test_w4_plan_refusals():
    """PIA_ERR_INVALID (AssertionError) before any launch: N or K not a multiple of 128, a group that is not a multiple
    of 128, ReLU"""
    from painlessinferenceacceleration_b200 import _lib as L
    ops = _ops()
    x = torch.zeros((64, 256), dtype=torch.bfloat16, device=DEV)
    codes = torch.zeros((1, 1, 128, 128), dtype=torch.uint8, device=DEV)
    s, z = torch.ones((4, 256), dtype=torch.bfloat16, device=DEV), torch.zeros((4, 256), dtype=torch.uint8, device=DEV)
    lib = L.load()
    before = ops.launch_count()
    for N, K, gs in ((192, 256, 128), (256, 192, 64), (256, 256, 64), (256, 256, 96)):
        h = L.vp()
        rc = lib.pia_gemm_plan_create_w4(codes.data_ptr(), s.data_ptr(), z.data_ptr(), 0, None, N, K, gs, x.data_ptr(),
                                         64, 1, ctypes.byref(h))
        assert rc == L.PIA_ERR_INVALID, (N, K, gs)
    g = ops.Gemm.w4(torch.zeros((2, 1, 128, 128), dtype=torch.uint8, device=DEV), s[:2].contiguous(),
                    z[:2].contiguous(), 128, x)
    with pytest.raises(AssertionError, match='ReLU'):
        g.set_relu()
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------ models
def _cls(family):
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.mistral.modeling_mistral import MistralForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    return {'llama': LlamaForCausalLM, 'mistral': MistralForCausalLM, 'qwen2': Qwen2ForCausalLM}[family]


def _load(name, tmp_path, cls=None):
    d = tmp_path / name
    w4_ckpt.write(name, str(d))
    return (cls or _cls(w4_ckpt.FIXTURES[name][0])).from_pretrained(str(d), device=torch.device(DEV))


CT = [n for n, f in w4_ckpt.FIXTURES.items() if f[1] == 'compressed-tensors']


@pytest.mark.parametrize('name', CT)
def test_w4_verify_logits_against_the_eager_model(name, tmp_path):
    """verify logits vs the eager transformers model of the same checkpoint (fp32): max |error| <= 2 x the eager bf16
    model's error + 0.02; the loaded weights are the checkpoint's codes"""
    m = _load(name, tmp_path)
    assert m._w4
    _, _, codes = w4_ckpt.build(name)
    layer = m.model.layers[1]
    u, s, z = codes['model.layers.1.mlp.up_proj']
    got = layer.mlp.up_proj.codes()
    assert torch.equal(got[0].cpu(), u) and torch.equal(got[1].cpu(), s) and torch.equal(got[2].cpu(), z)
    p = w4_ckpt.prompt(name).to(DEV)
    T = p.shape[1]
    m01 = torch.tril(torch.ones((1, 1, T, T), dtype=torch.long, device=DEV))
    ours = OursBackend(m).forward(p, m01, None)[0].float().cpu()
    truth, eager = torch.from_numpy(GOLDEN[name + '/fp32']), torch.from_numpy(GOLDEN[name + '/bf16'])
    e_ours, e_eager = (ours - truth).abs().max().item(), (eager - truth).abs().max().item()
    print(f'int4 verify logits {name}: err vs eager fp32 {e_ours:.4f}, eager bf16 {e_eager:.4f}')
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)


def test_w4_gptq_and_compressed_tensors_give_identical_logits(tmp_path):
    """the GPTQ v1 checkpoint and the compressed-tensors checkpoint of the same codes load to identical bytes and give
    identical verify logits"""
    a = _load('llama_ct_asym_g128_fp16', tmp_path)
    b = _load('llama_gptq_asym_g128_fp16', tmp_path)
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert sorted(pa) == sorted(pb)
    for k in pa:
        assert torch.equal(pa[k].view(-1).view(torch.uint8), pb[k].view(-1).view(torch.uint8)), k
    p = w4_ckpt.prompt('llama_ct_asym_g128_fp16').to(DEV)
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    assert torch.equal(OursBackend(a).forward(p, m01, None), OursBackend(b).forward(p, m01, None))


@pytest.mark.parametrize('name,penalty', [('llama_ct_sym_g128_bf16', 1.0), ('mistral_ct_asym_g128_bf16', 1.1),
                                          ('qwen2_ct_asym_g128_fp16', 1.0)])
def test_w4_loop_is_exact_given_the_same_logits(name, penalty, tmp_path):
    """the oracle loop drives one int4 copy through OursBackend, the fused device loop another: tokens, dls and edls
    identical for every request, tries carried across requests"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    a, b = _load(name, tmp_path / 'a'), _load(name, tmp_path / 'b')
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 3, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=48, eos_token_id=[2], repetition_penalty=penalty,
                                     decoding_length=64,
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=90 + 48 + 129))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (name, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (name, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def test_w4_lookahead_equals_own_greedy(tmp_path):
    """lossless: drafts never change the int4 model's output (up to near-ties), at 64 and 128 draft nodes"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    m = _load('qwen2_ct_sym_g128_bf16', tmp_path)
    m.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    same = total = 0
    for dl in (64, 128):
        for p in prompts(33, 4, 16, 200):
            p = p.to(DEV)
            g = m.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
            for _ in range(2):
                o = m.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, return_dict_in_generate=True,
                               decoding_kwargs={'use_lookahead': True, 'decoding_length': dl, 'branch_length': 8})
            assert sum(o.kwargs['edls']) == o.sequences.shape[1] - 16
            total += 1
            if o.sequences[0].tolist() == g[0].tolist():
                same += 1
                assert max(o.kwargs['edls']) > 1
    assert same >= total - 2, (same, total)


def test_w4_batched_loop_matches_single_request_loop(tmp_path):
    """the batched Llama class (bs = 3) on the same int4 checkpoint: every request equals the single-request loop,
    except where they part on a near-tie of the model's own logits"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.llama.modeling_llama_batch import LlamaForCausalLM as Batched
    single = _load('llama_ct_sym_g128_bf16', tmp_path / 's')
    batched = _load('llama_ct_sym_g128_bf16', tmp_path / 'b', cls=Batched)
    ps = torch.cat([p for p in prompts(61, 3, 20, 200)], dim=0).to(DEV)
    dk = {'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8}
    batched.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    single.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    outb = batched.generate(input_ids=ps, max_new_tokens=32, eos_token_id=2, decoding_kwargs=dict(dk))
    outb = outb.sequences if hasattr(outb, 'sequences') else outb
    for i in range(3):
        s = single.generate(input_ids=ps[i:i + 1], max_new_tokens=32, eos_token_id=2, decoding_kwargs=dict(dk))[0].tolist()
        bt = outb[i].tolist()[:len(s)]
        if bt == s:
            continue
        k = next(j for j in range(min(len(bt), len(s))) if bt[j] != s[j])
        m01 = torch.tril(torch.ones((1, 1, k, k), dtype=torch.long, device=DEV))
        lg = single.forward(torch.tensor([s[:k]], device=DEV), m01)[0][0, -1].float()
        top = torch.topk(lg, 2).values
        assert (top[0] - top[1]).item() < EPS, (i, k)


def test_w4_gemm_knobs_and_fp8_are_refused(tmp_path, monkeypatch):
    """int4 weights have no other GEMM: PIA_GEMM=0 / PIA_GEMM_SET raise ValueError, so do quantize_fp8() and
    quantization='fp8' on an int4 checkpoint"""
    m = _load('llama_ct_sym_g128_bf16', tmp_path)
    with pytest.raises(ValueError, match='int4'):
        m.quantize_fp8()
    with pytest.raises(ValueError, match='already quantised'):
        type(m).from_pretrained(str(tmp_path / 'llama_ct_sym_g128_bf16'), device=torch.device(DEV), quantization='fp8')
    for i, env in enumerate(({'PIA_GEMM': '0'}, {'PIA_GEMM_SET': 'gate_up'})):
        m = _load('llama_ct_sym_g128_bf16', tmp_path / str(i))
        p = prompts(3, 1, 16, 200)[0].to(DEV)
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            with pytest.raises(ValueError, match='int4'):
                m.generate(input_ids=p, max_new_tokens=4, eos_token_id=2, decoding_kwargs={'use_lookahead': False})


# ------------------------------------------------------------------------------------------------ big
def synth_w4(cls, cfg, seed=0, group_size=128):
    """bench.synth_fill for the bf16 parameters, seeded random codes (tests/w4_ckpt.py) for every projection, built
    layer by layer on the GPU"""
    import zlib
    import bench

    def fill(name, shape):
        g = torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()) ^ (seed * 7919))
        N, K = shape
        u = torch.randint(0, 16, (N, K), generator=g, device=DEV, dtype=torch.uint8)
        s = ((0.5 + torch.rand((N, K // group_size), generator=g, device=DEV)) * 0.02 / 8).to(torch.bfloat16)
        z = torch.full((N, K // group_size), 8, dtype=torch.uint8, device=DEV)
        return u, s, z, group_size
    return cls.build_w4(cfg, lambda m: bench.synth_fill(m, cfg, seed), fill, device=torch.device(DEV))


@pytest.mark.big
def test_w4_loop_is_exact_at_llama2_7b_shape():
    """Llama-2-7B shape, all 32 layers, int4 group 128: the oracle loop through one copy, the device loop another"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg, _ = bench.make_config('llama2-7b')
    a, b = synth_w4(LlamaForCausalLM, cfg), synth_w4(LlamaForCausalLM, cfg)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=cfg.vocab_size)
    otrie = OracleLookaheadCache(eos_ids=[2])
    ps = bench.phrase_bank_prompts(3, cfg.vocab_size)
    edl_all = []
    for rep in range(2):
        for p in ps:
            p = torch.tensor([p], device=DEV)
            out = a.generate(input_ids=p, max_new_tokens=96, eos_token_id=2, return_dict_in_generate=True,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
            ref = lookahead_generate(None, otrie, p, max_new_tokens=96, eos_token_id=[2],
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=256 + 96 + 65))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), rep
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], rep
            if rep == 1:
                edl_all += ref['edls'][1:]
    assert max(edl_all) > 2
