# -*- coding: utf-8 -*-
"""Int4 (GPTQ / compressed-tensors W4A16) Mixtral on the H100: the grouped int4 GEMM (k_gemm_w4 with one expert per
group) against fp64 at Mixtral-8x7B down shapes and bit for bit against separate per-expert int4 launches and the bf16
grouped GEMM on the dequantised stack, the stacked gate_up + SiLU launch against per-expert gate_up + silu_mul, and the
int4 Mixtral checkpoints of tests/w4_moe_ckpt.py end to end - verify logits against the eager transformers model of each
checkpoint (tests/golden/w4_mixtral_logits.npz), GPTQ against compressed-tensors, loop exactness against the oracle
loop and the lossless property; `big`: Mixtral-8x7B with all 32 layers in int4."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import gemm_ref, w4_moe_ckpt
from tests.test_gpu_generate import OursBackend
from tests.tiny_models import prompts

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'w4_mixtral_logits.npz'))


def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


def _stack_codes(G, N, K, gs, sdt, seed, sym=False):
    """G experts' (u [G, N, K], s [G, N, K/gs], z) on the GPU: uniform codes, scales around 0.02, zero points 6..10"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    u = torch.randint(0, 16, (G, N, K), generator=g, device=DEV, dtype=torch.uint8)
    s = (0.01 + 0.02 * torch.rand((G, N, K // gs), generator=g, device=DEV)).to(sdt)
    z = torch.full((G, N, K // gs), 8, dtype=torch.uint8, device=DEV) if sym else \
        torch.randint(6, 11, (G, N, K // gs), generator=g, device=DEV, dtype=torch.uint8)
    return u, s, z


def _grouped(u, s, z, gs, x):
    ops = _ops()
    G, N, K = u.shape
    return ops.Gemm.grouped_w4(ops.tile_weight_w4(u.reshape(G * N, K)), s.reshape(G * N, -1).t().contiguous(),
                               z.reshape(G * N, -1).t().contiguous(), gs, G, x)


# (G, N, K, scale dtype): Mixtral-8x7B's down projection (8 experts of [4096, 14336]) and a K = 384 shape whose last k
# chunk is a half chunk
DOWN = [(8, 4096, 14336, torch.bfloat16), (8, 4096, 14336, torch.float16), (4, 256, 384, torch.bfloat16),
        (3, 384, 384, torch.float16)]
ROWS = (1, 5, 64, 128, 256)


@pytest.mark.parametrize('G,N,K,sdt', DOWN)
def test_grouped_w4_against_fp64(G, N, K, sdt):
    """out[g] = bf16(X[:, gK:(g+1)K] @ W_g^T) of the dequantised weights against fp64 with tests/gemm_ref.py's
    comparator, for 1..256 rows; two runs bit-identical; rows beyond `rows` untouched in every group"""
    ops = _ops()
    u, s, z = _stack_codes(G, N, K, 128, sdt, seed=G * N + K)
    x = torch.randn((256, G * K), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV).to(torch.bfloat16)
    plan = _grouped(u, s, z, 128, x)
    assert plan.out.shape == (G, 256, N)
    refs = []
    for g in range(G):
        w = ops.dequantize_w4(u[g], s[g], z[g], 128)
        refs.append(gemm_ref.reference(x[:, g * K:(g + 1) * K], w))
    for rows in ROWS:
        plan.out.fill_(7.0)
        o1 = plan.run(rows).clone()
        o2 = plan.run(rows).clone()
        assert torch.equal(o1, o2), rows
        assert (o1[:, rows:] == 7.0).all(), rows
        for g, (ref, mass) in enumerate(refs):
            gemm_ref.assert_close(o1[g, :rows], ref[:rows], mass[:rows], K, 1, f'group {g} rows {rows}')


@pytest.mark.parametrize('G,N,K,sdt', [(8, 4096, 14336, torch.float16), (4, 256, 384, torch.bfloat16)])
def test_grouped_w4_equals_per_expert_launches_and_k_gemm_ws(G, N, K, sdt):
    """bit for bit: the grouped launch == G separate Gemm.w4 plans (one per expert), for 1..256 rows, and == the bf16
    grouped GEMM (k_gemm_ws, 64 rows) on the dequantised stack"""
    ops = _ops()
    u, s, z = _stack_codes(G, N, K, 128, sdt, seed=5 + K)
    x = torch.randn((256, G * K), generator=torch.Generator(device=DEV).manual_seed(2), device=DEV).to(torch.bfloat16)
    plan = _grouped(u, s, z, 128, x)
    xs = [x[:, g * K:(g + 1) * K].contiguous() for g in range(G)]
    singles = [ops.Gemm.w4(ops.tile_weight_w4(u[g]), s[g].t().contiguous(), z[g].t().contiguous(), 128, xs[g])
               for g in range(G)]
    for rows in ROWS:
        got = plan.run(rows)
        for g in range(G):
            assert torch.equal(got[g, :rows], singles[g].run(rows)[:rows]), (g, rows)
    w = torch.stack([ops.dequantize_w4(u[g], s[g], z[g], 128) for g in range(G)]).contiguous()
    ws = ops.Gemm.grouped(w, x[:64].contiguous())
    for rows in (1, 17, 64):
        got = plan.run(rows)
        want = ws.run(rows)
        for g in range(G):
            assert torch.equal(got[g, :rows], want[g, :rows]), (g, rows)


def test_grouped_w4_plan_refusals():
    """PIA_ERR_INVALID before any launch: groups < 1, N or K not a multiple of 128, a bad group size, misalignment,
    x_rows < 64; SiLU and ReLU on a grouped int4 plan"""
    from painlessinferenceacceleration_b200 import _lib as L
    ops = _ops()
    lib = L.load()
    x = torch.zeros((64, 2 * 256), dtype=torch.bfloat16, device=DEV)
    codes = torch.zeros((4, 1, 128, 128), dtype=torch.uint8, device=DEV)
    s, z = torch.ones((2, 512), dtype=torch.bfloat16, device=DEV), torch.zeros((2, 512), dtype=torch.uint8, device=DEV)
    before = ops.launch_count()
    cases = [(0, 256, 256, 128, 0, 64), (2, 192, 256, 128, 0, 64), (2, 256, 192, 64, 0, 64), (2, 256, 256, 64, 0, 64),
             (2, 256, 256, 96, 0, 64), (2, 256, 256, 512, 0, 64), (2, 256, 256, 128, 2, 64), (2, 256, 256, 128, 0, 32)]
    for G, N, K, gs, off, x_rows in cases:
        h = L.vp()
        rc = lib.pia_gemm_plan_create_grouped_w4(codes.data_ptr() + off, s.data_ptr(), z.data_ptr(), 0, G, N, K, gs,
                                                 x.data_ptr(), x_rows, ctypes.byref(h))
        assert rc == L.PIA_ERR_INVALID, (G, N, K, gs, off, x_rows)
    g = ops.Gemm.grouped_w4(codes, s, z, 128, 2, x)
    with pytest.raises(AssertionError, match='group'):
        g.set_silu()
    with pytest.raises(AssertionError, match='ReLU'):
        g.set_relu()
    assert ops.launch_count() == before


@pytest.mark.parametrize('rows', [5, 64, 200])
def test_stacked_gate_up_silu_equals_per_expert_gate_up_then_silu_mul(rows):
    """the stacked, per-expert interleaved gate_up of all experts in one SiLU*up launch == per expert: the plain int4
    gate_up GEMM + pia_silu_mul, bit for bit (Mixtral-8x7B's gate_up: 8 experts of [2 x 14336, 4096])"""
    ops = _ops()
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import Int4Stack
    E, I, H = 8, 14336, 4096
    u, s, z = _stack_codes(E, 2 * I, H, 128, torch.bfloat16, seed=11)
    st = Int4Stack(u, s, z, 128, interleaved=True)
    x = torch.randn((256, H), generator=torch.Generator(device=DEV).manual_seed(5), device=DEV).to(torch.bfloat16)
    act = torch.full((256, E * I), 7.0, dtype=torch.bfloat16, device=DEV)
    st.gemm(x, out=act).set_silu().run(rows)
    assert (act[rows:] == 7.0).all()
    for e in range(E):
        gu = ops.Gemm.w4(ops.tile_weight_w4(u[e]), s[e].t().contiguous(), z[e].t().contiguous(), 128, x).run(rows)
        ref = torch.empty((rows, I), dtype=torch.bfloat16, device=DEV)
        ops.silu_mul(gu[:rows].contiguous(), ref)
        assert torch.equal(act[:rows, e * I:(e + 1) * I], ref), e


# ------------------------------------------------------------------------------------------------ models
def _load(name, tmp_path, shards=1):
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    d = tmp_path / name
    w4_moe_ckpt.write(name, str(d), shards=shards)
    return MixtralForCausalLM.from_pretrained(str(d), device=torch.device(DEV))


CT = [n for n, f in w4_moe_ckpt.FIXTURES.items() if f[0] == 'compressed-tensors']


def _restatement(m, ids, dtype):
    """test_gpu_fp8.py's layer-by-layer torch restatement of Mixtral on the model's dequantised weights"""
    from tests.test_gpu_fp8 import _mixtral_restatement
    for layer in m.model.layers:   # the restatement reads the fused q|k|v weight under its fp8 name
        layer.self_attn.__dict__['qkv_fp8'] = layer.self_attn.qkv_w4
    with torch.no_grad():
        return _mixtral_restatement(m, ids, dtype)


@pytest.mark.parametrize('name', CT)
def test_w4_mixtral_verify_logits_against_the_eager_model(name, tmp_path):
    """verify logits vs the eager transformers model of the same checkpoint (fp32): max |error| <= 2 x the bf16 error
    + 0.02, the bf16 error being the larger of the eager bf16 model's and that of a bf16 torch restatement on the same
    weights.  Two bf16 references, because one token of these tiny models can swing by more than a logit under bf16
    rounding (in the 8-expert checkpoint one row errs by 0.45 in eager bf16 but by 1.46 in the bf16 restatement, whose
    fp32 twin equals the eager fp32 logits); a wrong expert, scale or row order errs far beyond both.  The loaded
    experts are the checkpoint's codes."""
    m = _load(name, tmp_path, shards=3 if name == 'mixtral_ct_sym_g128_bf16' else 1)
    assert m._w4
    _, _, codes = w4_moe_ckpt.build(name)
    u, s, z = codes['model.layers.1.block_sparse_moe.experts.2.w2']
    got = m.model.layers[1].mlp.experts.down_proj.codes()
    assert torch.equal(got[0][2].cpu(), u) and torch.equal(got[1][2].cpu(), s) and torch.equal(got[2][2].cpu(), z)
    p = w4_moe_ckpt.prompt(name).to(DEV)
    T = p.shape[1]
    m01 = torch.tril(torch.ones((1, 1, T, T), dtype=torch.long, device=DEV))
    ours = OursBackend(m).forward(p, m01, None)[0].float().cpu()
    truth, eager = torch.from_numpy(GOLDEN[name + '/fp32']), torch.from_numpy(GOLDEN[name + '/bf16'])
    restated = _restatement(m, p[0], torch.bfloat16).cpu()
    assert (_restatement(m, p[0], torch.float32).cpu() - truth).abs().max().item() < 1e-3   # the same model as the golden
    e_ours, e_eager = (ours - truth).abs().max().item(), (eager - truth).abs().max().item()
    e_restated = (restated - truth).abs().max().item()
    print(f'int4 Mixtral verify logits {name}: err vs eager fp32 {e_ours:.4f}, eager bf16 {e_eager:.4f}, bf16 '
          f'restatement {e_restated:.4f}')
    assert e_ours <= 2 * max(e_eager, e_restated) + 0.02, (e_ours, e_eager, e_restated)


def test_w4_mixtral_gptq_and_compressed_tensors_give_identical_logits(tmp_path):
    """the GPTQ v1 checkpoint and the compressed-tensors checkpoint of the same codes load to identical bytes and give
    identical verify logits"""
    a = _load('mixtral_ct_asym_g128_fp16', tmp_path)
    b = _load('mixtral_gptq_asym_g128_fp16', tmp_path)
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert sorted(pa) == sorted(pb)
    for k in pa:
        assert torch.equal(pa[k].view(-1).view(torch.uint8), pb[k].view(-1).view(torch.uint8)), k
    p = w4_moe_ckpt.prompt('mixtral_ct_asym_g128_fp16').to(DEV)
    m01 = torch.tril(torch.ones((1, 1, p.shape[1], p.shape[1]), dtype=torch.long, device=DEV))
    assert torch.equal(OursBackend(a).forward(p, m01, None), OursBackend(b).forward(p, m01, None))


@pytest.mark.parametrize('name,penalty', [('mixtral_ct_sym_g128_bf16', 1.0), ('mixtral_ct_asym_g128_e8', 1.1)])
def test_w4_mixtral_loop_is_exact_given_the_same_logits(name, penalty, tmp_path):
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
        for p in prompts(57, 3, 90, 200):
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


def test_w4_mixtral_lookahead_equals_own_greedy(tmp_path):
    """lossless: drafts never change the int4 Mixtral's output (up to near-ties), at 64 and 128 draft nodes"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    m = _load('mixtral_ct_sym_g128_i384', tmp_path)
    m.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    same = total = 0
    for dl in (64, 128):
        for p in prompts(35, 4, 16, 200):
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


def test_w4_mixtral_knobs_are_refused(tmp_path, monkeypatch):
    """int4 experts have no other GEMM: PIA_GEMM=0, PIA_GEMM_SET and PIA_MOE_GEMM=0 raise ValueError at the first
    forward"""
    for i, env in enumerate(({'PIA_GEMM': '0'}, {'PIA_GEMM_SET': 'gate_up'}, {'PIA_MOE_GEMM': '0'})):
        m = _load('mixtral_ct_sym_g128_bf16', tmp_path / str(i))
        p = prompts(3, 1, 16, 200)[0].to(DEV)
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            with pytest.raises(ValueError, match='int4'):
                m.generate(input_ids=p, max_new_tokens=4, eos_token_id=2, decoding_kwargs={'use_lookahead': False})


# ------------------------------------------------------------------------------------------------ big
def synth_w4_mixtral(cfg, seed=0, group_size=128):
    """bench.synth_fill for the bf16 parameters, seeded random codes for every projection and expert (scales as
    tests/test_gpu_w4.py's synth_w4), built layer by layer on the GPU"""
    import zlib
    import bench
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM

    def fill(name, shape):
        g = torch.Generator(device=DEV).manual_seed(zlib.crc32(name.encode()) ^ (seed * 7919))
        N, K = shape
        u = torch.randint(0, 16, (N, K), generator=g, device=DEV, dtype=torch.uint8)
        s = ((0.5 + torch.rand((N, K // group_size), generator=g, device=DEV)) * 0.02 / 8).to(torch.bfloat16)
        z = torch.full((N, K // group_size), 8, dtype=torch.uint8, device=DEV)
        return u, s, z, group_size
    return MixtralForCausalLM.build_w4(cfg, lambda m: bench.synth_fill(m, cfg, seed), fill, device=torch.device(DEV))


@pytest.mark.big
def test_w4_mixtral_8x7b_all_32_layers():
    """Mixtral-8x7B with all 32 layers in int4 (group 128): built layer by layer (no bf16 expert exists), resident and
    peak GB printed, generate() runs, and one verify step's logits are within 2 x the eager bf16 error (+0.02) of an
    fp32 torch restatement on the dequantised weights (test_gpu_fp8.py's restatement)"""
    import bench
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    cfg, _ = bench.make_config('mixtral-8x7b-16l')
    cfg.num_hidden_layers = 32
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    model = synth_w4_mixtral(cfg)
    built, peak = torch.cuda.memory_allocated() - base, torch.cuda.max_memory_allocated() - base
    print(f'int4 Mixtral-8x7B 32 layers: {built / 1e9:.2f} GB resident, build peak {peak / 1e9:.2f} GB')
    assert built < 30e9 and peak < built + 10e9, (built, peak)
    model.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=cfg.vocab_size)
    p = torch.tensor([bench.phrase_bank_prompts(1, cfg.vocab_size)[0]], device=DEV)
    for _ in range(2):
        out = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, return_dict_in_generate=True,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
        assert out.sequences.shape[1] > p.shape[1] and sum(out.kwargs['edls']) == out.sequences.shape[1] - p.shape[1]
    print(f'int4 Mixtral-8x7B generate peak {torch.cuda.max_memory_allocated() / 1e9:.2f} GB')
    model._rt = None
    torch.cuda.empty_cache()
    ids = p[:, :48]
    m01 = torch.tril(torch.ones((1, 1, 48, 48), dtype=torch.long, device=DEV))
    got = OursBackend(model).forward(ids, m01, None)[0].float()
    truth = _restatement(model, ids[0], torch.float32)
    eager = _restatement(model, ids[0], torch.bfloat16)
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    print(f'int4 Mixtral-8x7B verify logits: err vs dequantised fp32 {e_ours:.4f}, eager bf16 {e_eager:.4f}')
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)
