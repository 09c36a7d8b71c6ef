# -*- coding: utf-8 -*-
"""FP8 (e4m3) weight-only mode on the H100: the fp8 weight-streaming GEMM (k_gemm_fp8) against exact decodes and fp32
references, and the models' fp8 mode end to end - loop exactness against the oracle loop, verify logits against an fp32
evaluation of the dequantised weights, the lossless property, the batched loop, loading and refusals."""
import numpy as np
import pytest
import torch

from tests import gemm_ref
from tests.test_gpu_generate import EPS, OursBackend
from tests.tiny_models import prompts, tiny_hf_model
from tests.tiny_qwen2 import qwen2_hf_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


def _e4m3_value(codes):
    c = codes.long()
    e, m, neg = (c >> 3) & 0xF, c & 7, (c >> 7) & 1
    v = torch.where(e == 0, m.double() / 8 * 2.0 ** -6, (1 + m.double() / 8) * torch.pow(2.0, (e - 7).double()))
    return torch.where(neg == 1, -v, v)


# ------------------------------------------------------------------------------------------------ the GEMM
def test_fp8_exact_dequantisation():
    """W holds every finite e4m3 code (subnormals, +-448 and both zeros), power-of-two row scales, X one-hot rows: each
    output is one decoded code times its scale, exact in bf16, so the in-register conversion must be exact.  A -0 code
    comes out as +0 (the fp32 accumulator starts at +0; +0 + -0 = +0), so zeros are compared by value."""
    ops = _ops()
    N, K = 256, 256
    finite = torch.tensor([c for c in range(256) if c not in (0x7F, 0xFF)], dtype=torch.uint8)
    codes = finite[torch.arange(N * K) % len(finite)].view(N, K)
    codes = codes[:, torch.randperm(K, generator=torch.Generator().manual_seed(0))].contiguous()
    scale = torch.pow(2.0, (torch.arange(N) % 5 - 2).float())
    want = (_e4m3_value(codes) * scale.double()[:, None]).t()        # out[t, n] with X[t] = e_t
    qw = ops.tile_weight_fp8(codes.view(torch.float8_e4m3fn).to(DEV))
    x = torch.eye(K, dtype=torch.bfloat16, device=DEV)
    g = ops.Gemm.fp8(qw, scale.to(DEV), x)
    out = g.run(K).cpu()
    w16 = want.to(torch.bfloat16)
    assert torch.equal(w16.double(), want), 'the expected values are exact in bf16'
    nz = want != 0
    assert torch.equal(out.view(torch.int16)[nz], w16.view(torch.int16)[nz])
    assert (out[~nz] == 0).all()


def _quantised(shape, seed):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = (torch.randn(shape, generator=g, device=DEV) * 0.02).to(torch.bfloat16)
    q, s = ops.quantize_fp8(w)
    return q, s


# (name, N, K, bias, split modes): Llama-2-7B qkv / o / gate_up / down, Qwen2-7B qkv (biased) and down
SHAPES = [('llama_qkv', 12288, 4096, False, (1, -2)), ('llama_o', 4096, 4096, False, (1, -4, 4)),
          ('llama_gate_up', 22016, 4096, False, (1,)), ('llama_down', 4096, 11008, False, (1, -4, 4)),
          ('qwen2_qkv', 4608, 3584, True, (1, -4)), ('qwen2_down', 3584, 18944, False, (-4, -8))]
ROWS = (1, 5, 64, 128, 256)


@pytest.mark.parametrize('name,N,K,biased,splits', SHAPES)
def test_fp8_gemm_against_fp32(name, N, K, biased, splits):
    """out = bf16(X @ deq(W)^T (+ bias)) against the fp64 reference with the comparator of tests/gemm_ref.py, for
    1..256 rows and every split mode (plain, cluster split-K, fp32 slices); two runs bit-identical; rows beyond `rows`
    untouched"""
    ops = _ops()
    q, s = _quantised((N, K), seed=N + K)
    qw = ops.tile_weight_fp8(q)
    x = torch.randn((256, K), generator=torch.Generator(device=DEV).manual_seed(1), device=DEV).to(torch.bfloat16)
    bias = (torch.randn(N, device=DEV) * 2).to(torch.bfloat16).float() if biased else None
    ref, mass = gemm_ref.reference(x, q, s, bias)
    for sk in splits:
        g = ops.Gemm.fp8(qw, s, x, bias=bias, split_k=sk)
        for rows in ROWS:
            g.out.fill_(7.0)
            o1 = g.run(rows).clone()
            o2 = g.run(rows).clone()
            assert torch.equal(o1, o2), (name, sk, rows)
            if g.splits > 1:   # fp32 slices [splits, 256, N], summed in slice order
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


def test_fp8_mixtral_stacked_gate_up_and_grouped_down():
    """Mixtral-8x7B expert shapes: the stacked gate_up [E * 2I, H] as one plan (two experts here) and all eight experts'
    down projections [E, H, I] as one grouped launch"""
    ops = _ops()
    H, I, E = 4096, 14336, 8
    q, s = _quantised((2 * 2 * I, H), seed=3)
    x = torch.randn((256, H), generator=torch.Generator(device=DEV).manual_seed(2), device=DEV).to(torch.bfloat16)
    g = ops.Gemm.fp8(ops.tile_weight_fp8(q), s, x)
    for rows in (1, 64, 256):
        ref, mass = gemm_ref.reference(x[:rows], q, s)
        gemm_ref.assert_close(g.run(rows)[:rows], ref, mass, H, 1, f'gate_up rows {rows}')
    del g, q, s
    q, s = _quantised((E, H, I), seed=4)
    xa = torch.randn((256, E * I), generator=torch.Generator(device=DEV).manual_seed(3), device=DEV).to(torch.bfloat16)
    g = ops.Gemm.grouped_fp8(ops.tile_weight_fp8(q), s, xa)
    for rows in (1, 5, 64, 128, 256):
        g.out.fill_(7.0)
        out = g.run(rows)
        assert (out[:, rows:] == 7.0).all()
        for e in (0, 5, 7):
            ref, mass = gemm_ref.reference(xa[:rows, e * I:(e + 1) * I], q[e], s[e])
            gemm_ref.assert_close(out[e, :rows], ref, mass, I, 1, f'expert {e} rows {rows}')


@pytest.mark.parametrize('rows', [5, 64, 200])
def test_fp8_silu_epilogue_equals_gate_up_then_silu_mul(rows):
    """the fused SiLU*up epilogue on the interleaved fp8 gate/up weight == the plain fp8 GEMM + pia_silu_mul, bit for bit"""
    ops = _ops()
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import _gate_up_order
    H, I = 4096, 11008
    g0 = torch.Generator(device=DEV).manual_seed(5)
    w = (torch.randn((2 * I, H), generator=g0, device=DEV) * 0.02).to(torch.bfloat16)
    q, s = ops.quantize_fp8(_gate_up_order(w))
    qw = ops.tile_weight_fp8(q)
    x = (torch.randn((256, H), generator=g0, device=DEV)).to(torch.bfloat16)
    act = torch.full((256, I), 7.0, dtype=torch.bfloat16, device=DEV)
    ops.Gemm.fp8(qw, s, x, out=act).set_silu().run(rows)
    assert (act[rows:] == 7.0).all()
    gu_int = ops.Gemm.fp8(qw, s, x).run(rows)[:rows]                # interleaved columns
    gu = _gate_up_order(gu_int.t(), inverse=True).t().contiguous()   # [gate; up] columns
    ref = torch.empty((rows, I), dtype=torch.bfloat16, device=DEV)
    ops.silu_mul(gu, ref)
    assert torch.equal(act[:rows], ref)


# ------------------------------------------------------------------------------------------------ models
def _fp8_pair(family, seed):
    """HF bf16 model + two fp8 copies of ours with identical bytes"""
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    if family == 'qwen2':
        hf = qwen2_hf_model(seed=seed, dtype=torch.bfloat16, device=DEV, vocab=200)
    else:
        hf = tiny_hf_model(family, seed=seed, dtype=torch.bfloat16, device=DEV, vocab=200)
    cls = {'mixtral': MixtralForCausalLM, 'qwen2': Qwen2ForCausalLM}.get(family, LlamaForCausalLM)
    models = []
    for _ in range(2):
        m = cls(hf.config, device=torch.device(DEV))
        res = m.load_state_dict(hf.state_dict(), strict=False)
        assert not res.missing_keys, res
        models.append(m.quantize_fp8())
    return hf, models[0], models[1]


def _same_bytes(a, b):
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert sorted(pa) == sorted(pb)
    for k in pa:
        assert pa[k].dtype == pb[k].dtype and torch.equal(pa[k].view(-1).view(torch.uint8), pb[k].view(-1).view(torch.uint8)), k


class OursBackend128(OursBackend):
    """OursBackend on a 128-node runtime, as the fused loop runs at decoding_length = 128: the prompt goes through the
    same prefill (128-row chain chunks), every draft through the verify forward at 128 rows whatever its size"""

    def forward(self, ids_in, m01, pos):
        m, n, R = self.m, ids_in.shape[1], 128
        if self.P == 0:
            rt = m._runtime(self.max_seq, R)
            rt.set_request(0, 0, 1 << 30)
            rt.seq[0, :n] = ids_in[0].to(device=rt.device, dtype=torch.int32)
            m._prefill_logits(rt, n)
            self.P = n
            return rt.logits[0:1].clone()[None]
        rt, P = m._rt, self.P
        assert rt.max_nodes == R and n <= R and tuple(m01.shape[-2:]) == (n, P + n)
        tree = m01[0, 0, :, P:].to('cpu').numpy().astype(np.uint8)
        packed = np.packbits(np.pad(tree, ((0, R - n), (0, R - n))), axis=1, bitorder='little')
        rt.mask.copy_(torch.from_numpy(packed.view(np.int64).reshape(R, R // 64)).to(rt.device))
        rt.ids[:n] = ids_in[0].to(device=rt.device, dtype=torch.int32)
        rt.n.fill_(n)
        rt.prefix_len.fill_(P)
        rt.set_request(0, 0, 1 << 30)
        m._verify_layers(rt)
        self.P = P + n
        return rt.logits[:n].clone()[None]


@pytest.mark.parametrize('family,penalty,dl', [('llama', 1.0, 64), ('mistral', 1.1, 64), ('qwen2', 1.0, 64),
                                               ('mixtral', 1.0, 64), ('llama', 1.0, 128)])
def test_fp8_loop_is_exact_given_the_same_logits(family, penalty, dl):
    """the oracle loop drives one fp8 copy through OursBackend, the fused device loop another copy with identical
    bytes: tokens, dls and edls identical for every request, tries carried across requests.  decoding_length = 128:
    both run the fp8 plans at 128 rows (two 64-row token blocks per launch)"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, a, b = _fp8_pair(family, seed=6)
    _same_bytes(a, b)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    backend = OursBackend128 if dl == 128 else OursBackend
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 3, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': dl, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=48, eos_token_id=[2], repetition_penalty=penalty,
                                     decoding_length=dl,
                                     backend=backend(b, prefill_like_generate=True, max_seq=90 + 48 + 2 * dl + 1))
            assert a._rt.max_nodes == (128 if dl == 128 else 64)
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (family, dl, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (family, dl, rep)
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


def _dequantised_state(hf, ours):
    """HF state dict whose projections are ours' dequantised fp8 weights (fp32)"""
    sd = {k: v.float() for k, v in hf.state_dict().items()}
    for i, layer in enumerate(ours.model.layers):
        pre = f'model.layers.{i}.'
        a = layer.self_attn
        for n in ('q_proj', 'k_proj', 'v_proj', 'o_proj'):
            sd[pre + f'self_attn.{n}.weight'] = getattr(a, n).dequantize()
        if hasattr(layer.mlp, 'experts'):
            sd[pre + 'mlp.experts.gate_up_proj'] = layer.mlp.experts.gate_up_proj.dequantize()
            sd[pre + 'mlp.experts.down_proj'] = layer.mlp.experts.down_proj.dequantize()
        else:
            for n in ('gate_proj', 'up_proj', 'down_proj'):
                sd[pre + f'mlp.{n}.weight'] = getattr(layer.mlp, n).dequantize()
    return sd


@pytest.mark.parametrize('family', ['llama', 'mistral', 'qwen2', 'mixtral'])
def test_fp8_verify_logits_within_tolerance(family):
    """fp8 verify logits vs an fp32 evaluation of the dequantised weights: max |error| <= 2 x the eager bf16 error of
    the same weights + 0.02; the error against the original bf16 weights' fp32 truth is logged"""
    hf, ours, _ = _fp8_pair(family, seed=8)
    mk = (lambda dt: qwen2_hf_model(seed=8, dtype=dt, device=DEV, vocab=200)) if family == 'qwen2' else \
        (lambda dt: tiny_hf_model(family, seed=8, dtype=dt, device=DEV, vocab=200))
    orig = {k: v.float() for k, v in hf.state_dict().items()}
    deq = _dequantised_state(hf, ours)
    hf32 = mk(torch.float32)
    p = prompts(77, 1, 100, 200)[0].to(DEV)
    with torch.no_grad():
        hf32.load_state_dict(orig)
        truth_orig = hf32(input_ids=p).logits[0].float()
        hf32.load_state_dict(deq)
        truth = hf32(input_ids=p).logits[0].float()
        eager_m = mk(torch.bfloat16)
        eager_m.load_state_dict({k: v.to(torch.bfloat16) for k, v in deq.items()})
        eager = eager_m(input_ids=p).logits[0].float()
    m01 = torch.tril(torch.ones((1, 1, 100, 100), dtype=torch.long, device=DEV))
    got = OursBackend(ours).forward(p, m01, None)[0].float()
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    e_orig = (got - truth_orig).abs().max().item()
    print(f'fp8 verify logits {family}: err vs dequantised fp32 {e_ours:.4f}, eager bf16 {e_eager:.4f}, '
          f'vs original weights {e_orig:.4f}')
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)


def test_fp8_lookahead_equals_own_greedy():
    """lossless: drafts never change the fp8 model's output (up to near-ties), at 64 and at 128 draft nodes"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    _, ours, _ = _fp8_pair('llama', seed=4)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    same = total = 0
    for dl in (64, 128):
        for p in prompts(33, 4, 16, 200):
            p = p.to(DEV)
            g = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
            for _ in range(2):
                o = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, return_dict_in_generate=True,
                                  decoding_kwargs={'use_lookahead': True, 'decoding_length': dl, 'branch_length': 8})
            assert o.sequences.shape[1] <= 16 + 40
            assert sum(o.kwargs['edls']) == o.sequences.shape[1] - 16
            total += 1
            if o.sequences[0].tolist() == g[0].tolist():
                same += 1
                assert max(o.kwargs['edls']) > 1
    assert same >= total - 2, (same, total)


def test_fp8_batched_loop_matches_single_request_loop():
    """the batched loop (bs = 3) on fp8 weights: every request equals the single-request fp8 loop, except where they
    part on a near-tie of the fp8 model's own logits (top-2 margin < EPS)"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.llama.modeling_llama_batch import LlamaForCausalLM as Batched
    hf, single, _ = _fp8_pair('llama', seed=14)
    batched = Batched(hf.config, device=torch.device(DEV))
    batched.load_state_dict(hf.state_dict(), strict=False)
    batched.quantize_fp8()
    _same_bytes(single, batched)
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


@pytest.mark.parametrize('tied', [False, True])
def test_fp8_from_pretrained_equals_quantize_fp8(tmp_path, tied):
    """from_pretrained(..., quantization='fp8') gives the bytes quantize_fp8() gives the bf16-loaded model; the peak
    allocation stays below the fp8 model plus a few bf16 tensors; a missing tensor still raises"""
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    L = 12
    hf = qwen2_hf_model(seed=10, dtype=torch.bfloat16, device=DEV, vocab=200, tie_word_embeddings=tied,
                        num_hidden_layers=L, layer_types=['full_attention'] * L)
    hf.save_pretrained(str(tmp_path))
    del hf
    ref = Qwen2ForCausalLM.from_pretrained(str(tmp_path), device=torch.device(DEV))
    bf16_bytes = sum(p.numel() * p.element_size() for p in ref.parameters())
    layer_bf16 = sum(p.numel() * p.element_size() for n, p in ref.model.layers[0].named_parameters()
                     if n.endswith('proj.weight'))
    ref.quantize_fp8()
    fp8_bytes = sum(p.numel() * p.element_size() for p in ref.parameters())
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = Qwen2ForCausalLM.from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')
    peak = torch.cuda.max_memory_allocated() - base
    _same_bytes(ref, got)
    # one layer in flight: its bf16 projections, their fused copies and the quantiser's fp32 temporaries
    assert peak < fp8_bytes + 4 * layer_bf16 < bf16_bytes, (peak, fp8_bytes, layer_bf16, bf16_bytes)
    # a missing tensor raises
    from safetensors.torch import load_file, save_file
    f = next(tmp_path.glob('*.safetensors'))
    sd = load_file(str(f))
    del sd['model.layers.1.mlp.down_proj.weight']
    save_file(sd, str(f), metadata={'format': 'pt'})
    with pytest.raises(RuntimeError, match='missing'):
        Qwen2ForCausalLM.from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')


def test_fp8_from_pretrained_mixtral_experts_across_shards(tmp_path):
    """a Mixtral checkpoint in the published layout (block_sparse_moe.experts.N.w1/w2/w3), each layer's experts split
    over two shards: from_pretrained(..., quantization='fp8') quantises the stacks once _convert_checkpoint_keys has
    assembled them and gives the bytes of quantize_fp8() on the bf16-loaded model"""
    from safetensors.torch import save_file
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    hf = tiny_hf_model('mixtral', seed=16, dtype=torch.bfloat16, device=DEV, vocab=200)
    ours = MixtralForCausalLM(hf.config, device=torch.device(DEV))
    ours.load_state_dict(hf.state_dict(), strict=False)
    E, I = hf.config.num_local_experts, hf.config.intermediate_size
    shards = [{}, {}]
    for k, v in ours.state_dict().items():
        v = v.detach().cpu().contiguous()
        if k.endswith('mlp.experts.gate_up_proj') or k.endswith('mlp.experts.down_proj'):
            pre = k[:k.index('.mlp.')] + '.block_sparse_moe.experts.'
            for e in range(E):
                dst = shards[e % 2]   # every layer's experts straddle both shards
                if k.endswith('gate_up_proj'):
                    dst[f'{pre}{e}.w1.weight'] = v[e, :I].clone()
                    dst[f'{pre}{e}.w3.weight'] = v[e, I:].clone()
                else:
                    dst[f'{pre}{e}.w2.weight'] = v[e].clone()
        elif k.endswith('.mlp.gate.weight'):
            shards[1][k.replace('.mlp.gate.weight', '.block_sparse_moe.gate.weight')] = v
        else:
            shards[0][k] = v
    hf.config.save_pretrained(str(tmp_path))
    for i, sd in enumerate(shards):
        save_file(sd, str(tmp_path / f'model-0000{i + 1}-of-00002.safetensors'), metadata={'format': 'pt'})
    ref = MixtralForCausalLM.from_pretrained(str(tmp_path), device=torch.device(DEV))
    assert torch.equal(ref.model.layers[1].mlp.experts.down_proj, ours.model.layers[1].mlp.experts.down_proj)
    ref.quantize_fp8()
    got = MixtralForCausalLM.from_pretrained(str(tmp_path), device=torch.device(DEV), quantization='fp8')
    _same_bytes(ref, got)


def test_fp8_refusals(monkeypatch):
    """fp8 weights have no other GEMM: PIA_GEMM=0 and PIA_GEMM_SET raise ValueError; so does a misaligned shape"""
    from transformers import LlamaConfig
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    for env in ({'PIA_GEMM': '0'}, {'PIA_GEMM_SET': 'gate_up'}):
        _, ours, _ = _fp8_pair('llama', seed=1)
        p = prompts(3, 1, 16, 200)[0].to(DEV)
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            with pytest.raises(ValueError, match='fp8'):
                ours.generate(input_ids=p, max_new_tokens=4, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
    ops = _ops()   # the SiLU epilogue has no expert index: a grouped plan refuses it
    xg = torch.zeros((64, 256), dtype=torch.bfloat16, device=DEV)
    grouped = ops.Gemm.grouped_fp8(torch.zeros((2, 1, 1, 128, 128), dtype=torch.uint8, device=DEV),
                                   torch.ones(256, device=DEV), xg)
    with pytest.raises(AssertionError, match='one group'):
        grouped.set_silu()
    cfg = LlamaConfig(vocab_size=64, hidden_size=192, intermediate_size=512, num_hidden_layers=1,
                      num_attention_heads=2, num_key_value_heads=2, rms_norm_eps=1e-6)
    with pytest.raises(ValueError):
        LlamaForCausalLM(cfg, device=torch.device(DEV)).quantize_fp8()


# ------------------------------------------------------------------------------------------------ big
@pytest.mark.big
def test_fp8_loop_is_exact_at_llama2_7b_shape():
    """Llama-2-7B shape, all 32 layers, fp8: the oracle loop through one copy, the fused device loop through another"""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg, _ = bench.make_config('llama2-7b')
    a = LlamaForCausalLM(cfg, device=torch.device(DEV)).init_weights(seed=0).quantize_fp8()
    b = LlamaForCausalLM(cfg, device=torch.device(DEV)).init_weights(seed=0).quantize_fp8()
    _same_bytes(a, b)
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


def _synth_fp8(cls, cfg, seed=0):
    """bench.synth_fill's weights in fp8 without the bf16 model: LlamaForCausalLM.build_fp8 with synth_fill for the
    bf16 parameters (the projections are still meta tensors then) and synth_fill's per-name fill for each projection"""
    import zlib
    import bench
    return cls.build_fp8(cfg, lambda m: bench.synth_fill(m, cfg, seed),
                         lambda name, t: bench.hashed_normal_(t, zlib.crc32(name.encode()) ^ (seed * 7919), 0.02),
                         device=torch.device(DEV))


def _mixtral_restatement(model, ids, dtype):
    """Mixtral's forward written out in torch, layer by layer, on the dequantised fp8 weights (dequantised one layer at
    a time), in `dtype`: RMSNorm, RoPE, causal GQA attention, fp32 router softmax -> top-k -> renormalise -> `dtype`,
    every expert's SiLU MLP weighted and summed in expert order, final norm, bf16 lm_head"""
    import torch.nn.functional as F
    c = model.config
    hd, nh, nkv, eps = c.hidden_size // c.num_attention_heads, c.num_attention_heads, c.num_key_value_heads, c.rms_norm_eps
    T = ids.numel()
    rp = getattr(c, 'rope_parameters', None) or {}
    theta = float(getattr(c, 'rope_theta', None) or rp.get('rope_theta', 10000.0))
    inv = 1.0 / (theta ** (torch.arange(0, hd, 2, device=DEV).float() / hd))
    fr = torch.arange(T, device=DEV).float()[:, None] * inv[None]
    cos, sin = torch.cat([fr, fr], -1).cos().to(dtype), torch.cat([fr, fr], -1).sin().to(dtype)

    def rms(v, w):
        v32 = v.float()
        return w.to(dtype) * (v32 * torch.rsqrt(v32.pow(2).mean(-1, keepdim=True) + eps)).to(dtype)

    def rope(t):   # [heads, T, hd]
        return t * cos + torch.cat([-t[..., hd // 2:], t[..., :hd // 2]], -1) * sin

    causal = torch.ones((T, T), dtype=torch.bool, device=DEV).tril()
    x = model.model.embed_tokens.weight[ids].to(dtype)
    for layer in model.model.layers:
        a, moe = layer.self_attn, layer.mlp
        h = rms(x, layer.input_layernorm.weight)
        qkv = h @ a.qkv_fp8.dequantize().to(dtype).t()
        q, k, v = qkv.split([nh * hd, nkv * hd, nkv * hd], -1)
        q = rope(q.view(T, nh, hd).transpose(0, 1))
        k = rope(k.view(T, nkv, hd).transpose(0, 1)).repeat_interleave(nh // nkv, 0)
        v = v.view(T, nkv, hd).transpose(0, 1).repeat_interleave(nh // nkv, 0)
        s = (q @ k.transpose(-1, -2)) / hd ** 0.5
        p = torch.softmax(s.float().masked_fill(~causal, float('-inf')), -1).to(dtype)
        o = (p @ v).transpose(0, 1).reshape(T, nh * hd)
        x = x + o @ a.o_proj.dequantize().to(dtype).t()
        h = rms(x, layer.post_attention_layernorm.weight)
        probs = torch.softmax((h @ moe.gate.weight.to(dtype).t()).float(), -1)
        tv, ti = probs.topk(moe.top_k, -1)
        tv = (tv / tv.sum(-1, keepdim=True)).to(dtype)
        gu, dn = moe.experts.gate_up_proj.dequantize(), moe.experts.down_proj.dequantize()
        out = torch.zeros_like(x)
        for e in range(moe.num_experts):
            w_e = (tv * (ti == e)).sum(-1, keepdim=True)
            g, u = (h @ gu[e].to(dtype).t()).chunk(2, -1)
            out = out + ((F.silu(g) * u) @ dn[e].to(dtype).t()) * w_e
        del gu, dn
        x = x + out
    return (rms(x, model.model.norm.weight) @ model.lm_head.weight.to(dtype).t()).float()


@pytest.mark.big
def test_fp8_mixtral_8x7b_all_32_layers():
    """Mixtral-8x7B with all 32 layers in fp8 on one 80 GB card: built layer by layer (the bf16 model never exists) with
    a bounded peak allocation, generate() completes, and one verify step's logits are within 2 x the eager bf16 error
    (+0.02) of an fp32 torch restatement on the dequantised weights"""
    import bench
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    cfg, _ = bench.make_config('mixtral-8x7b-16l')
    cfg.num_hidden_layers = 32
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    model = _synth_fp8(MixtralForCausalLM, cfg)
    built, peak = torch.cuda.memory_allocated() - base, torch.cuda.max_memory_allocated() - base
    print(f'fp8 Mixtral-8x7B 32 layers: {built / 1e9:.2f} GB resident, build peak {peak / 1e9:.2f} GB')
    assert built < 50e9 and peak < built + 8e9, (built, peak)
    model.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=cfg.vocab_size)
    p = torch.tensor([bench.phrase_bank_prompts(1, cfg.vocab_size)[0]], device=DEV)
    for _ in range(2):
        out = model.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, return_dict_in_generate=True,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
        assert out.sequences.shape[1] > p.shape[1] and sum(out.kwargs['edls']) == out.sequences.shape[1] - p.shape[1]
    assert torch.cuda.max_memory_allocated() < 75e9
    model._rt = None
    torch.cuda.empty_cache()
    ids = p[:, :48]
    m01 = torch.tril(torch.ones((1, 1, 48, 48), dtype=torch.long, device=DEV))
    got = OursBackend(model).forward(ids, m01, None)[0].float()
    with torch.no_grad():
        truth = _mixtral_restatement(model, ids[0], torch.float32)
        eager = _mixtral_restatement(model, ids[0], torch.bfloat16)
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    print(f'fp8 Mixtral-8x7B verify logits: err vs dequantised fp32 {e_ours:.4f}, eager bf16 {e_eager:.4f}')
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)
