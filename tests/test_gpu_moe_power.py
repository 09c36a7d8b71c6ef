# -*- coding: utf-8 -*-
"""Tests of k_moe_router and k_moe_combine (csrc/fused_ops.cu) and of Mixtral's composed MoE block that can fail: the
router against an fp64 reference whose comparator tolerates only real ties (tests/moe_ref.py), on inputs whose logits
are exact so that only the softmax can leave a tie; the router against the reference's eager torch ops on this GPU;
the combine bit for bit against the reference's sparse index_add_ loop, also when an unselected expert's output is
inf or NaN; every intermediate of the decode block at Mixtral-8x7B and 8x22B shapes on the bf16 plans, the cuBLAS
path and the fp8 plans.

The first half runs without a GPU: the comparator accepts an emulation of the router's fp32 arithmetic and rejects
every wrong router of moe_ref's list, the combine reference equals the dense emulation and rejects every wrong
combine, the reference's weight rounding differs from transformers', and the exact inputs hold the ties, underflows
and gaps they claim."""
import types

import pytest
import torch

from tests import gemm_ref
from tests import moe_ref as M

DEV = 'cuda:0'
BF16 = torch.bfloat16
SENT = 0x7FA5                 # a NaN bit pattern no kernel writes
ROUTER_E = (1, 2, 3, 8, 16, 63, 64)
ROUTER_HIDDEN = (8, 264, 4096, 4104, 6144, 14336)
ROUTER_ROWS = (1, 5, 64, 257)
COMBINE_E = (1, 2, 8, 16, 64)
COMBINE_HIDDEN = (8, 2048, 2056, 4096, 6144)
COMBINE_TOPK = {1: 1, 2: 2, 8: 2, 16: 4, 64: 6}
MAX_NEEDED = 0.02             # share of random rows that may differ from the fp64 reference's own answer (ties)
MIN_FORMULA_DIFF = 0.10       # share of outputs where bf16(ye * bf16(w)) and bf16(ye * w_fp32) must differ


def _bits(t):
    return t.view(torch.int16)


def _sentinel(shape, device):
    return torch.full(shape, SENT, dtype=torch.int16, device=device).view(BF16)


def _topks(E):
    return sorted({k for k in (1, 2, 3, E) if k <= E})


def _same(a, b):
    """bit-equal, with any NaN matching any NaN"""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(_bits(a)[~na], _bits(b)[~nb])


# ---------------------------------------------------------------------------------------------------------------
# the CPU half
# ---------------------------------------------------------------------------------------------------------------
CPU_EXACT = [(64, 264, 8, 2), (48, 8, 16, 3), (24, 4104, 64, 3), (12, 264, 3, 3), (24, 264, 2, 1), (30, 264, 63, 2)]
CPU_RANDOM = [(64, 4096, 8, 2), (32, 6144, 8, 2), (32, 264, 16, 4)]


def _router_cases():
    for i, (rows, hidden, E, k) in enumerate(CPU_EXACT):
        y, gate = M.exact_router_inputs(rows, hidden, E, seed=10 + i)
        yield dict(y=y, gate=gate, k=k, exact=True)
    for i, (rows, hidden, E, k) in enumerate(CPU_RANDOM):
        y, gate = M.random_router_inputs(rows, hidden, E, seed=20 + i)
        yield dict(y=y, gate=gate, k=k, exact=False)


def test_moe_mutation_lists_are_complete():
    assert set(M.ROUTER_MUTATIONS) == {'no_renormalisation', 'prob_bf16', 'highest_index_wins_ties', 'smallest_k',
                                       'fp32_logits', 'bf16_exp', 'truncate_weights', 'top_k_minus_1'}
    assert set(M.COMBINE_MUTATIONS) == {'reverse_order', 'fp32_accumulate', 'product_unrounded', 'weight_after_sum',
                                        'no_zero_skip'}


def test_router_comparator_accepts_the_kernel_and_rejects_every_mutation():
    cases = list(_router_cases())
    for c in cases:
        got = M.emulate_router(c['y'], c['gate'], c['k'])
        r = M.router_check(got, c['y'], c['gate'], c['k'], exact=c['exact'])
        assert r['bad'] == 0, (c['y'].shape, c['gate'].shape[0], c['k'], r)
        if c['exact']:
            assert r['open_logit'] == 0
    for mut in M.ROUTER_MUTATIONS:
        hits = [M.router_check(M.emulate_router(c['y'], c['gate'], c['k'], mut=mut), c['y'], c['gate'], c['k'],
                               exact=c['exact'])['bad'] > 0 for c in cases]
        assert any(hits), mut


def test_exact_inputs_hold_what_they_claim():
    """fp32 sums exact in the kernel's order (emulated unrounded logits == fp64); exactly equal logits at the k-th
    place; rows whose selected second weight underflows to 0; logit gaps over 88; selected weights that are bf16
    subnormals; all-zero rows; negative logits"""
    ties = underflow = gaps = subnormal = 0
    for i, (rows, hidden, E, k) in enumerate(CPU_EXACT):
        y, gate = M.exact_router_inputs(rows, hidden, E, seed=10 + i)
        L, _ = M.logits64(y, gate)
        assert torch.equal(M.emulate_logits(y, gate, mut='fp32_logits').double(), L)
        lg = M.bf16_rne(L)
        w, sel = M.router_ref(y, gate, k)
        srt = lg.sort(-1, descending=True).values
        if k < E:
            ties += int((srt[:, k - 1] == srt[:, k]).sum())
        if E >= 2:
            gaps += int((srt[:, 0] - srt[:, 1] > 88).sum())
            assert (lg < 0).any()
        underflow += int((sel & (w == 0)).any(-1).sum())
        subnormal += int((sel & (w > 0) & (w < 2.0 ** -126)).any(-1).sum())
        assert (lg[::6] == 0).all()
    assert ties >= 20 and underflow >= 10 and gaps >= 20 and subnormal >= 5, (ties, underflow, gaps, subnormal)


def _combine_case(E, rows, cap, hidden, k, seed, fill=None):
    y, gate = M.random_router_inputs(rows, hidden, E, seed=seed)
    dense = M.emulate_router(y, gate, k)
    ye = M.expert_outputs(E, cap, hidden, seed=seed + 1)
    if fill is not None:
        unsel = torch.ones((E, cap), dtype=torch.bool)
        unsel[:, :rows] = (dense == 0).t()
        ye[unsel] = fill
    return ye, dense


COMBINE_CPU = [(1, 7, 8, 64, 1), (2, 9, 16, 2056, 2), (8, 13, 16, 512, 2), (16, 5, 8, 264, 4), (64, 6, 8, 64, 6)]


def test_combine_reference_equals_the_dense_emulation():
    """finite outputs: the sparse loop and the dense sum (zero weights skipped) agree to the bit; the unfixed kernel
    (`no_zero_skip`, ye * 0 added) agrees too.  inf / NaN in an unselected expert's output: the sparse loop never
    reads it, the dense sum skips it, the unfixed kernel turns the token's sum into NaN"""
    for i, (E, rows, cap, hidden, k) in enumerate(COMBINE_CPU):
        ye, dense = _combine_case(E, rows, cap, hidden, k, seed=40 + i)
        ref = M.combine_ref(ye, dense)
        assert _same(M.emulate_combine(ye, dense), ref)
        assert _same(M.emulate_combine(ye, dense, mut='no_zero_skip'), ref)
        for fill in (float('inf'), float('-inf'), float('nan'), 3e38):
            ye2, _ = _combine_case(E, rows, cap, hidden, k, seed=40 + i, fill=fill)
            assert _same(M.combine_ref(ye2, dense), ref)
            assert _same(M.emulate_combine(ye2, dense), ref)
            if E > k and fill != 3e38:
                assert torch.isnan(M.emulate_combine(ye2, dense, mut='no_zero_skip')).any(), (E, fill)


def test_combine_rejects_every_mutation():
    for mut in M.COMBINE_MUTATIONS:
        hits = []
        for i, (E, rows, cap, hidden, k) in enumerate(COMBINE_CPU):
            for fill in (None, float('inf')):
                ye, dense = _combine_case(E, rows, cap, hidden, k, seed=40 + i, fill=fill)
                hits.append(not _same(M.emulate_combine(ye, dense, mut=mut), M.combine_ref(ye, dense)))
        assert any(hits), mut


def _formula_share(E, rows, hidden, k, seed, device='cpu'):
    y, gate = M.random_router_inputs(rows, hidden, E, seed=seed)
    dense, w32 = M.emulate_router(y, gate, k), M.emulate_router(y, gate, k, fp32_weights=True)
    ye = M.expert_outputs(E, rows, hidden, seed=seed + 1).to(device)
    a, b = M.combine_ref(ye, dense.to(device)), M.combine_transformers(ye, w32.to(device))
    return (a != b).double().mean().item()


def test_reference_and_transformers_formulas_differ():
    """the reference rounds the routing weights to bf16 before scaling, transformers 5.5 scales by the fp32 weights:
    on these inputs the two differ on more than MIN_FORMULA_DIFF of the outputs, so the combine tests tell them apart"""
    for E, rows, hidden, k in ((8, 64, 4096, 2), (16, 32, 2056, 4)):
        share = _formula_share(E, rows, hidden, k, seed=E)
        print(f'E {E} top-{k}: the two formulas differ on {100 * share:.1f} % of the outputs')
        assert share > MIN_FORMULA_DIFF, share


# ---------------------------------------------------------------------------------------------------------------
# the GPU half
# ---------------------------------------------------------------------------------------------------------------
def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


def _route(y, gate, k):
    """one pia_moe_router call into a buffer with two sentinel rows after `rows`"""
    rows, E = y.shape[0], gate.shape[0]
    dense = _sentinel((rows + 2, E), y.device)
    _ops().moe_router(y, gate, k, dense[:rows])
    torch.cuda.synchronize()
    assert (_bits(dense[rows:]) == SENT).all()
    return dense[:rows]


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', ROUTER_HIDDEN)
@pytest.mark.parametrize('E', ROUTER_E)
def test_router_exact_logits(E, hidden):
    """logits exact in fp32 in any order: the kernel equals the fp64 reference up to softmax-budget ties, at every
    top-k and row count; rows past `rows` keep their sentinel"""
    n_open = n_need = n = 0
    for ri, rows in enumerate(ROUTER_ROWS):
        y, gate = M.exact_router_inputs(rows, hidden, E, seed=E * 1000 + hidden + ri, device=DEV)
        for k in _topks(E):
            r = M.router_check(_route(y, gate, k), y, gate, k, exact=True)
            assert r['bad'] == 0 and r['open_logit'] == 0, (rows, k, r)
            n_open, n = n_open + r['open_select'], n + r['n']
            n_need += int(r['needed'].sum())
    assert n_open <= 0.01 * n and n_need <= 0.01 * n, (n_open, n_need, n)


SHAPES = {'mixtral-8x7b': (4096, 14336, 32), 'mixtral-8x22b': (6144, 16384, 48)}   # hidden, inter, heads


@pytest.mark.gpu
@pytest.mark.parametrize('shape', list(SHAPES))
def test_router_matches_eager_torch(shape):
    """the reference's own ops on this GPU (bf16 F.linear, fp32 softmax, torch.topk, renormalise, cast): kernel and
    torch both pass the fp64 comparator, they differ only on rows the comparator leaves open, and few rows of either
    needed the tie allowance (differ from the fp64 reference's own answer)"""
    import torch.nn.functional as F
    hidden = SHAPES[shape][0]
    n = n_open = n_diff = n_need_k = n_need_t = 0
    for seed in range(4):
        y, gate = M.random_router_inputs(257, hidden, 8, seed=seed + hidden, device=DEV)
        got = _route(y, gate, 2)
        probs = F.softmax(F.linear(y, gate), dim=1, dtype=torch.float)
        w, sel = torch.topk(probs, 2, dim=-1)
        w = (w / w.sum(dim=-1, keepdim=True)).to(BF16)
        want = torch.zeros((257, 8), dtype=BF16, device=DEV).scatter_(1, sel, w)
        rk = M.router_check(got, y, gate, 2)
        rt = M.router_check(want, y, gate, 2)
        assert rk['bad'] == 0 and rt['bad'] == 0, (rk, rt)
        diff = (_bits(got) != _bits(want)).any(-1)
        assert not (diff & ~rk['open']).any(), int((diff & ~rk['open']).sum())
        n, n_open, n_diff = n + rk['n'], n_open + int(rk['open'].sum()), n_diff + int(diff.sum())
        n_need_k, n_need_t = n_need_k + int(rk['needed'].sum()), n_need_t + int(rt['needed'].sum())
    print(f'{shape}: {n} rows, {n_open} left open by the comparator; needed the tie allowance: kernel {n_need_k}, '
          f'torch {n_need_t}; kernel != torch on {n_diff}')
    assert n_need_k <= MAX_NEEDED * n and n_need_t <= MAX_NEEDED * n, (n_need_k, n_need_t, n)


@pytest.mark.gpu
@pytest.mark.parametrize('E', [8, 16, 64])
def test_torch_topk_takes_the_lowest_index_among_ties(E):
    """the kernel's tie rule is the reference's: among exactly equal probabilities torch.topk on this GPU selects the
    lowest indices, and the kernel's top-k set is the same on the same logits"""
    n_ties = 0
    for k in (1, 2, 3):
        y, gate = M.exact_router_inputs(257, 264, E, seed=E + k, device=DEV)
        L, _ = M.logits64(y, gate)
        lg = M.bf16_rne(L).float()
        probs = torch.softmax(lg, dim=1, dtype=torch.float)
        idx = torch.topk(probs, k, dim=-1).indices
        torch_set = torch.zeros_like(probs, dtype=torch.bool).scatter_(1, idx, True)
        low = torch.sort(probs.cpu(), dim=-1, descending=True, stable=True).indices[:, :k].to(DEV)
        low_set = torch.zeros_like(torch_set).scatter_(1, low, True)
        srt = probs.sort(-1, descending=True).values
        tied = srt[:, k - 1] == srt[:, k]
        n_ties += int(tied.sum())
        assert torch.equal(torch_set, low_set), int((torch_set != low_set).any(-1).sum())
        assert not ((_route(y, gate, k) != 0) & ~torch_set).any()
    print(f'E {E}: {n_ties} rows with exactly equal probabilities at the k-th place, torch.topk took the lowest '
          'indices in all of them')
    assert n_ties > 50


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', COMBINE_HIDDEN)
@pytest.mark.parametrize('E', COMBINE_E)
def test_combine_matches_the_reference_loop(E, hidden):
    """weights from the kernel router; the reference's index_add_ loop on this GPU, bit for bit, rows past `rows`
    untouched; then +inf, -inf, NaN and 3e38 in every unselected expert output change nothing"""
    ops = _ops()
    k = COMBINE_TOPK[E]
    for cap in (64, 256):
        ye0 = M.expert_outputs(E, cap, hidden, seed=E + hidden + cap, device=DEV)
        for rows in (1, 63, 64):
            y, gate = M.random_router_inputs(rows, hidden, E, seed=rows + hidden, device=DEV)
            dense = _route(y, gate, k)
            assert ((dense != 0).sum(-1) == k).all()      # no selected weight underflows: nonzero == selected
            ref = M.combine_ref(ye0, dense)
            for fill in (None, float('inf'), float('-inf'), float('nan'), 3e38):
                ye = ye0
                if fill is not None:
                    ye = ye0.clone()
                    unsel = torch.ones((E, cap), dtype=torch.bool, device=DEV)
                    unsel[:, :rows] = (dense == 0).t()
                    ye[unsel] = fill
                    assert _same(M.combine_ref(ye, dense), ref)
                out = _sentinel((cap + 1, hidden), DEV)
                ops.moe_combine(ye, dense, out)
                torch.cuda.synchronize()
                assert _same(out[:rows], ref), (cap, rows, fill)
                assert (_bits(out[rows:]) == SENT).all()


def _mixtral_layer(shape, seed):
    from transformers import MixtralConfig
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    H, I, heads = SHAPES[shape]
    cfg = MixtralConfig(vocab_size=256, hidden_size=H, intermediate_size=I, num_hidden_layers=1,
                        num_attention_heads=heads, num_key_value_heads=8, max_position_embeddings=4096,
                        num_local_experts=8, num_experts_per_tok=2, rms_norm_eps=1e-5, sliding_window=None)
    m = MixtralForCausalLM(cfg, device=torch.device(DEV))
    m.init_weights(seed=seed, std=0.02)
    return m, m.model.layers[0]


def _check_gemm(got, x, w, K, msg, scale=None):
    ref, mass = gemm_ref.reference(x, w, scale)
    gemm_ref.assert_close(got, ref, mass, K, 1, msg)


def _check_combine(out, ye, dense, rows):
    ref = M.combine_ref(ye, dense[:rows])
    assert _same(out[:rows], ref)


def _blow_up(moe, dense):
    """the expert fewest rows selected gets a down projection of 2^127s: its outputs overflow for every row"""
    e = int((dense != 0).sum(0).argmin())
    moe.experts.down_proj.data[e] = 2.0 ** 127
    return e


@pytest.mark.gpu
@pytest.mark.big
@pytest.mark.parametrize('shape', list(SHAPES))
def test_decode_block_intermediates(shape):
    """one Mixtral layer's MoE block as _mlp runs it on the decode plans: the stacked gate_up GEMM, SiLU*up over the
    [rows * E, 2I] view against each expert's own [gate; up] columns, the grouped down GEMM per expert, the combine
    against the reference loop; the same for the cuBLAS path and the fp8 plans.  Then an expert whose outputs overflow
    leaves the rows that did not select it finite and equal to the reference"""
    ops = _ops()
    m, layer = _mixtral_layer(shape, seed=7)
    moe = layer.mlp
    E, two_i, H = moe.experts.gate_up_proj.shape
    I = two_i // 2
    gu_w, dn_w = moe.experts.gate_up_proj.data, moe.experts.down_proj.data
    y = torch.randn((64, H), generator=torch.Generator(device=DEV).manual_seed(3), device=DEV).to(BF16)

    # bf16 decode plans
    b = types.SimpleNamespace(rows=64, y=y)
    plans = m._layer_gemm_plans(layer, b)
    assert set(plans) == {'moe_gate_up', 'moe_down'}
    out, _ = m._mlp(None, layer, y, plans, b=b)
    torch.cuda.synchronize()
    assert M.router_check(b.moe_dense, y, moe.gate.weight, moe.top_k)['bad'] == 0
    _check_gemm(b.moe_gu, y, gu_w.view(E * two_i, H), H, 'stacked gate_up')
    ye = plans['moe_down'].out
    for e in range(E):
        gu_e = b.moe_gu[:, e * two_i:(e + 1) * two_i]
        _check_gemm(gu_e[:, :I], y, gu_w[e, :I], H, f'gate {e}')
        _check_gemm(gu_e[:, I:], y, gu_w[e, I:], H, f'up {e}')
        want = torch.nn.functional.silu(gu_e[:, :I]) * gu_e[:, I:]
        assert torch.equal(_bits(b.moe_act[:, e * I:(e + 1) * I]), _bits(want)), e
        _check_gemm(ye[e], b.moe_act[:, e * I:(e + 1) * I], dn_w[e], I, f'down {e}')
    _check_combine(out, ye, b.moe_dense, 64)

    # the cuBLAS path: per expert torch.mm, silu_mul, torch.mm, then the masked add
    out_fb, _ = m._mlp(None, layer, y)
    dense = b.moe_dense.clone()
    ye_fb = torch.empty((E, 64, H), dtype=BF16, device=DEV)
    act = torch.empty((64, I), dtype=BF16, device=DEV)
    for e in range(E):
        ops.silu_mul(torch.mm(y, gu_w[e].t()), act)
        ye_fb[e] = torch.mm(act, dn_w[e].t())
    torch.cuda.synchronize()
    _check_combine(out_fb, ye_fb, dense, 64)

    # one expert's outputs overflow: rows that did not select it stay finite, every row equals the reference loop
    e_big = _blow_up(moe, dense)
    keep = dense[:, e_big] == 0
    b2 = types.SimpleNamespace(rows=64, y=y)
    plans2 = m._layer_gemm_plans(layer, b2)
    out2, _ = m._mlp(None, layer, y, plans2, b=b2)
    out_fb2, _ = m._mlp(None, layer, y)
    torch.cuda.synchronize()
    assert not torch.isfinite(plans2['moe_down'].out[e_big, :64]).all()
    assert keep.any() and torch.isfinite(out2[keep]).all() and torch.isfinite(out_fb2[keep]).all()
    _check_combine(out2, plans2['moe_down'].out, b2.moe_dense, 64)
    ops.silu_mul(torch.mm(y, gu_w[e_big].t()), act)
    ye_fb[e_big] = torch.mm(act, dn_w[e_big].t())
    _check_combine(out_fb2, ye_fb, dense, 64)
    del m, layer, moe, gu_w, dn_w, plans, plans2, b, b2, ye_fb
    torch.cuda.empty_cache()

    # fp8 plans: the gate_up SiLU epilogue over the stacked weight, the grouped fp8 down, the same combine
    m2, layer2 = _mixtral_layer(shape, seed=7)
    m2.quantize_fp8()
    ex = layer2.mlp.experts
    qkv_n = layer2.self_attn.qkv_fp8.shape[0]
    b3 = types.SimpleNamespace(rows=64, y=y, qkv=torch.empty((64, qkv_n), dtype=BF16, device=DEV),
                               attn=torch.zeros((64, H), dtype=BF16, device=DEV),
                               fp8_out=torch.empty((64, H), dtype=BF16, device=DEV))
    n_sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    p3 = m2._layer_fp8_plans(layer2, b3, n_sm)
    out3, _ = m2._mlp(None, layer2, y, p3, b=b3)
    torch.cuda.synchronize()
    q, s = ex.down_proj.codes()
    ye3 = p3['moe_down'].out
    for e in range(E):
        _check_gemm(ye3[e], b3.moe_act[:, e * I:(e + 1) * I], q[e], I, f'fp8 down {e}', scale=s[e])
    _check_combine(out3, ye3, b3.moe_dense, 64)
    assert torch.equal(_bits(b3.moe_dense), _bits(dense))


@pytest.mark.gpu
def test_router_and_combine_cuda_graph_replay_the_eager_bits():
    ops = _ops()
    E, H, k = 8, 4096, 2
    y, gate = M.random_router_inputs(64, H, E, seed=5, device=DEV)
    ye = M.expert_outputs(E, 64, H, seed=6, device=DEV)
    dense, out = torch.empty((64, E), dtype=BF16, device=DEV), torch.empty((64, H), dtype=BF16, device=DEV)
    ops.moe_router(y, gate, k, dense)
    ops.moe_combine(ye, dense, out)
    torch.cuda.synchronize()
    want = (dense.clone(), out.clone())
    dense.zero_()
    out.zero_()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ops.moe_router(y, gate, k, dense)
            ops.moe_combine(ye, dense, out)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        dense.zero_()
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(dense), _bits(want[0])) and torch.equal(_bits(out), _bits(want[1]))
    assert _same(want[1], M.combine_ref(ye, want[0]))


@pytest.mark.gpu
def test_router_and_combine_refuse_bad_arguments():
    """E = 0 or 65, top_k = 0 or > E, hidden not a positive multiple of 8, rows > rows_cap: an error, no launch, the
    output untouched"""
    from painlessinferenceacceleration_b200 import _lib
    L = _lib.load()
    y = torch.ones((4, 4096), dtype=BF16, device=DEV)
    gate = torch.ones((65, 4096), dtype=BF16, device=DEV)
    ye = torch.ones((65, 8, 4096), dtype=BF16, device=DEV)
    w = torch.ones((8, 65), dtype=BF16, device=DEV)
    out = _sentinel((8, 4096), DEV)
    dense = _sentinel((4, 65), DEV)
    p = lambda t: t.data_ptr()   # noqa: E731
    router = [(4, 4096, 0, 1), (4, 4096, 65, 2), (4, 4096, 8, 0), (4, 4096, 8, 9), (4, 12, 8, 2), (4, 0, 8, 2),
              (0, 4096, 8, 2)]
    combine = [(0, 4, 8, 4096), (8, 9, 8, 4096), (8, 4, 8, 12), (8, 4, 8, 0), (8, 0, 8, 4096)]
    torch.cuda.synchronize()
    n0 = L.pia_launch_count()
    for rows, hidden, E, k in router:
        assert L.pia_moe_router(p(y), p(gate), rows, hidden, E, k, p(dense), None) != 0, (rows, hidden, E, k)
    for E, rows, cap, hidden in combine:
        assert L.pia_moe_combine(p(ye), p(w), E, rows, cap, hidden, p(out), None) != 0, (E, rows, cap, hidden)
    torch.cuda.synchronize()
    assert L.pia_launch_count() == n0
    assert (_bits(out) == SENT).all() and (_bits(dense) == SENT).all()
    with pytest.raises(AssertionError):
        _ops().moe_router(y, gate, 2, dense)
    with pytest.raises(AssertionError):
        _ops().moe_router(y, gate[:8], 9, dense[:, :8].contiguous())
