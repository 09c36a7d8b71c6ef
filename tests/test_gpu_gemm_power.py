# -*- coding: utf-8 -*-
"""Tests of the weight-streaming GEMMs (csrc/gemm_ws.cu: k_gemm_ws, k_gemm_stream, k_gemm_sk, k_gemm_fp8, k_gemm_w4)
that can fail: every plan path and every launched kernel instance chosen on purpose from the device's SM count,
exact-integer operands compared bit for bit (int4: power-of-two scales whose dequantised weight is exact), an fp64
reference with a scale-aware comparator (tests/gemm_ref.py), one-hot routing probes over every (n, k) pair, sentinels
around every output, a CUDA-graph chain in which a library kernel writes X right before each PDL-launched GEMM, and
(`big`) k_gemm_stream at the gate/up and lm_head shapes of 7B-13B models.

The first half runs without a GPU: it checks that the exactness check and the comparator accept an emulation of the
kernels' arithmetic and reject every wrong kernel of `gemm_ref.MUTATIONS`, that the stream-K fix-up workspace is sized
from the partition the kernel uses, that the case table reaches every path, and that it reaches every kernel instance
csrc/gemm_ws.cu launches."""
import os
import re
from collections import namedtuple

import pytest
import torch

from tests import gemm_ref as R

DEV = 'cuda:0'
N_SM = 132                  # H100 SXM; the GPU tests read the real count
ROWS = (1, 2, 3, 4, 5, 31, 33, 63, 64)
ROWS_F8 = (65, 127, 128, 200, 256)
GUARD = 1024                # output elements after the output that must stay untouched
SENT16, SENT32 = 0x7FA5, 0x7FA5A5A5   # NaN bit patterns no kernel writes

# kind: ws (pia_gemm_plan_create; split-1 plans without SiLU run k_gemm_stream), grouped (_create_grouped), sk
# (split -1), fp8 (_create_fp8), fp8grouped, w4 (_create_w4, or _create_grouped_w4 when groups > 1)
# split: the split_k argument; x_rows: rows of the activation buffer the plan is bound to; gs / f16: the int4 scale
# group (K: channel-wise) and scale dtype
Case = namedtuple('Case', 'kind N K split tiled groups silu x_rows gs f16', defaults=(128, False))


def cases(S):
    """the case table for a device with S SMs: the shapes that pick nstage 4 / 3 / 2, k_gemm_stream's 64- or 128-row
    tiles and the stream-K regimes follow S"""
    ws = lambda N, K, split=1, tiled=False, silu=False: Case('ws', N, K, split, tiled, 1, silu, 64)  # noqa: E731
    sk = lambda N, K: Case('sk', N, K, -1, True, 1, False, 64)  # noqa: E731
    f8 = lambda N, K, split=1, silu=False, x_rows=256: Case('fp8', N, K, split, True, 1, silu, x_rows)  # noqa: E731
    w4 = lambda N, K, split=1, gs=128, f16=False, silu=False, groups=1, x_rows=256: Case(  # noqa: E731
        'w4', N, K, split, True, groups, silu, x_rows, gs, f16)
    wide = 3 * S // 2                                   # 128-row tiles of the widest tiled k_gemm_stream<1,4> plan
    odd = 3 * S + 1 if (3 * S + 1) % 2 else 3 * S + 2   # 64-row tiles past 3 S, an odd count: N % 128 == 64
    return {
        'ws-row-split1-n200': ws(200, 512),
        'ws-tiled-split1-nstage4': ws(128 * (S + 4), 256, tiled=True),
        'ws-row-slices-even-n320': ws(320, 1024, 4),
        'ws-tiled-slices-uneven': ws(256, 448, 3, tiled=True),
        'ws-row-cluster2-n328': ws(328, 512, -2),
        'ws-tiled-cluster4': ws(512, 1024, -4, tiled=True),
        'ws-row-cluster8-n1000': ws(1000, 1024, -8),
        'ws-tiled-cluster8-nstage4': ws(128 * (S // 8 + 2), 1024, -8, tiled=True),
        'ws-silu': ws(512, 512, tiled=True, silu=True),
        'ws-grouped': Case('grouped', 256, 320, 1, False, 4, False, 64),
        'ws-grouped-nstage4': Case('grouped', 256, 128, 1, False, S // 2 + 1, False, 64),
        'sk-units-le-ctas': sk(256, 64 * (S // 2)),
        'sk-ratio-1-2': sk(128, 64 * (S + 1)),
        'sk-integer-ratio': sk(384, 64 * S),
        'sk-large-ratio': sk(4096, 64 * 65),
        'sk-qwen2.5-0.5b-down': sk(896, 4864),
        'sk-qwen2-1.5b-o': sk(1536, 1536),
        'f8-split1': f8(256, 512),
        'f8-cluster2': f8(256, 512, -2),
        'f8-cluster4': f8(384, 1024, -4),
        'f8-cluster8': f8(512, 1024, -8),
        'f8-slices-uneven': f8(256, 640, 2),
        'f8-silu': f8(512, 512, silu=True),
        'f8-grouped': Case('fp8grouped', 256, 384, 1, True, 3, False, 200),
        'f8-xrows200': f8(256, 256, x_rows=200),
        'f8-nstage3': f8(128 * (S + 2), 256, x_rows=64),
        # k_gemm_stream<1,4> while ceil(N / 64) <= 3 S, then <2,4>: both sides of the boundary, partial tiles
        'stream1-row-n192': ws(192, 512),
        'stream1-tiled-last-64-row-plan': ws(128 * wide, 256, tiled=True),
        'stream2-tiled-first-128-row-plan': ws(128 * (wide + 1), 256, tiled=True),
        'stream2-row-n%128=64': ws(64 * odd, 256),
        'stream2-row-n%64=40': ws(64 * 3 * S + 40, 256),
        # k_gemm_w4: nstage 4 / 2 x bf16 / fp16 scales x one group / grouped; group sizes 128, 256, 384 and K
        # (channel-wise); K % 256 == 128 (a last 128-k half chunk) under split 1, slices, a cluster and groups
        'w4-split1': w4(256, 512),
        'w4-split1-f16-g256': w4(384, 1024, gs=256, f16=True),
        'w4-nstage2': w4(128 * (S + 2), 256, x_rows=64),
        'w4-nstage2-f16-channel-half': w4(128 * (S + 2), 384, gs=384, f16=True, x_rows=64),
        'w4-cluster2-half': w4(256, 640, -2),
        'w4-cluster4-g256-f16': w4(384, 1024, -4, gs=256, f16=True),
        'w4-cluster8-g384-half': w4(256, 1920, -8, gs=384),
        'w4-slices-even-f16': w4(256, 1024, 4, f16=True),
        'w4-slices-uneven-channel': w4(256, 1280, 2, gs=1280),
        'w4-slices-channel-half-f16': w4(256, 896, 2, gs=896, f16=True),
        'w4-silu-g256': w4(512, 512, gs=256, silu=True),
        'w4-grouped-half': w4(256, 384, groups=3, x_rows=200),
        'w4-grouped-f16-g384': w4(128, 768, gs=384, f16=True, groups=4),
        'w4-grouped-nstage2-g256': w4(256, 256, gs=256, groups=S // 2 + 1, x_rows=64),
        'w4-grouped-nstage2-f16-half': w4(256, 384, f16=True, groups=S // 2 + 1, x_rows=64),
        'w4-xrows200-f16': w4(256, 256, f16=True, x_rows=200),
    }


def plan_of(c, S, bias=False):
    fp8 = c.kind.startswith('fp8')
    return R.plan(c.N, c.K, c.split, c.tiled, fp8=fp8, groups=c.groups, bias=bias, n_sm=S, silu=c.silu,
                  w4=c.kind == 'w4', group=c.gs, f16=c.f16)


def bias_modes(c, p):
    """fp8 and int4 plans that take a bias run with and without one"""
    return (False, True) if p.kind in ('fp8', 'w4') and (p.n_split == 1 or p.cluster) and not c.silu and \
        c.groups == 1 else (False,)


def rows_of(c):
    """row counts a case runs: 1..64, and up to x_rows (several 64-row token blocks) for fp8 and int4"""
    return [r for r in ROWS + (ROWS_F8 if c.kind.startswith('fp8') or c.kind == 'w4' else ()) if r <= c.x_rows]


def paths(c, S):
    """the paths one case reaches, by the plan rules"""
    p = plan_of(c, S)
    out = set()
    if p.kind == 'sk':
        U, G = p.tiles * p.n_chunks, p.sk_grid
        if U <= G:
            out.add(('sk', 'units <= CTAs'))
        elif U < 2 * G:
            out.add(('sk', '1 < units/CTAs < 2'))
        elif U % G == 0:
            out.add(('sk', 'integer ratio'))
        elif U > 8 * G:
            out.add(('sk', 'large non-integer ratio'))
        if (c.N, c.K) in ((896, 4864), (1536, 1536)):
            out.add(('sk', f'{c.N}x{c.K}'))
        return out
    if p.kind == 'stream':
        out.add(('stream', p.wg, 'tiled' if c.tiled else 'row-major'))
        if c.N % 64:
            out.add(('stream', p.wg, 'N % 64 != 0'))
        elif c.N % 128:
            out.add(('stream', p.wg, 'N % 128 == 64'))
        t = R._ceil(c.N, 64)
        if 3 * S - 2 < t <= 3 * S:
            out.add(('stream', 'last 64-row plan: ceil(N / 64) <= 3 S'))
        if 3 * S < t <= 3 * S + 2:
            out.add(('stream', 'first 128-row plan: ceil(N / 64) > 3 S'))
        return out
    k = p.kind
    if p.cluster:
        mode = f'cluster{p.cluster}'
    elif p.n_split == 1:
        mode = 'split1'
    else:
        mode = 'slices-uneven' if split_lengths(p)[-1] < split_lengths(p)[0] else 'slices-even'
    out |= {(k, mode), (k, 'nstage', p.nstage)}
    if k == 'ws':
        out.add((k, 'tiled' if c.tiled else 'row-major'))
        if c.N % 128:
            out.add((k, 'N % 128 != 0', mode if p.n_split == 1 or p.cluster else 'slices'))
        if p.groups > 1 and min(rows_of(c)) < 64:
            out.add((k, 'grouped rows < 64'))
    else:
        for b in bias_modes(c, p):
            out.add((k, mode, 'bias' if b else 'no bias'))
        if p.groups > 1:
            out.add((k, 'grouped'))
        out |= {(k, 'rows', r) for r in rows_of(c) if r > 64}
        if c.x_rows == 200:
            out.add((k, 'x_rows 200'))
    if k == 'w4':
        out.add((k, 'nstage', p.nstage, 'fp16' if p.f16 else 'bf16', 'grouped' if p.groups > 1 else 'one group'))
        out.add((k, 'group', 'channel' if p.group == p.K else p.group))
        if p.K % 256 == 128:
            out.add((k, 'K % 256 == 128', 'cluster' if p.cluster else 'slices' if p.n_split > 1 else
                     'grouped' if p.groups > 1 else 'split1'))
        if p.groups > 1 and max(rows_of(c)) > 64:
            out.add((k, 'grouped rows > 64'))
    if c.silu:
        out.add((k, 'silu'))
    return out


def split_lengths(p):
    return [c1 - c0 for c0, c1 in R.split_ranges(p)]


REQUIRED = ({('ws', m) for m in ('split1', 'slices-even', 'slices-uneven', 'cluster2', 'cluster4', 'cluster8',
                                 'tiled', 'row-major', 'silu', 'grouped rows < 64')} |
            {('ws', 'N % 128 != 0', m) for m in ('slices', 'cluster2', 'cluster8')} |
            {('stream', wg, m) for wg in (1, 2) for m in ('tiled', 'row-major', 'N % 128 == 64', 'N % 64 != 0')} |
            {('stream', 'last 64-row plan: ceil(N / 64) <= 3 S'),
             ('stream', 'first 128-row plan: ceil(N / 64) > 3 S')} |
            {('ws', 'nstage', 4), ('ws', 'nstage', 8)} |
            {('sk', r) for r in ('units <= CTAs', '1 < units/CTAs < 2', 'integer ratio', 'large non-integer ratio',
                                 '896x4864', '1536x1536')} |
            {('fp8', m, b) for m in ('split1', 'cluster2', 'cluster4', 'cluster8') for b in ('bias', 'no bias')} |
            {('fp8', m) for m in ('slices-uneven', 'silu', 'grouped', 'x_rows 200')} |
            {('fp8', 'rows', r) for r in ROWS_F8} | {('fp8', 'nstage', 3), ('fp8', 'nstage', 6)} |
            {('w4', m, b) for m in ('split1', 'cluster2', 'cluster4', 'cluster8') for b in ('bias', 'no bias')} |
            {('w4', m) for m in ('slices-even', 'slices-uneven', 'silu', 'grouped', 'grouped rows > 64',
                                 'x_rows 200')} |
            {('w4', 'rows', r) for r in ROWS_F8} |
            {('w4', 'nstage', n, sd, gr) for n in (2, 4) for sd in ('bf16', 'fp16')
             for gr in ('one group', 'grouped')} |
            {('w4', 'group', g) for g in (128, 256, 384, 'channel')} |
            {('w4', 'K % 256 == 128', m) for m in ('split1', 'slices', 'cluster', 'grouped')})


@pytest.mark.parametrize('S', [N_SM, 114])
def test_case_table_reaches_every_path(S):
    """on an H100 SXM (132 SMs) and PCIe (114 SMs) alike, the case table reaches every listed path"""
    cs = cases(S)
    got = set().union(*(paths(c, S) for c in cs.values()))
    assert REQUIRED <= got, sorted(REQUIRED - got)


GEMM_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       'painlessinferenceacceleration_b200', 'csrc', 'gemm_ws.cu')


def launch_sites(path=GEMM_CU):
    """the kernel instances csrc/gemm_ws.cu launches (launch_kernel / launch_kernel_cluster sites), spelled as
    gemm_ref.instance spells them: no spaces, defaulted template arguments written out"""
    out = set()
    for name, args in re.findall(r'launch_kernel(?:_cluster)?\(\s*(k_gemm_\w+)(?:<([^>]*)>)?', open(path).read()):
        a = [t.strip() for t in args.split(',')] if args else []
        if name == 'k_gemm_w4' and len(a) == 2:
            a.append('false')   # GROUPED = false
        out.add(name + (f'<{",".join(a)}>' if a else ''))
    return out


def test_case_table_reaches_every_launched_kernel_instance():
    """every kernel instance pia_gemm_run launches has a case at 132 SMs (a kernel that lands without cases fails
    here), and the plan model names no instance the library does not launch"""
    sites = launch_sites()
    assert {'k_gemm_sk', 'k_gemm_ws<8>', 'k_gemm_stream<1,4>', 'k_gemm_stream<2,4>', 'k_gemm_fp8<3>',
            'k_gemm_w4<2,true,false>', 'k_gemm_w4<4,false,true>'} <= sites, sites
    assert len(sites) == 15, sorted(sites)
    reached = {R.instance(plan_of(c, N_SM, b)) for c in cases(N_SM).values() for b in bias_modes(c, plan_of(c, N_SM))}
    assert sites <= reached, sorted(sites - reached)
    assert reached <= sites, sorted(reached - sites)


def test_stream_instance_follows_the_row_count_alone():
    """k_gemm_stream<1,4> while ceil(N / 64) <= 3 S, <2,4> beyond, whatever the split-1 stage count k_gemm_ws would
    use; <2,8> would need ceil(N / 64) > 3 S and ceil(N / 128) <= S at once, which no S allows"""
    for S in (114, 132):
        for N in (64 * 3 * S - 63, 64 * 3 * S, 64 * 3 * S + 1, 128 * S, 128 * S + 1, 64 * 3 * S + 64 * S):
            for tiled in (False, True):
                if tiled and N % 128:
                    continue
                p = R.plan(N, 256, 1, tiled, n_sm=S)
                assert R.instance(p) == f'k_gemm_stream<{1 if R._ceil(N, 64) <= 3 * S else 2},4>', (S, N)
                assert not (R._ceil(N, 64) > 3 * S and R._ceil(N, 128) <= S)


@pytest.mark.parametrize('kw', [dict(N=192, K=256), dict(N=256, K=192, group=64), dict(N=256, K=256, group=64),
                                dict(N=256, K=256, group=96), dict(N=256, K=512, group=384),
                                dict(N=256, K=640, split_k=-4), dict(N=256, K=640, split_k=2, bias=True),
                                dict(N=256, K=640, split_k=0), dict(N=256, K=256, groups=2, split_k=2),
                                dict(N=256, K=256, groups=2, bias=True), dict(N=256, K=512, split_k=2, silu=True),
                                dict(N=256, K=512, bias=True, silu=True), dict(N=256, K=512, groups=2, silu=True)])
def test_plan_model_refuses_what_the_int4_library_refuses(kw):
    """pia_gemm_plan_create_w4 / _grouped_w4 / set_silu refuse these (PIA_ERR_INVALID, test_gpu_w4 and
    test_gpu_w4_mixtral check the library); the model raises ValueError"""
    with pytest.raises(ValueError):
        R.plan(w4=True, **kw)


# ---------------------------------------------------------------------------------------------------------------
# detection power, the stream-K workspace, on the CPU
# ---------------------------------------------------------------------------------------------------------------
SELF = {   # (plan arguments, inputs): one plan per mutation family
    'cluster4': (dict(N=256, K=1024, split_k=-4, tiled=True), {}),
    'slices-uneven': (dict(N=256, K=448, split_k=3, tiled=True), {}),
    'fp8-cluster2-bias': (dict(N=256, K=512, split_k=-2, fp8=True, bias=True), dict(fp8=True, bias=True)),
    'fp8-slices': (dict(N=256, K=640, split_k=2, fp8=True), dict(fp8=True)),
    'grouped': (dict(N=128, K=192, groups=3), dict(groups=3)),
    'stream-K 133/132': (dict(N=128, K=64 * 133, split_k=-1, tiled=True), {}),
    'row-major N=200': (dict(N=200, K=512), {}),
    'stream1-tiled': (dict(N=256, K=256, tiled=True), {}),
    'w4-cluster2-bias-f16-half': (dict(N=256, K=640, split_k=-2, w4=True, f16=True, bias=True), dict(bias=True)),
    'w4-slices-g384-half': (dict(N=128, K=1152, split_k=2, w4=True, group=384), {}),
    'w4-grouped-half': (dict(N=128, K=384, groups=3, w4=True), dict(groups=3)),
}


def _exact(p, rows, gen, bias=False, device='cpu'):
    """exact-integer operands for plan p (tests/gemm_ref.py), int4 codes for an int4 plan"""
    if p.kind == 'w4':
        return R.exact_operands_w4(rows, p.N, p.K, p.group, gen, groups=p.groups, f16=p.f16, bias=bias,
                                   device=device)
    return R.exact_operands(rows, p.N, p.K, gen, groups=p.groups, fp8=p.kind == 'fp8', bias=bias, device=device)


def _random_operands(p, gen, fp8=False, bias=False, groups=1, rows=64):
    """the old tests' inputs: x ~ N(0, 1), w ~ 0.05 N(0, 1) bf16, or fp8 quantised 0.02 N(0, 1) with a 2 N(0, 1) bias;
    int4: uniform codes, zero points 0..16, scales 0.01 .. 0.03 in the plan's scale dtype, the same bias"""
    from painlessinferenceacceleration_b200.common import ops
    x = torch.randn((rows, groups * p.K), generator=gen).to(torch.bfloat16)
    if p.kind == 'w4':
        ng = p.K // p.group
        u = torch.randint(0, 16, (groups, p.N, p.K), generator=gen).to(torch.uint8)
        s = (0.01 + 0.02 * torch.rand((groups, p.N, ng), generator=gen)).to(torch.float16 if p.f16 else torch.bfloat16)
        z = torch.randint(0, 17, (groups, p.N, ng), generator=gen).to(torch.uint8)
        b = (2 * torch.randn(p.N, generator=gen)).to(torch.bfloat16).float() if bias else None
        return x, R.W4(u, s, z, p.group), None, b
    if not fp8:
        return x, (0.05 * torch.randn((groups, p.N, p.K), generator=gen)).to(torch.bfloat16), None, None
    q, s = ops.quantize_fp8(0.02 * torch.randn((groups, p.N, p.K), generator=gen))
    b = (2 * torch.randn(p.N, generator=gen)).to(torch.bfloat16).float() if bias else None
    return x, q, s.reshape(-1), b


def _refs(p, x, w, s, b):
    w = R.dense(w)
    rm = [R.reference(x[:, g * p.K:(g + 1) * p.K], w[g], None if s is None else s[g * p.N:(g + 1) * p.N], b)
          for g in range(p.groups)]
    if p.groups == 1:
        return rm[0]
    return torch.stack([r for r, _ in rm]), torch.stack([m for _, m in rm])


def _verdicts(p, x, w, s, b, out, exact):
    """(passes, old tolerance passes): exact operands bit for bit, random ones through the comparator"""
    ref, mass = _refs(p, x, w, s, b)
    slices = p.n_split > 1 and not p.cluster
    if exact:
        want = R.exact_slices(p, x, w, s) if slices else R.bf16_exact(ref)
        ok = torch.equal(out.double(), want.double()) and (slices or torch.equal(out.view(torch.int16),
                                                                                 want.view(torch.int16)))
        return ok, None
    got = R.slice_sum(out) if slices else out
    return R.worst(got, ref, mass, p.K, p.n_split) <= 1.0, R.old_close(got, ref)


def test_checks_accept_the_kernel_arithmetic_and_reject_every_mutation():
    """the emulated kernels pass the exactness check and the comparator; every wrong kernel fails at least one of
    them on these inputs.  Prints which wrong kernels the old allclose(atol=2e-2, rtol=1.6e-2) accepted."""
    seen, old_accepts = set(), set()
    for name, (pa, kw) in SELF.items():
        p = R.plan(**pa)
        gen = torch.Generator().manual_seed(len(name))
        ops_x = _exact(p, 64, gen, bias=kw.get('bias', False))
        ops_r = _random_operands(p, gen, **kw)
        for operands, exact in ((ops_x, True), (ops_r, False)):
            ok, _ = _verdicts(p, *operands, R.emulate(p, *operands), exact)
            assert ok, (name, 'emulation', 'exact' if exact else 'random')
        for m in R.mutation_names(p):
            seen.add(m)
            ok_x, _ = _verdicts(p, *ops_x, R.emulate(p, *ops_x, mut=m), True)
            ok_r, old = _verdicts(p, *ops_r, R.emulate(p, *ops_r, mut=m), False)
            assert not (ok_x and ok_r), f'{name}: the checks accept the wrong kernel "{m}"'
            if old:
                old_accepts.add(m)
    assert seen == set(R.MUTATIONS)
    print(f'\nGEMM-POWER wrong kernels the old tolerance accepts: {sorted(old_accepts)}')
    # the two rounding faults hide inside one bf16 rounding of the old tolerance; the comparator and the exact
    # operands do not let them through
    assert {'round toward zero (__float2bfloat16_rz)', 'cluster partials rounded to bf16 before the sum'} <= old_accepts


@pytest.mark.parametrize('N,K,old,needed', [(896, 4864, 17, 19), (1536, 1536, 9, 10), (128, 8512, 68, 131)])
def test_stream_k_slots_sized_from_the_partition(N, K, old, needed):
    """on 132 SMs the old fix-up slot count ceil(n_chunks / ceil(U / G)) + 1 is short of the contributor slots the
    kernel writes (ranges of floor(U / G) units let a tile span more CTAs); the plan now counts them per tile.  Every
    contributor's slot b - owner - 1 is below the count, and each tile's segments tile its chunks exactly."""
    tiles, chunks = N // 128, K // 64
    p = R.plan(N, K, -1, True, n_sm=N_SM)
    assert (p.tiles * p.n_chunks, p.sk_grid) == (tiles * chunks, min(tiles * chunks, N_SM))
    assert R.sk_slots_old(tiles, chunks, p.sk_grid) == old < needed == R.sk_slots_needed(tiles, chunks, p.sk_grid)
    U = tiles * chunks
    for t in range(tiles):
        segs = R.sk_segments(t, chunks, U, p.sk_grid)
        assert segs[0][1] == 0 and segs[-1][2] == chunks and all(a[2] == b[1] for a, b in zip(segs, segs[1:]))
        assert all(b - segs[0][0] - 1 < needed for b, _, _ in segs[1:])


def test_stream_k_slots_of_the_case_table():
    """the stream-K cases include shapes the old slot count was short for, on 132 SMs"""
    short = [n for n, c in cases(N_SM).items() if c.kind == 'sk' and
             R.sk_slots_old(c.N // 128, c.K // 64, plan_of(c, N_SM).sk_grid) <
             R.sk_slots_needed(c.N // 128, c.K // 64, plan_of(c, N_SM).sk_grid)]
    assert set(short) >= {'sk-ratio-1-2', 'sk-qwen2.5-0.5b-down', 'sk-qwen2-1.5b-o'}, short


# ---------------------------------------------------------------------------------------------------------------
# the kernels on the H100
# ---------------------------------------------------------------------------------------------------------------
def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _deinterleave(v):
    """columns of a SiLU-interleaved GEMM output (per 128: 64 gate, 64 up) -> [gate | up]"""
    r, n = v.shape
    t = v.view(r, n // 128, 2, 64)
    return torch.cat([t[:, :, 0].reshape(r, -1), t[:, :, 1].reshape(r, -1)], 1).contiguous()


class _Rig(object):
    """one case's plan bound to fixed buffers (the plan holds their addresses), an output with a guard band"""

    def __init__(self, c, S, bias):
        ops = self.ops = _ops()
        self.c, self.fp8, self.w4, G, N, K = c, c.kind.startswith('fp8'), c.kind == 'w4', c.groups, c.N, c.K
        self.p = plan_of(c, S, bias)
        self.x = torch.zeros((c.x_rows, G * K), dtype=torch.bfloat16, device=DEV)
        self.bias = torch.zeros(N, device=DEV) if bias else None
        if self.w4:
            self.codes = torch.zeros((G * N // 128, R._ceil(K, 256), 128, 128), dtype=torch.uint8, device=DEV)
            self.st = torch.ones((K // c.gs, G * N), dtype=torch.float16 if c.f16 else torch.bfloat16, device=DEV)
            self.zt = torch.zeros((K // c.gs, G * N), dtype=torch.uint8, device=DEV)
            if G > 1:
                self.g = ops.Gemm.grouped_w4(self.codes, self.st, self.zt, c.gs, G, self.x)
            else:
                self.g = ops.Gemm.w4(self.codes, self.st, self.zt, c.gs, self.x, bias=self.bias, split_k=c.split)
            self.plain = ops.Gemm.w4(self.codes, self.st, self.zt, c.gs, self.x) if c.silu else None
        elif self.fp8:
            self.wq = torch.zeros(((G,) if G > 1 else ()) + (N // 128, K // 128, 128, 128), dtype=torch.uint8,
                                  device=DEV)
            self.scale = torch.ones(G * N, device=DEV)
            if G > 1:
                self.g = ops.Gemm.grouped_fp8(self.wq, self.scale, self.x)
            else:
                self.g = ops.Gemm.fp8(self.wq, self.scale, self.x, bias=self.bias, split_k=c.split)
            self.plain = ops.Gemm.fp8(self.wq, self.scale, self.x) if c.silu else None
        else:
            self.w = torch.zeros((G, N, K), dtype=torch.bfloat16, device=DEV)
            if G > 1:
                self.g = ops.Gemm.grouped(self.w, self.x)
            else:
                self.wt = ops.tile_weight(self.w[0]) if c.tiled else self.w[0]
                self.g = ops.Gemm(self.wt, self.x, split_k=c.split, tiled=c.tiled)
            self.plain = ops.Gemm(self.wt, self.x, tiled=True) if c.silu else None
        if c.silu:
            self.g.set_silu()
        assert self.g.splits == R.splits_reported(self.p), (self.g.splits, self.p)
        self.slices = self.p.n_split > 1 and not self.p.cluster
        cap = c.x_rows if self.fp8 or self.w4 else 64
        cols = N // 2 if c.silu else N
        self.shape = (G, cap, cols) if G > 1 else ((self.p.n_split, cap, cols) if self.slices else (cap, cols))
        self.n = G * cap * cols * (self.p.n_split if self.slices else 1)
        self.dt, self.it, self.sent = ((torch.float32, torch.int32, SENT32) if self.slices else
                                       (torch.bfloat16, torch.int16, SENT16))
        self.buf = torch.empty(self.n + GUARD, dtype=self.dt, device=DEV)

    def load(self, x, w, scale, bias):
        """x [x_rows, G K], w [G, N, K] (bf16 / e4m3, or int4 W4 codes), scale [G N], bias [N]"""
        ops = self.ops
        self.x.copy_(x)
        if self.w4:
            G, N, K = w.u.shape
            self.codes.copy_(ops.tile_weight_w4(w.u.reshape(G * N, K).to(DEV)))
            self.st.copy_(w.s.reshape(G * N, -1).t())
            self.zt.copy_(w.z.reshape(G * N, -1).t())
            if self.bias is not None:
                self.bias.copy_(bias)
            w = R.W4(*(t.to(DEV) for t in w[:3]), w.group)
        elif self.fp8:
            self.wq.copy_(ops.tile_weight_fp8(w.to(DEV)).view(self.wq.shape))
            self.scale.copy_(scale)
            if self.bias is not None:
                self.bias.copy_(bias)
        else:
            self.w.copy_(w)
            if self.c.tiled and self.c.groups == 1:
                self.wt.copy_(ops.tile_weight(self.w[0]))
        self.ops_in = (x.to(DEV), w if self.w4 else w.to(DEV), None if scale is None else scale.to(DEV),
                       None if self.bias is None else bias.to(DEV))

    def sentinel(self):
        b = torch.empty_like(self.buf)
        b.view(self.it).fill_(self.sent)
        return b

    def launch(self, rows, g=None):
        self.buf.view(self.it).fill_(self.sent)
        (g or self.g).run(rows, out=self.buf[:self.n].view(self.shape))
        torch.cuda.synchronize()
        return self.buf.clone()

    def view(self, buf, rows):
        return buf[:self.n].view(self.shape)[..., :rows, :]

    def expected(self, rows):
        """the exact output of exact-integer operands, inside a sentinel buffer"""
        p, c = self.p, self.c
        x, w, s, b = self.ops_in
        ref, _ = _refs(p, x[:rows], w, s, b)
        if self.slices:
            want = R.exact_slices(p, x[:rows], w, s).float()
        elif c.silu:
            gu = _deinterleave(R.bf16_exact(ref))
            want = torch.empty((rows, c.N // 2), dtype=torch.bfloat16, device=DEV)
            self.ops.silu_mul(gu, want)
        else:
            want = R.bf16_exact(ref)
        e = self.sentinel()
        self.view(e, rows).copy_(want)
        return e

    def untouched(self, got, rows):
        """everything but the live rows still holds the sentinel"""
        e, g = self.sentinel(), got.clone()
        self.view(g, rows).copy_(self.view(e, rows))
        return torch.equal(g.view(self.it), e.view(self.it))


def _case_params():
    return [pytest.param(k, marks=pytest.mark.gpu) for k in cases(N_SM)]


WORST = {}


@pytest.mark.parametrize('name', _case_params())
def test_gemm_case(name):
    """exact-integer operands bit for bit at every row count (a stream-K plan relaunched at changing row counts also
    shows that its fix-up flags reset themselves), rows past `rows`, the guard band after the output and the other
    groups' rows untouched; random operands through the comparator; a relaunch and a launch without PDL repeat the
    bits"""
    S = _n_sm()
    c = cases(S)[name]
    p0 = plan_of(c, S)
    for bias in bias_modes(c, p0):
        r = _Rig(c, S, bias)
        p = r.p
        gen = torch.Generator().manual_seed(c.N + 7 * c.K + c.groups + bias)
        r.load(*_exact(p, c.x_rows, gen, bias=bias))
        for rows in rows_of(c):
            got = r.launch(rows)
            want = r.expected(rows)
            if not torch.equal(got.view(r.it), want.view(r.it)):
                live = torch.equal(r.view(got, rows).view(r.it), r.view(want, rows).view(r.it))
                assert False, f'{name} bias={bias} rows {rows}: live rows exact {live}, untouched {r.untouched(got, rows)}'
        rows = max(rows_of(c))
        xr, wr, sr, br = _random_operands(p, gen, fp8=r.fp8, bias=bias, groups=c.groups, rows=c.x_rows)
        r.load(xr, wr, sr, br)
        base = r.launch(rows)
        assert r.untouched(base, rows)
        assert torch.equal(r.launch(rows).view(r.it), base.view(r.it)), 'relaunch differs'
        r.g.set_pdl(False)
        assert torch.equal(r.launch(rows).view(r.it), base.view(r.it)), 'PDL off differs from PDL on'
        r.g.set_pdl(True)
        x, w, s, b = r.ops_in
        if c.silu:   # the plain GEMM of the same weight through the comparator, the SiLU epilogue = pia_silu_mul of it
            plain = r.plain.run(rows)[:rows].clone()
            ref, mass = _refs(p, x[:rows], w, s, b)
            score = R.assert_close(plain, ref, mass, c.K, 1, name)
            want = torch.empty((rows, c.N // 2), dtype=torch.bfloat16, device=DEV)
            r.ops.silu_mul(_deinterleave(plain), want)
            torch.cuda.synchronize()
            assert torch.equal(r.view(base, rows), want)
        else:
            ref, mass = _refs(p, x[:rows], w, s, b)
            got = r.view(base, rows)
            if r.slices:
                got = R.slice_sum(got)
            score = R.assert_close(got, ref, mass, c.K, p.n_split, f'{name} bias={bias}')
        kern = R.instance(p)
        WORST[kern] = max(WORST.get(kern, 0.0), score)
        print(f'\nGEMM-POWER {name} bias={bias}: {R.describe(p)} paths {sorted(map(str, paths(c, S)))} '
              f'worst score {score:.3f} (per kernel so far {WORST})')


@pytest.mark.gpu
@pytest.mark.parametrize('layout,N,K,split', [('row-major', 200, 512, 1), ('tiled', 256, 640, 1),
                                              ('row-major cluster4', 328, 1024, -4), ('fp8 tiled', 256, 512, 1)])
def test_one_hot_routing_probe(layout, N, K, split):
    """X row t one-hot at k = 64 c + t, c over every 64-k offset: out[t, n] == W[n, 64 c + t] bit for bit, so every
    (n, k) pair of the weight is routed to its place once (swizzle, descriptor and tiling errors show up here)"""
    ops = _ops()
    gen = torch.Generator().manual_seed(N + K)
    x = torch.zeros((64, K), dtype=torch.bfloat16, device=DEV)
    out = torch.empty((64, N), dtype=torch.bfloat16, device=DEV)
    if layout.startswith('fp8'):
        codes = torch.randint(0, 256, (N, K), generator=gen, dtype=torch.uint8)
        codes[(codes & 0x7F) == 0x7F] = 0x38            # no NaN codes
        q = codes.view(torch.float8_e4m3fn)
        scale = torch.pow(2.0, (torch.arange(N) % 5 - 2).float())
        want_w = (q.float() * scale[:, None]).to(torch.bfloat16).to(DEV)   # exact: e4m3 x 2^j is a bf16 value
        assert torch.equal(want_w.double().cpu(), q.float().double() * scale.double()[:, None])
        g = ops.Gemm.fp8(ops.tile_weight_fp8(q.to(DEV)), scale.to(DEV), x, out=out)
    else:
        w = torch.randn((N, K), generator=gen).to(torch.bfloat16).to(DEV)
        want_w = w
        g = ops.Gemm(ops.tile_weight(w) if layout == 'tiled' else w, x, split_k=split, tiled=layout == 'tiled')
    _probe(g, x, out, want_w[None], K)


def _probe(g, x, out, want_w, K):
    """run the one-hot probe: x [64, G K] one-hot at k = 64 c + t in every group's columns, out [G, 64, N] (or [64, N])
    must hold want_w[g, n, 64 c + t] bit for bit for every offset c"""
    G = want_w.shape[0]
    o3 = out.view(G, 64, -1)
    for c in range(K // 64):
        x.copy_(R.onehot_x(K, c, device=DEV).repeat(1, G))
        out.fill_(7.0)
        g.run(64, out=out)
        torch.cuda.synchronize()
        for gi in range(G):
            want = want_w[gi, :, 64 * c:64 * c + 64].t()
            nz = want != 0      # a -0 weight comes out as +0 (the accumulator starts at +0)
            assert torch.equal(o3[gi].view(torch.int16)[nz], want.view(torch.int16)[nz]), f'group {gi} offset {c}'
            assert (o3[gi][~nz] == 0).all(), f'group {gi} offset {c}'


@pytest.mark.gpu
@pytest.mark.parametrize('layout', ['tiled', 'row-major'])
def test_one_hot_routing_probe_past_the_stream_boundary(layout):
    """k_gemm_stream<2,4> (128-row tiles) with N just past ceil(N / 64) = 3 S: the tiled weight in 16 KB blocks, and
    a row-major weight whose last tile holds 40 rows"""
    ops = _ops()
    S = _n_sm()
    N, K = (128 * (3 * S // 2 + 1), 256) if layout == 'tiled' else (64 * 3 * S + 40, 256)
    assert R.instance(R.plan(N, K, 1, layout == 'tiled', n_sm=S)) == 'k_gemm_stream<2,4>'
    gen = torch.Generator(device=DEV).manual_seed(N + K)
    w = torch.randn((N, K), generator=gen, device=DEV).to(torch.bfloat16)
    x = torch.zeros((64, K), dtype=torch.bfloat16, device=DEV)
    out = torch.empty((64, N), dtype=torch.bfloat16, device=DEV)
    g = ops.Gemm(ops.tile_weight(w) if layout == 'tiled' else w, x, tiled=layout == 'tiled')
    _probe(g, x, out, w[None], K)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['group256', 'channelwise-k896-fp16', 'nstage2', 'grouped-fp16'])
def test_one_hot_routing_probe_w4(name):
    """k_gemm_w4 with X one-hot: out[t, n] == the dequantised W[n, 64 c + t] bit for bit, every (n, k) pair once, at
    group size 256, channel-wise scales with a last half chunk (Qwen2.5-0.5B's K = 896), nstage 2, and grouped
    (every expert's own codes, table columns and X columns)"""
    ops = _ops()
    S = _n_sm()
    N, K, gs, f16, G = {'group256': (256, 512, 256, False, 1), 'channelwise-k896-fp16': (256, 896, 896, True, 1),
                        'nstage2': (128 * (S + 1), 256, 128, False, 1), 'grouped-fp16': (128, 384, 128, True, 3)}[name]
    p = R.plan(N, K, groups=G, w4=True, group=gs, f16=f16, n_sm=S)
    assert p.nstage == (2 if name == 'nstage2' else 4)
    gen = torch.Generator().manual_seed(N + K)
    sdt = torch.float16 if f16 else torch.bfloat16
    q = R.W4(torch.randint(0, 16, (G, N, K), generator=gen).to(torch.uint8),
             (0.001 + 0.05 * torch.rand((G, N, K // gs), generator=gen)).to(sdt),
             torch.randint(0, 17, (G, N, K // gs), generator=gen).to(torch.uint8), gs)
    want_w = R.dequant_w4(q).to(DEV)
    codes = ops.tile_weight_w4(q.u.reshape(G * N, K).to(DEV))
    st, zt = (t.reshape(G * N, -1).t().contiguous().to(DEV) for t in (q.s, q.z))
    x = torch.zeros((64, G * K), dtype=torch.bfloat16, device=DEV)
    g = ops.Gemm.grouped_w4(codes, st, zt, gs, G, x) if G > 1 else ops.Gemm.w4(codes, st, zt, gs, x)
    _probe(g, x, g.out, want_w, K)


@pytest.mark.gpu
def test_graph_chain_library_kernel_writes_x_before_each_pdl_gemm():
    """three steps captured in one CUDA graph; in each, pia_embed_gather writes X (integer table rows) right before a
    PDL-launched GEMM reads it: a bf16 GEMM (exact), then an fp32 split-K slices GEMM followed by
    pia_rmsnorm_partials, whose residual_out must equal torch's bf16(bf16(sum of slices) + r) bit for bit.  The graph
    is replayed twice with new ids; every step's outputs are checked against their own exact reference."""
    ops = _ops()
    gen = torch.Generator().manual_seed(11)
    V, K, N1, H, steps = 96, 1024, 384, 512, 3
    xt, w1, _, _ = R.exact_operands(V, N1, K, gen)
    _, w2, _, _ = R.exact_operands(1, H, K, gen)
    table, w1, w2 = xt.to(DEV), w1[0].to(DEV), w2[0].to(DEV)
    xa = torch.zeros((64, K), dtype=torch.bfloat16, device=DEV)
    xb = torch.zeros((64, K), dtype=torch.bfloat16, device=DEV)
    g1 = ops.Gemm(ops.tile_weight(w1), xa, tiled=True)
    g2 = ops.Gemm(w2, xb, split_k=3)
    p2 = R.plan(H, K, 3)
    assert g2.splits == p2.n_split == 3 and split_lengths(p2) == [6, 6, 4]
    ids = torch.zeros((steps, 2, 64), dtype=torch.int32, device=DEV)
    n = torch.full((1,), 64, dtype=torch.int32, device=DEV)
    resid = (torch.randint(-300, 300, (steps, 64, H), generator=gen).float()).to(torch.bfloat16).to(DEV)
    nw = torch.ones(H, dtype=torch.bfloat16, device=DEV)
    y1 = torch.empty((steps, 64, N1), dtype=torch.bfloat16, device=DEV)
    sl = torch.empty((steps, 3, 64, H), dtype=torch.float32, device=DEV)
    r_out = torch.empty((steps, 64, H), dtype=torch.bfloat16, device=DEV)
    y_out = torch.empty((steps, 64, H), dtype=torch.bfloat16, device=DEV)

    def step(s):
        ops.embed_gather(table, ids[s, 0], n, xa)
        g1.run(64, out=y1[s])
        ops.embed_gather(table, ids[s, 1], n, xb)
        g2.run(64, out=sl[s])
        ops.rmsnorm_partials(sl[s], resid[s], nw, 1e-6, r_out[s], y_out[s])

    ids.copy_(torch.randint(0, V, ids.shape, generator=gen))
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for s in range(steps):   # warm-up outside the capture
            step(s)
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for s in range(steps):
            step(s)
    for rep in range(2):
        ids.copy_(torch.randint(0, V, ids.shape, generator=gen))
        for t in (y1, sl, r_out):
            t.view(torch.uint8).fill_(0xA5)
        graph.replay()
        torch.cuda.synchronize()
        for s in range(steps):
            xa_s, xb_s = table[ids[s, 0].long()], table[ids[s, 1].long()]
            ref1, _ = R.reference(xa_s, w1)
            assert torch.equal(y1[s].view(torch.int16), R.bf16_exact(ref1).view(torch.int16)), (rep, s)
            want = R.exact_slices(p2, xb_s, w2[None]).float()
            assert torch.equal(sl[s], want), (rep, s)
            want_r = (want.sum(0).to(torch.bfloat16) + resid[s])   # three exact integer slices: any order is exact
            assert torch.equal(r_out[s].view(torch.int16), want_r.view(torch.int16)), (rep, s)


# ---------------------------------------------------------------------------------------------------------------
# big: k_gemm_stream<2,4> at model shapes
# ---------------------------------------------------------------------------------------------------------------
# (label, N, K, tiled): the split-1 bf16 gate/up of 7B-13B models (Llama-3-8B and Mistral-7B, Qwen2-7B, Llama-2-13B)
# and lm_heads of 32000 .. 151936 rows, all past 3 S 64-row tiles on 114 and 132 SMs; a 32001-row vocabulary is not a
# multiple of 128, so its weight stays row-major and the last 128-row tile holds one row
STREAM_SHAPES = [('gate_up-28672x4096', 28672, 4096, True), ('gate_up-37888x3584', 37888, 3584, True),
                 ('gate_up-27648x5120', 27648, 5120, True), ('lm_head-32000x4096', 32000, 4096, True),
                 ('lm_head-32768x4096', 32768, 4096, True), ('lm_head-64000x4096', 64000, 4096, True),
                 ('lm_head-65024x4096', 65024, 4096, True), ('lm_head-125696x4096', 125696, 4096, True),
                 ('lm_head-128256x4096', 128256, 4096, True), ('lm_head-151936x3584', 151936, 3584, True),
                 ('lm_head-32001x4096-row-major', 32001, 4096, False)]


@pytest.mark.gpu
@pytest.mark.big
@pytest.mark.parametrize('name,N,K,tiled', STREAM_SHAPES, ids=[s[0] for s in STREAM_SHAPES])
def test_stream_at_model_shapes(name, N, K, tiled):
    """random operands generated on the device against fp64 through the comparator at 1, 37 and 64 rows; the rows past
    `rows` and a guard band after the output keep their sentinel"""
    ops = _ops()
    S = _n_sm()
    p = R.plan(N, K, 1, tiled, n_sm=S)
    assert R.instance(p) == 'k_gemm_stream<2,4>', R.describe(p)
    gen = torch.Generator(device=DEV).manual_seed(N + K)
    w = (0.05 * torch.randn((N, K), generator=gen, device=DEV)).to(torch.bfloat16)
    x = torch.randn((64, K), generator=gen, device=DEV).to(torch.bfloat16)
    g = ops.Gemm(ops.tile_weight(w) if tiled else w, x, tiled=tiled)
    buf = torch.empty(64 * N + GUARD, dtype=torch.bfloat16, device=DEV)
    out = buf[:64 * N].view(64, N)
    score = 0.0
    for rows in (1, 37, 64):
        buf.view(torch.int16).fill_(SENT16)
        g.run(rows, out=out)
        torch.cuda.synchronize()
        assert (out[rows:].view(torch.int16) == SENT16).all() and (buf[64 * N:].view(torch.int16) == SENT16).all()
        for n0 in range(0, N, 16384):
            ref, mass = R.reference(x[:rows], w[n0:n0 + 16384])
            score = max(score, R.assert_close(out[:rows, n0:n0 + 16384], ref, mass, K, 1, f'{name} rows {rows}'))
    print(f'\nGEMM-POWER {name}: {R.describe(p)} worst score {score:.3f}')
