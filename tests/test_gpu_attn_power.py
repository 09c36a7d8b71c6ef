# -*- coding: utf-8 -*-
"""Tests of k_tree_attn that can fail: every KV-split / tile / head-layout path chosen on purpose, an fp64 reference
with a scale-aware comparator (tests/attn_ref.py), beacon inputs on which single-key errors are large, and exact
invariance - what a row must not see cannot change its output by a single bit.

The first half runs without a GPU: it checks that the comparator accepts an emulation of the kernel's arithmetic and
rejects every wrong rule of `attn_ref.mutations`, so a pass on the H100 means something."""
import ctypes as C
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

from tests import attn_ref as A

DEV = 'cuda:0'
SQ2, SQ80 = math.sqrt(2.0), math.sqrt(128.0 / 80.0)   # scale_mul of head dim 64 / 80 on the 128 kernel (BLOOM, GPT-2)
N_SM = 132                                            # H100 SXM; the GPU tests read the real count

# mode: plain (pia_tree_attn_fwd), fused (pia_tree_attn_fused_fwd), alibi (pia_tree_attn_alibi_fwd, D = 128);
# k: AttnPlan(kv_split_max=k); tpc: PIA_ATTN_TILES_PER_CTA (None: unset); slots: (n, P, pad) per request slot
Case = namedtuple('Case', 'mode D R Hq Hkv k tpc scale slots')
CASES = {
    'mha8-p3968': Case('plain', 128, 64, 8, 8, 0, None, 1.0, [(64, 3968, 5)]),
    'gqa4-pad-covers-split': Case('plain', 64, 64, 32, 8, 8, None, 1.0, [(33, 1000, 300)]),
    'g3-root-only-empty': Case('plain', 128, 64, 6, 2, 1, None, SQ2, [(1, 0, 0)]),
    'mha40-3split': Case('fused', 128, 64, 40, 40, 0, None, 1.0, [(64, 1000, 1)]),
    'g2-l127': Case('fused', 64, 64, 8, 4, 2, None, 1.0, [(64, 63, 0)]),
    'alibi-mha5-5split': Case('alibi', 128, 64, 5, 5, 5, None, SQ2, [(33, 600, 127)]),
    'alibi-r128-p3968': Case('alibi', 128, 128, 8, 2, 6, None, SQ80, [(128, 3968, 128)]),
    'alibi-r128-p300': Case('alibi', 128, 128, 8, 2, 4, None, SQ80, [(128, 300, 128)]),
    'r128-l257': Case('plain', 128, 128, 7, 1, 7, None, 1.0, [(65, 192, 1)]),
    'gqa4-7split': Case('plain', 128, 64, 16, 4, 7, None, 1.0, [(64, 2000, 127)]),
    'g7-tpc2': Case('plain', 64, 64, 7, 1, 8, 2, 1.0, [(64, 1000, 5)]),
    'fused-gqa4-tpc3': Case('fused', 128, 64, 16, 4, 8, 3, SQ80, [(64, 1100, 128)]),
    'empty-last-split': Case('plain', 128, 64, 16, 4, 4, None, 1.0, [(47, 1100, 5)]),
    'fused-g3-empty-last-split': Case('fused', 64, 64, 6, 2, 4, None, SQ2, [(33, 1000, 1)]),
    'batched-plain': Case('plain', 128, 64, 32, 8, 8, None, 1.0, [(64, 300, 0), (33, 1500, 128), (0, 7, 0),
                                                                   (1, 50, 130)]),
    'batched-fused': Case('fused', 128, 64, 8, 2, 8, None, 1.0, [(64, 700, 300), (0, 5, 0), (17, 129, 1),
                                                                 (40, 0, 0)]),
    'batched-alibi': Case('alibi', 128, 64, 8, 2, 8, None, 1.0, [(33, 900, 5), (0, 3, 0), (64, 200, 200),
                                                                 (5, 1300, 0)]),
    'r128-d64-l256-tpc3': Case('plain', 64, 128, 4, 4, 3, 3, SQ2, [(128, 128, 0)]),
    'l128-one-tile': Case('plain', 128, 64, 2, 2, 6, None, 1.0, [(64, 64, 0)]),
    'g7-l129': Case('plain', 64, 64, 14, 2, 0, None, SQ80, [(1, 128, 5)]),
    'fused-r128-l255-tpc2': Case('fused', 128, 128, 4, 2, 5, 2, SQ2, [(65, 190, 190)]),
    'alibi-mha40-3split': Case('alibi', 128, 64, 40, 40, 3, None, 1.0, [(64, 3904, 0)]),
    'mha25-5split': Case('plain', 128, 64, 25, 25, 0, None, SQ2, [(64, 2000, 5)]),
    'mha20-6split': Case('plain', 64, 64, 20, 20, 0, None, SQ2, [(33, 900, 1)]),
    'mha32-4split': Case('plain', 128, 64, 32, 32, 0, None, 1.0, [(64, 3968, 7)]),
    'r128-d64-8split': Case('plain', 64, 128, 8, 2, 0, None, 1.0, [(128, 3000, 300)]),
    'g2-one-split-long': Case('plain', 128, 64, 8, 4, 1, None, 1.0, [(64, 3968, 300)]),
}
# the CPU self-test: a P ~ 3968 case, GQA, odd G, 128-node drafts, ALiBi.  (Not ALiBi at P ~ 3968: there the slopes
# leave the oldest keys no weight at all, and no comparator can see them go missing.)
SELF = ['mha8-p3968', 'gqa4-pad-covers-split', 'fused-g3-empty-last-split', 'alibi-mha5-5split', 'alibi-r128-p300',
        'r128-d64-8split']


def _ceil(a, b):
    return (a + b - 1) // b


def max_seq_of(c):
    return max(P + n for n, P, _ in c.slots) + 200


def plan_grid(c, n_sm, max_seq):
    """(n_split, n_groups) that pia_attn_plan_create picks: 2 query heads per 128-row tile at 64 draft rows, 1 at 128;
    kv_split_max, or one wave of clusters over the SMs, capped by the cache's tiles and 8"""
    hpc = 2 if c.R == 64 else 1
    n_groups = c.Hkv * _ceil(c.Hq // c.Hkv, hpc)
    ns = c.k if c.k > 0 else n_sm // n_groups
    return max(1, min(ns, _ceil(max_seq, 128), 8)), n_groups


def launch_split(c, plan_ns, n, P):
    """(splits, tiles) of one slot in one launch, as the kernel derives them from the live length"""
    tiles = _ceil(P, 128) + 1 if c.mode == 'fused' else _ceil(P + n, 128)
    ns = max(1, plan_ns // len(c.slots))
    return max(1, min(_ceil(tiles, c.tpc or 1), ns)), tiles


def split_edges(c, plan_ns, n, P):
    """first and last key of each split's key range (fused mode: prefix tiles of the cache, then the draft tile)"""
    ns, tiles = launch_split(c, plan_ns, n, P)
    tps = _ceil(tiles, ns)
    edges = []
    for sp in range(ns):
        t0, t1 = sp * tps, min(sp * tps + tps, tiles)
        if t1 <= t0:
            continue
        if c.mode == 'fused':   # tiles [0, Tp) hold the cache's prefix, tile Tp the draft
            a, b = 128 * t0, min(128 * min(t1, _ceil(P, 128)), P)
            if b > a:
                edges += [a, b - 1]
            if t1 == tiles:
                edges += [P, P + n - 1]
        else:
            edges += [128 * t0, min(128 * t1, P + n) - 1]
    return edges


def merge_paths(c, plan_ns):
    """the (n_split, tiles_per_cta, merge buffers, rows per owner CTA) combinations one launch of the case takes"""
    hpc = 2 if c.R == 64 else 1
    G = c.Hq // c.Hkv
    out = set()
    for n, P, _ in c.slots:
        if n == 0:
            continue
        ns, _ = launch_split(c, plan_ns, n, P)
        for j in range(_ceil(G, hpc)):
            rows = min(hpc, G - j * hpc) * c.R
            if ns == 1:
                out.add((1, c.tpc or 1, '-', '-'))
            else:
                RS = _ceil(rows, ns)
                out.add((ns, c.tpc or 1, 'dedicated' if rows == 64 else 'aliased',
                         'pow2' if RS & (RS - 1) == 0 else 'ragged'))
    return out


def test_sweep_covers_the_listed_values():
    """the case table reaches every value the sweep is meant to cover"""
    cs = list(CASES.values())
    assert {c.mode for c in cs} == {'plain', 'fused', 'alibi'} and all(c.D == 128 for c in cs if c.mode == 'alibi')
    assert {(c.mode, c.D) for c in cs} >= {('plain', 64), ('plain', 128), ('fused', 64), ('fused', 128)}
    assert {n for c in cs if c.R == 64 for n, _, _ in c.slots} >= {1, 33, 64}
    assert {n for c in cs if c.R == 128 for n, _, _ in c.slots} >= {65, 128}
    assert {c.Hq // c.Hkv for c in cs if c.R == 64} >= {1, 2, 3, 4, 7}
    assert {c.k for c in cs} == set(range(9)) and {c.tpc for c in cs} == {None, 2, 3}
    assert {P + n for c in cs for n, P, _ in c.slots if n} >= {127, 128, 129, 255, 256, 257}
    assert {P for c in cs for n, P, _ in c.slots if n} >= {0, 3968}
    assert {pad for c in cs for _, _, pad in c.slots} >= {0, 1, 5, 127, 128, 300}
    assert any(n and pad >= P > 0 for c in cs for n, P, pad in c.slots)
    assert {c.scale for c in cs} == {1.0, SQ2, SQ80}
    assert any(len(c.slots) == 4 and c.k == 8 and sum(n == 0 for n, _, _ in c.slots) == 1 for c in cs)
    # a slot whose last split has no tile, and a pad that hides a whole split's key range
    empty, hidden = False, False
    for c in cs:
        pns = plan_grid(c, N_SM, max_seq_of(c))[0]
        for n, P, pad in c.slots:
            ns, tiles = launch_split(c, pns, n, P)
            tps = _ceil(tiles, ns)
            empty |= n > 0 and ns > 1 and (ns - 1) * tps >= tiles
            hidden |= n > 0 and ns > 1 and c.mode == 'plain' and pad >= 128 * tps
    assert empty and hidden
    paths = set().union(*(merge_paths(c, plan_grid(c, N_SM, max_seq_of(c))[0]) for c in cs))
    assert {p[0] for p in paths} == set(range(1, 9))
    assert {p[2:] for p in paths if p[0] > 1} == {('dedicated', 'pow2'), ('dedicated', 'ragged'), ('aliased', 'pow2'),
                                                  ('aliased', 'ragged')}


# ---------------------------------------------------------------------------------------------------------------
# detection power of the comparator, on the CPU
# ---------------------------------------------------------------------------------------------------------------
def _self_inputs(c, beacon):
    n, P, pad = c.slots[0]
    rng = np.random.default_rng(P + n + c.Hq)
    gen = torch.Generator().manual_seed(P * 7 + n)
    parent, rows = A.tree(rng, n, max_depth=12)
    if beacon:
        edges = split_edges(c, plan_grid(c, N_SM, max_seq_of(c))[0], n, P)
        q, k, v = A.beacon_data(parent, n, P, pad, c.Hq, c.Hkv, c.D, P + n, c.scale, edges, gen)
    else:
        q = (0.7 * torch.randn((n, c.Hq, c.D), generator=gen)).to(torch.bfloat16)
        k = (0.7 * torch.randn((c.Hkv, P + n, c.D), generator=gen)).to(torch.bfloat16)
        v = (0.7 * torch.randn((c.Hkv, P + n, c.D), generator=gen)).to(torch.bfloat16)
    from painlessinferenceacceleration_b200.common import ops
    slopes = ops.alibi_slopes(c.Hq) if c.mode == 'alibi' else None
    return parent, rows, q, k, v, slopes


@pytest.mark.parametrize('data', ['random', 'beacon'])
@pytest.mark.parametrize('name', SELF)
def test_comparator_accepts_the_kernel_arithmetic_and_rejects_wrong_rules(name, data):
    """the emulated kernel (one split, and three splits merged in fp32) passes; every wrong rule that changes
    something on the case fails in at least one element"""
    c = CASES[name]
    n, P, pad = c.slots[0]
    parent, rows, q, k, v, slopes = _self_inputs(c, data == 'beacon')
    assert pad > 0 and A.sibling_pair(parent) is not None and (c.R == 64 or n > 64)
    kw = dict(scale_mul=c.scale, slopes=slopes)
    ref = A.reference(q, k, v, rows, n, P, pad, **kw)
    for ns in (1, 3):
        A.assert_close(A.emulate(q, k, v, rows, n, P, pad, n_split=ns, **kw), ref, f'emulation, {ns} split(s)')
    muts = A.mutations(parent, rows, n, P, pad, c.Hq, c.Hkv, c.scale, alibi=c.mode == 'alibi')
    if c.Hq != c.Hkv and c.Hkv > 1:
        assert 'GQA map h % Hkv' in muts
    if c.mode == 'alibi':
        assert 'ALiBi qpos without the pad' in muts and 'ALiBi draft key at its DFS index' in muts
        assert (n > 64) == ('ALiBi depth over mask word 0 only' in muts)
    assert set(A.SINGLE_KEY) <= set(muts)
    weak = {}
    for mname, mkw in muts.items():
        got = A.reference(q, k, v, rows, n, P, pad, **{**kw, **mkw}).to(torch.bfloat16)
        w = A.worst(got, ref)
        if w <= 1.0:
            weak[mname] = w
    assert not weak, f'wrong rules the comparator accepts: {weak}'


def test_old_tolerance_accepts_a_wrong_rule_the_comparator_rejects():
    """why the fixed allclose(atol=1.5e-2, rtol=2e-2) is gone: at P = 3968 it accepts a hidden key P - 1"""
    c = CASES['mha32-4split']
    n, P, pad = c.slots[0]
    parent, rows, q, k, v, _ = _self_inputs(c._replace(Hq=8, Hkv=8), False)
    ref = A.reference(q, k, v, rows, n, P, pad)
    wrong = A.reference(q, k, v, rows, n, P, pad, **A.mutations(parent, rows, n, P, pad, 8, 8)['key P-1 hidden'])
    wrong = wrong.to(torch.bfloat16)
    assert torch.allclose(wrong.double(), ref, atol=1.5e-2, rtol=2e-2)
    assert A.worst(wrong, ref) > 1.0


# ---------------------------------------------------------------------------------------------------------------
# the kernel on the H100
# ---------------------------------------------------------------------------------------------------------------
def _rope_tables(max_pos, D):
    """bf16 RoPE tables whose first frequency is the identity (cos 1, sin 0): head dims 0 and D / 2 pass through, so
    the beacon direction (dim 0) survives the rotation of the fused kernel"""
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, device=DEV).float() / D))
    ang = torch.arange(max_pos, device=DEV).float()[:, None] * inv[None]
    ang[:, 0] = 0.0
    return ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()


class _Run(object):
    """one case on the GPU: slot s of the launch uses cache slot 1 + s (cache slot 0 belongs to nobody), layer 1
    (layer 0 belongs to nobody), rows [s * R, s * R + n) of q / qkv / mask / out"""

    def __init__(self, c):
        from painlessinferenceacceleration_b200.common import ops
        self.c, self.ops = c, ops
        B, D = len(c.slots), c.D
        self.B, self.rps = B, c.R
        self.max_seq = max_seq_of(c)
        self.k = torch.zeros((B + 1, 2, c.Hkv, self.max_seq, D), dtype=torch.bfloat16, device=DEV)
        self.v = torch.zeros_like(self.k)
        self.plan = ops.AttnPlan(self.k, self.v, c.Hq, c.Hkv, D, c.R, kv_split_max=c.k)
        ns, ng = C.c_int(0), C.c_int(0)
        assert self.plan.lib.pia_attn_plan_grid(self.plan.h, C.byref(ns), C.byref(ng)) == 0
        self.grid = (ns.value, ng.value)
        n_sm = torch.cuda.get_device_properties(0).multi_processor_count
        assert self.grid == plan_grid(c, n_sm, self.max_seq), (self.grid, plan_grid(c, n_sm, self.max_seq))
        rng = np.random.default_rng(sum(P + 3 * n + pad for n, P, pad in c.slots) + c.Hq)
        self.trees = [A.tree(rng, n, max_depth=12) for n, _, _ in c.slots]
        self.rows = [t[1] for t in self.trees]
        self.mask = A.mask_words(self.rows, c.R, self.rps, DEV)
        t = lambda i: torch.tensor([s[i] for s in c.slots], dtype=torch.int32, device=DEV)  # noqa: E731
        self.slots = ops.Slots(t(0), t(1), t(2), self.rps, self.plan.slot_stride if B > 1 else 0, kv_first_slot=1)
        rows_all = B * self.rps
        self.q = torch.zeros((rows_all, c.Hq, D), dtype=torch.bfloat16, device=DEV)
        self.qkv = torch.zeros((rows_all, (c.Hq + 2 * c.Hkv) * D), dtype=torch.bfloat16, device=DEV)
        self.cos, self.sin = _rope_tables(self.max_seq + 8, D)
        self.slopes = ops.alibi_slopes(c.Hq).to(DEV) if c.mode == 'alibi' else None
        self.out = torch.empty((rows_all, c.Hq, D), dtype=torch.bfloat16, device=DEV)

    def launch(self):
        c = self.c
        self.out.fill_(9.0)
        if c.mode == 'fused':
            self.plan.forward_fused(1, self.qkv, self.mask, self.slots, self.cos, self.sin, self.out, scale_mul=c.scale)
        else:
            self.plan.forward(1, self.q, self.mask, self.slots, self.out, scale_mul=c.scale, alibi_slopes=self.slopes)
        torch.cuda.synchronize()
        return self.out.clone()

    def qkv_cols(self, part, hkv=None):
        """column slice of qkv: part 0 = Q heads, 1 = K head hkv, 2 = V head hkv"""
        c, D = self.c, self.c.D
        if part == 0:
            return slice(0, c.Hq * D)
        h0 = c.Hq + (part - 1) * c.Hkv + hkv
        return slice(h0 * D, (h0 + 1) * D)

    def set_draft_kv(self, s_, j, k, v):
        """node j of slot s_: K / V [Hkv, D] into the cache row (plain / ALiBi) or the projection output (fused)"""
        P = self.c.slots[s_][1]
        if self.c.mode == 'fused':
            for h in range(self.c.Hkv):
                self.qkv[s_ * self.rps + j, self.qkv_cols(1, h)] = k[h]
                self.qkv[s_ * self.rps + j, self.qkv_cols(2, h)] = v[h]
        else:
            self.k[1 + s_, 1, :, P + j] = k
            self.v[1 + s_, 1, :, P + j] = v

    def fill(self, beacon, gen):
        """random 0.7 randn inputs everywhere, then (beacon) each live slot's layer-1 keys / queries as beacon data"""
        c, D = self.c, self.c.D
        for t in (self.k, self.v):
            t.copy_((0.7 * torch.randn(t.shape, generator=gen)).to(torch.bfloat16))
        self.q.copy_((0.7 * torch.randn(self.q.shape, generator=gen)).to(torch.bfloat16))
        self.qkv.copy_((0.7 * torch.randn(self.qkv.shape, generator=gen)).to(torch.bfloat16))
        if not beacon:
            return
        for s_, (n, P, pad) in enumerate(c.slots):
            if n == 0:
                continue
            edges = split_edges(c, self.grid[0], n, P)
            q, k, v = A.beacon_data(self.trees[s_][0], n, P, pad, c.Hq, c.Hkv, D, P + n + 2, c.scale, edges, gen)
            r0 = s_ * self.rps
            self.q[r0:r0 + n] = q.to(DEV)
            self.qkv[r0:r0 + n, self.qkv_cols(0)] = q.reshape(n, -1).to(DEV)
            self.k[1 + s_, 1, :, :P + n + 2] = k.to(DEV)
            self.v[1 + s_, 1, :, :P + n + 2] = v.to(DEV)
            for j in range(n):
                self.set_draft_kv(s_, j, k[:, P + j].to(DEV), v[:, P + j].to(DEV))

    def check_reference(self, out):
        """each live slot against the fp64 reference; returns the worst score.  Fused mode: Q and the appended draft
        keys come from pia_rope_kv_append on a copy of the caches (the same arithmetic, checked bit for bit)"""
        c = self.c
        q, k, v = self.q, self.k, self.v
        if c.mode == 'fused':
            q = torch.zeros_like(self.q)
            k, v = self.k.clone(), self.v.clone()
            self.ops.rope_kv_append(self.qkv, self.mask, self.slots, c.Hq, c.Hkv, c.D, self.cos, self.sin, q,
                                    k[1, 1], v[1, 1], self.max_seq)
        w = 0.0
        for s_, (n, P, pad) in enumerate(c.slots):
            r0 = s_ * self.rps
            assert float((out[r0 + n:r0 + self.rps].float() - 9.0).abs().sum()) == 0   # rows beyond the draft
            if n == 0:
                continue
            if c.mode == 'fused':   # the fused launch appended the same rows
                assert torch.equal(self.k[1 + s_, 1, :, P:P + n], k[1 + s_, 1, :, P:P + n])
                assert torch.equal(self.v[1 + s_, 1, :, P:P + n], v[1 + s_, 1, :, P:P + n])
            ref = A.reference(q[r0:], k[1 + s_, 1], v[1 + s_, 1], self.rows[s_], n, P, pad, scale_mul=c.scale,
                              slopes=self.slopes)
            w = max(w, A.assert_close(out[r0:r0 + n], ref, f'slot {s_}'))
        return w

    def hide_everything_unseen(self):
        """finite sentinels wherever no live row may look: cache rows [0, pad) and [L, max_seq) (fused: [P, max_seq),
        the draft rows are appended again by the launch), layer 0, cache slot 0, idle slots, and the q / qkv / mask
        rows of every slot beyond its draft"""
        c, D = self.c, self.c.D
        ks, vs = A.sentinel_kv(D, c.scale, device=DEV)
        for t, s in ((self.k, ks), (self.v, vs)):
            t[0] = s
            t[:, 0] = s
        for s_, (n, P, pad) in enumerate(c.slots):
            lo = P if c.mode == 'fused' else P + n
            for t, s in ((self.k, ks), (self.v, vs)):
                t[1 + s_, 1, :, :min(pad, P)] = s
                t[1 + s_, 1, :, lo:] = s
                if n == 0:
                    t[1 + s_] = s
            r0 = s_ * self.rps
            self.q[r0 + n:r0 + self.rps] = vs[None, None]
            self.qkv[r0 + n:r0 + self.rps] = A.SENTINEL_V
            self.mask[r0 + n:r0 + self.rps] = -1


def _case_params():
    return [pytest.param(k, marks=pytest.mark.gpu) for k in CASES]


@pytest.mark.parametrize('name', _case_params())
def test_kernel_against_reference_and_exact_invariance(name, monkeypatch):
    """random inputs and beacon inputs against the fp64 reference (comparator); then, bit for bit: sentinels in every
    place no row may look leave the output unchanged, a relaunch repeats it, and perturbing draft node j changes
    exactly the rows whose mask has bit j"""
    c = CASES[name]
    if c.tpc is None:
        monkeypatch.delenv('PIA_ATTN_TILES_PER_CTA', raising=False)
    else:
        monkeypatch.setenv('PIA_ATTN_TILES_PER_CTA', str(c.tpc))
    r = _Run(c)
    gen = torch.Generator().manual_seed(sum(P * 3 + n for n, P, _ in c.slots) + c.Hq)
    r.fill(False, gen)
    w_random = r.check_reference(r.launch())
    r.fill(True, gen)
    base = r.launch()
    w_beacon = r.check_reference(base)
    print(f'\nATTN-POWER {name}: grid {r.grid} paths {sorted(merge_paths(c, r.grid[0]))} '
          f'worst score random {w_random:.3f} beacon {w_beacon:.3f}')

    r.hide_everything_unseen()
    assert torch.equal(r.launch(), base), 'a hidden key, another layer / slot or a row beyond the draft leaked'
    assert torch.equal(r.launch(), base), 'relaunch differs'

    ks, vs = A.sentinel_kv(c.D, c.scale, (c.Hkv,), device=DEV)
    vs = -vs   # unlike the sentinel the beacon inputs may already hold at node j
    for pick in range(2):
        saved, nodes = [], []
        for s_, (n, P, pad) in enumerate(c.slots):
            if n == 0:
                nodes.append(None)
                continue
            sib = A.sibling_pair(r.trees[s_][0])
            j = (sib[1] if sib else n - 1) if pick == 0 else n // 2
            nodes.append(j)
            if c.mode == 'fused':
                saved.append(r.qkv[s_ * r.rps + j].clone())
            else:
                saved.append((r.k[1 + s_, 1, :, P + j].clone(), r.v[1 + s_, 1, :, P + j].clone()))
            r.set_draft_kv(s_, j, ks, vs)
        got = r.launch()
        for s_, (n, P, pad) in enumerate(c.slots):
            r0 = s_ * r.rps
            assert torch.equal(got[r0 + n:r0 + r.rps], base[r0 + n:r0 + r.rps])
            for i in range(n):
                sees = (r.rows[s_][i] >> nodes[s_]) & 1
                same = torch.equal(got[r0 + i], base[r0 + i])
                assert same != bool(sees), f'slot {s_} row {i} node {nodes[s_]}: sees it {bool(sees)}, changed {not same}'
        it = iter(saved)
        for s_, (n, P, pad) in enumerate(c.slots):
            if n == 0:
                continue
            sv = next(it)
            if c.mode == 'fused':
                r.qkv[s_ * r.rps + nodes[s_]] = sv
            else:
                r.k[1 + s_, 1, :, P + nodes[s_]], r.v[1 + s_, 1, :, P + nodes[s_]] = sv
