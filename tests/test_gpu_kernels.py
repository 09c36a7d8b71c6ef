# -*- coding: utf-8 -*-
"""Numerics of the verify-forward kernels against plain PyTorch fp32 restatements of the reference ops
(models/llama/modeling_llama.py:156-169, 185-186, 243-308; pretrained_model.py:764-892, 894-907).  RMSNorm, SiLU*up
and the embedding gather are tested in depth in tests/test_gpu_norm_power.py."""

import numpy as np
import pytest
import torch

from tests import attn_ref
from tests import gemm_ref

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _random_tree(rng, n, max_depth=8):
    """parent array of a DFS-pre-order tree (like the trie emits) and its ancestor bit rows"""
    parent = [-1]
    depth = [0]
    for i in range(1, n):
        # attach to a node on the current rightmost path so that the order stays a valid pre-order
        path = [i - 1]
        while parent[path[-1]] >= 0:
            path.append(parent[path[-1]])
        cands = [p for p in path if depth[p] < max_depth]
        p = cands[int(rng.integers(0, len(cands)))] if cands else 0
        parent.append(p)
        depth.append(depth[p] + 1)
    rows = np.zeros((n,), dtype=np.uint64)
    for i in range(n):
        j = i
        while j >= 0:
            rows[i] |= np.uint64(1) << np.uint64(j)
            j = parent[j]
    return parent, depth, rows


def _mask_tensor(rows, R):
    m = np.zeros((R, max(R // 64, 1)), dtype=np.uint64)
    m[:len(rows), 0] = rows
    return torch.from_numpy(m.view(np.int64)).to(DEV)


def _slots(ns, Ps, pads, rows_per_slot, stride=0, first=0):
    from painlessinferenceacceleration_b200.common import ops
    t = [torch.tensor(v, dtype=torch.int32, device=DEV) for v in (ns, Ps, pads)]
    return ops.Slots(t[0], t[1], t[2], rows_per_slot, stride, kv_first_slot=first)


def _ref_attention(q, kc, vc, rows, n, P, pad_len, G):
    """eager attention of the reference with the [n, P+n] lookahead mask, exact (fp64; tests/attn_ref.py)"""
    return attn_ref.reference(q, kc, vc, rows, n, P, pad_len, G)


@pytest.mark.parametrize('Hq,Hkv,P,n,pad', [(2, 2, 0, 64, 0), (4, 2, 37, 33, 0), (32, 32, 300, 64, 0),
                                             (32, 8, 1000, 47, 5), (8, 2, 127, 1, 0), (8, 8, 129, 64, 3),
                                             (32, 8, 2500, 64, 0), (32, 32, 140, 64, 0), (32, 32, 600, 64, 0),
                                             (32, 32, 520, 50, 0), (32, 32, 3900, 64, 7)])
def test_tree_attention(Hq, Hkv, P, n, pad):
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(P + n)
    torch.manual_seed(P * 7 + n)
    D, R, n_layers = 128, 64, 2
    max_seq = P + n + 70
    kc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    q = (torch.randn((R, Hq, D), device=DEV) * 0.7).to(torch.bfloat16)
    _, _, rows = _random_tree(rng, n)
    mask = _mask_tensor(rows, R)
    plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
    out = torch.zeros((R, Hq, D), dtype=torch.bfloat16, device=DEV)
    slots = _slots([n], [P], [pad], R)
    for layer in (1, 0):
        out.zero_()
        plan.forward(layer, q, mask, slots, out)
        torch.cuda.synchronize()
        ref = _ref_attention(q, kc[layer], vc[layer], rows, n, P, pad, Hq // Hkv)
        got = out[:n].float()
        err = (got - ref).abs().max().item()
        # tolerance: bf16 output rounding (2^-8 relative on |o| <~ 1) + fp32 accumulation order
        attn_ref.assert_close(got, ref, f'layer {layer} max abs err {err}')


def test_rope_kv_append_and_silu():
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(1)
    rng = np.random.default_rng(3)
    Hq, Hkv, D, R, n, P, pad = 4, 2, 128, 64, 40, 77, 2
    max_seq = 256
    qkv = torch.randn((R, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    _, depth, rows = _random_tree(rng, n)
    mask = _mask_tensor(rows, R)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, device=DEV).float() / D))
    ang = torch.arange(max_seq, device=DEV).float()[:, None] * inv[None]
    cos, sin = ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()
    qo = torch.zeros((R, Hq, D), dtype=torch.bfloat16, device=DEV)
    kc = torch.zeros((Hkv, max_seq, D), dtype=torch.bfloat16, device=DEV)
    vc = torch.zeros_like(kc)
    ops.rope_kv_append(qkv, mask, _slots([n], [P], [pad], R), Hq, Hkv, D, cos, sin, qo, kc, vc, max_seq)
    torch.cuda.synchronize()
    pos = torch.tensor([P - pad + d for d in depth], device=DEV)
    c = torch.cat([cos[pos], cos[pos]], -1)[:, None]  # [n,1,D] bf16  (modeling_llama.py:124-127)
    s = torch.cat([sin[pos], sin[pos]], -1)[:, None]

    def rot(x):
        return torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1)

    x = qkv[:n].view(n, Hq + 2 * Hkv, D)
    qk = x[:, :Hq + Hkv]
    ref = (qk * c) + (rot(qk) * s)  # bf16 eager arithmetic (:167-168)
    assert torch.equal(qo[:n], ref[:, :Hq])
    assert torch.equal(kc[:, P:P + n].transpose(0, 1), ref[:, Hq:])
    assert torch.equal(vc[:, P:P + n].transpose(0, 1), x[:, Hq + Hkv:])
    assert float(kc[:, :P].abs().sum()) == 0 and float(kc[:, P + n:].abs().sum()) == 0
    # left padding that reaches beyond the cached prefix (first prefill chunk of a padded prompt): no visible prefix
    # key, position = depth (rowsum(mask) - 1, modeling_llama.py:587)
    qo2 = torch.zeros_like(qo)
    kc2, vc2 = torch.zeros_like(kc), torch.zeros_like(vc)
    ops.rope_kv_append(qkv, mask, _slots([n], [3], [9], R), Hq, Hkv, D, cos, sin, qo2, kc2, vc2, max_seq)
    pos2 = torch.tensor(list(depth), device=DEV)
    c2 = torch.cat([cos[pos2], cos[pos2]], -1)[:, None]
    s2 = torch.cat([sin[pos2], sin[pos2]], -1)[:, None]
    ref2 = (qk * c2) + (rot(qk) * s2)
    assert torch.equal(qo2[:n], ref2[:, :Hq])
    assert torch.equal(kc2[:, 3:3 + n].transpose(0, 1), ref2[:, Hq:])
    # SiLU(gate) * up equals eager bf16 torch bit for bit (every gate value and the width tails:
    # tests/test_gpu_norm_power.py)
    gu = torch.randn((64, 2 * 1024), device=DEV).to(torch.bfloat16)
    out = torch.empty((64, 1024), dtype=torch.bfloat16, device=DEV)
    ops.silu_mul(gu, out)
    ref = torch.nn.functional.silu(gu[:, :1024]) * gu[:, 1024:]
    assert torch.equal(out, ref)


def _host_accept(ids, parent, row_tok):
    cur, toks, nodes = 0, [], []
    while True:
        t = row_tok[cur]
        toks.append(t)
        nodes.append(cur)
        nxt = [j for j in range(1, len(ids)) if parent[j] == cur and ids[j] == t]
        if not nxt:
            break
        cur = nxt[0]
    return toks, nodes


@pytest.mark.parametrize('penalty', [1.0, 1.1])
def test_accept_walk_and_kv_compact(penalty):
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(17)
    V, R = 1000, 64
    for trial in range(12):
        n = int(rng.integers(1, 65))
        parent, depth, rows = _random_tree(rng, n)
        ids = [int(rng.integers(3, 40))]
        for j in range(1, n):  # siblings carry distinct tokens (dict keys)
            used = {ids[k] for k in range(1, j) if parent[k] == parent[j]}
            t = int(rng.integers(3, 40))
            while t in used:
                t = int(rng.integers(3, 40))
            ids.append(t)
        logits = torch.randn((R, V), device=DEV).to(torch.bfloat16)
        # make the walk non-trivial: let most rows vote for one of their children
        for j in range(n):
            kids = [k for k in range(1, n) if parent[k] == j]
            if kids and rng.random() < 0.8:
                logits[j, ids[kids[int(rng.integers(0, len(kids)))]]] = 30.0
        seq_len0 = 20
        seq_host = rng.integers(3, 40, size=seq_len0).tolist()
        seq = torch.zeros((256,), dtype=torch.int32, device=DEV)
        seq[:seq_len0] = torch.tensor(seq_host, dtype=torch.int32)
        seq[seq_len0 - 1] = ids[0]
        seq_host[-1] = ids[0]
        # host restatement of :827-860 with RepetitionPenaltyLogitsProcessor semantics
        lf = logits.clone()
        row_tok = []
        for j in range(n):
            sc = lf[j].clone()
            if penalty != 1.0:
                ctx = set(seq_host)
                k = j
                while k >= 1:
                    ctx.add(ids[k])
                    k = parent[k]
                idx = torch.tensor(sorted(ctx), device=DEV)
                v = sc[idx]
                sc[idx] = torch.where(v < 0, v * penalty, v / penalty)
            row_tok.append(int(torch.argmax(sc)))
        toks, nodes = _host_accept(ids, parent, row_tok)
        acc = ops.Accept(V, R, penalty, [2], 10 ** 6, DEV)
        d = dict(ids=torch.zeros((R,), dtype=torch.int32, device=DEV), n=torch.tensor([n], dtype=torch.int32, device=DEV))
        d['ids'][:n] = torch.tensor(ids, dtype=torch.int32)
        mask = _mask_tensor(rows, R)
        seq_len = torch.tensor([seq_len0], dtype=torch.int32, device=DEV)
        P0 = seq_len0 - 1
        prefix = torch.tensor([P0], dtype=torch.int32, device=DEV)
        fin = torch.zeros((1,), dtype=torch.int32, device=DEV)
        at = torch.zeros((R,), dtype=torch.int32, device=DEV)
        ac = torch.zeros((1,), dtype=torch.int32, device=DEV)
        an = torch.zeros((R,), dtype=torch.int32, device=DEV)
        kc = torch.arange(2 * 2 * 128 * 16, device=DEV).float().view(2, 2, 128, 16).to(torch.bfloat16).contiguous()
        vc = (kc.float() + 0.5).to(torch.bfloat16).contiguous()
        k0, v0 = kc.clone(), vc.clone()
        acc.run(logits, d['ids'], mask, d['n'], seq, seq_len, at, ac, an, prefix, fin)
        ops.kv_compact(kc, vc, an, ac, prefix)
        torch.cuda.synchronize()
        c = int(ac)
        assert at[:c].tolist() == toks, (trial, at[:c].tolist(), toks)
        assert an[:c].tolist() == nodes
        assert int(seq_len) == seq_len0 + c and int(prefix) == P0 + c
        assert seq[seq_len0:seq_len0 + c].tolist() == toks
        assert int(fin) == (1 if 2 in toks else 0)
        # rows [0, P0] untouched, accepted draft rows moved next to the prefix (:894-907)
        keep = list(range(P0 + 1)) + [P0 + j for j in nodes[1:]]
        assert torch.equal(kc[:, :, :len(keep)], k0[:, :, keep]) and torch.equal(vc[:, :, :len(keep)], v0[:, :, keep])


@pytest.mark.parametrize('Hq,Hkv,rps,cases', [
    (4, 2, 16, [(16, 100, 0), (5, 0, 0), (0, 7, 0), (9, 257, 3)]),        # one idle slot, one empty context, padding
    (32, 8, 8, [(8, 300, 0), (3, 290, 0), (8, 310, 2), (1, 5, 0), (7, 128, 0), (8, 64, 0), (2, 500, 0), (6, 301, 0)]),
    (32, 32, 32, [(32, 420, 0), (11, 64, 0)])])
def test_batched_slots_rope_and_attention(Hq, Hkv, rps, cases):
    """the request-slot form of RoPE/KV-append and tree attention (pia_slots_t; batched loop,
    modeling_llama_batch.py:375-405): every slot has its own draft, cursor, padding and KV cache; one launch each must
    equal the per-slot single launches bit for bit, and rows beyond a slot's draft are never written"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(rps)
    torch.manual_seed(rps)
    D, R, n_layers, B = 128, 64, 2, len(cases)
    max_seq = max(P + n for n, P, _ in cases) + 70
    kc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    qkv = torch.randn((R, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, device=DEV).float() / D))
    ang = torch.arange(max_seq + 8, device=DEV).float()[:, None] * inv[None]
    cos, sin = ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()
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
    # batched: one launch each over all slots
    kb, vb = kc.clone(), vc.clone()
    planb = ops.AttnPlan(kb, vb, Hq, Hkv, D, R)
    qb = torch.full((R, Hq, D), 7.0, dtype=torch.bfloat16, device=DEV)
    ob = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
    sl = _slots(ns, Ps, pads, rps, stride=plan.slot_stride)
    ops.rope_kv_append(qkv, mask, sl, Hq, Hkv, D, cos, sin, qb, kb[0, layer], vb[0, layer], max_seq)
    planb.forward(layer, qb, mask, sl, ob)
    torch.cuda.synchronize()
    # slot by slot: single-slot launches on that slot's own cache / rows, then the fp32 reference
    for s_, (n, P, pad) in enumerate(cases):
        r0 = s_ * rps
        one = _slots([n], [P], [pad], rps, first=s_)
        q1 = torch.full((R, Hq, D), 7.0, dtype=torch.bfloat16, device=DEV)
        o1 = torch.full((R, Hq, D), 9.0, dtype=torch.bfloat16, device=DEV)
        ops.rope_kv_append(qkv[r0:], mask[r0:], one, Hq, Hkv, D, cos, sin, q1, kc[s_, layer], vc[s_, layer], max_seq)
        plan.forward(layer, q1, mask[r0:], one, o1)
        torch.cuda.synchronize()
        # RoPE / KV append: bit for bit.  Attention: a batch launch uses fewer KV splits per request (one wave of CTAs
        # over all slots), i.e. another fp32 summation order - equal to the last bf16 bit or so
        assert torch.equal(qb[r0:r0 + rps], q1[:rps])
        assert torch.allclose(ob[r0:r0 + n].float(), o1[:n].float(), atol=4e-3, rtol=2e-2)
        assert torch.equal(kb[s_], kc[s_]) and torch.equal(vb[s_], vc[s_])
        assert float((qb[r0 + n:r0 + rps].float() - 7.0).abs().sum()) == 0   # rows beyond the draft: untouched
        assert float((ob[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0
        if n:
            ref = _ref_attention(q1, kc[s_, layer], vc[s_, layer], trees[s_], n, P, pad, Hq // Hkv)
            attn_ref.assert_close(ob[r0:r0 + n].float(), ref)


@pytest.mark.parametrize('Hq,Hkv,rps,cases', [
    (32, 32, 64, [(64, 384, 0)]),                                  # the benchmark's mid-generation step, MHA
    (32, 8, 64, [(47, 1000, 5)]),                                  # GQA-4, ragged draft, left padding
    (8, 8, 64, [(1, 130, 0)]),                                     # a root-only draft right after a tile boundary
    (4, 2, 64, [(33, 0, 0)]),                                      # empty cache: the draft tile is the only tile
    (32, 8, 8, [(8, 300, 0), (3, 290, 0), (8, 310, 2), (1, 5, 0), (7, 128, 0), (8, 64, 0), (2, 500, 0), (6, 301, 0)]),
    (32, 32, 64, [(64, 2500, 0)])])                                # several prefix tiles per CTA behind the draft tile
def test_fused_rope_kv_append_attention(Hq, Hkv, rps, cases):
    """pia_tree_attn_fused_fwd (RoPE + KV append + tree attention in one launch; draft keys staged in shared memory,
    TMA only over the cached prefix) against the two-kernel path pia_rope_kv_append + pia_tree_attn_fwd on the same
    inputs: the cache rows it appends are bit identical (and nothing else in the cache moves), the attention output
    agrees to the fp32 summation order of the tiles, and with the fp32 reference"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(Hq + rps)
    torch.manual_seed(Hq * 3 + rps)
    D, R, n_layers, B = 128, 64, 2, len(cases)
    max_seq = max(P + n for n, P, _ in cases) + 70
    kc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    vc = (torch.randn((B, n_layers, Hkv, max_seq, D), device=DEV) * 0.7).to(torch.bfloat16)
    qkv = torch.randn((R, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, device=DEV).float() / D))
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
        assert torch.allclose(o2[r0:r0 + n].float(), o1[r0:r0 + n].float(), atol=4e-3, rtol=2e-2), s_
        assert float((o2[r0 + n:r0 + rps].float() - 9.0).abs().sum()) == 0      # rows beyond the draft: untouched
        ref = _ref_attention(q[r0:], kc[s_, layer], vc[s_, layer], trees[s_], n, P, pad, Hq // Hkv)
        attn_ref.assert_close(o2[r0:r0 + n].float(), ref, s_)


def test_prefill_chunks_share_one_cache():
    """a prefill pass = one table slot per 64-row chain chunk over the SAME cache (kv_slot_stride 0): chunk c must see
    the rows chunk c-1 appended in the same launch sequence; equals feeding the chunks one after the other"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(5)
    Hq, Hkv, D, R, C, n_layers = 8, 2, 128, 64, 3, 1
    lens = [64, 64, 23]
    max_seq = 400
    chain = np.array([(1 << (i + 1)) - 1 if i < 63 else 0xFFFFFFFFFFFFFFFF for i in range(R)], dtype=np.uint64)
    mask = torch.from_numpy(np.tile(chain, C).view(np.int64)).to(DEV).view(C * R, 1)
    qkv = torch.randn((C * R, (Hq + 2 * Hkv) * D), device=DEV).to(torch.bfloat16)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, device=DEV).float() / D))
    ang = torch.arange(max_seq, device=DEV).float()[:, None] * inv[None]
    cos, sin = ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()
    base = 40  # tokens already cached
    outs = []
    for batched in (True, False):
        kc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV, generator=torch.Generator(DEV).manual_seed(1)) * 0.7).to(torch.bfloat16)
        vc = (torch.randn((n_layers, Hkv, max_seq, D), device=DEV, generator=torch.Generator(DEV).manual_seed(2)) * 0.7).to(torch.bfloat16)
        plan = ops.AttnPlan(kc, vc, Hq, Hkv, D, R)
        q = torch.zeros((C * R, Hq, D), dtype=torch.bfloat16, device=DEV)
        o = torch.zeros((C * R, Hq, D), dtype=torch.bfloat16, device=DEV)
        if batched:
            sl = _slots(lens, [base + R * c for c in range(C)], [0] * C, R)
            ops.rope_kv_append(qkv, mask, sl, Hq, Hkv, D, cos, sin, q, kc[0], vc[0], max_seq)
            plan.forward(0, q, mask, sl, o)
        else:
            for c in range(C):
                sl = _slots([lens[c]], [base + R * c], [0], R)
                ops.rope_kv_append(qkv[R * c:], mask[R * c:], sl, Hq, Hkv, D, cos, sin, q[R * c:], kc[0], vc[0], max_seq)
            for c in range(C):
                sl = _slots([lens[c]], [base + R * c], [0], R)
                plan.forward(0, q[R * c:], mask[R * c:], sl, o[R * c:])
        torch.cuda.synchronize()
        outs.append((q.clone(), o.clone(), kc.clone(), vc.clone()))
    (q_a, o_a, k_a, v_a), (q_b, o_b, k_b, v_b) = outs
    assert torch.equal(q_a, q_b) and torch.equal(k_a, k_b) and torch.equal(v_a, v_b)
    assert torch.allclose(o_a.float(), o_b.float(), atol=4e-3, rtol=2e-2)   # KV split count differs (see above)


def test_batched_accept_walk_and_compaction():
    """pia_accept / pia_kv_compact over several request slots (pretrained_model_batch.py:810-918): each slot equals the
    single-slot run on its own rows; bound_walk caps the accepted tokens at max_length - len (:862); a slot that already
    finished and an idle slot accept nothing"""
    from painlessinferenceacceleration_b200.common import ops
    rng = np.random.default_rng(23)
    V, R, B, rps = 500, 64, 4, 16
    stride = 128
    ids = torch.zeros((R,), dtype=torch.int32, device=DEV)
    mask = torch.zeros((R, 1), dtype=torch.int64, device=DEV)
    logits = torch.randn((R, V), device=DEV).to(torch.bfloat16)
    seq = torch.zeros((B, stride), dtype=torch.int32, device=DEV)
    ns, lens, info = [], [], []
    for s_ in range(B):
        n = [16, 9, 0, 12][s_]
        ns.append(n)
        parent = [-1] + list(range(n - 1))          # one chain: every node's child continues it
        toks = [int(rng.integers(3, 40))] + rng.choice(np.arange(40, 400), size=max(n - 1, 0), replace=False).tolist()
        L0 = 20 + s_
        lens.append(L0)
        seq[s_, :L0] = torch.tensor(rng.integers(3, 40, size=L0).tolist(), dtype=torch.int32)
        if n:
            seq[s_, L0 - 1] = toks[0]
            ids[s_ * rps:s_ * rps + n] = torch.tensor(toks, dtype=torch.int32)
            rows = np.array([(1 << (i + 1)) - 1 for i in range(n)], dtype=np.uint64)
            mask[s_ * rps:s_ * rps + n, 0] = torch.from_numpy(rows.view(np.int64)).to(DEV)
            for j in range(n - 1):                   # row j votes for its child: the whole chain would be accepted
                logits[s_ * rps + j, toks[j + 1]] = 40.0
        info.append(toks)
    max_length = 30   # slot 0: len 20 -> at most 10 tokens; slot 1: len 21 -> 9 ; slot 3: len 23 -> 7
    dn = torch.tensor(ns, dtype=torch.int32, device=DEV)
    seq_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    prefix = seq_len - 1
    fin = torch.zeros((B,), dtype=torch.int32, device=DEV)
    fin[1] = 1                                       # slot 1 finished earlier: must be left alone
    at = torch.zeros((B, R), dtype=torch.int32, device=DEV)
    ac = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    an = torch.zeros((B, R), dtype=torch.int32, device=DEV)
    acc = ops.Accept(V, R, 1.0, [2], 10 ** 6, DEV, bound_walk=True)
    ml = torch.tensor([max_length], dtype=torch.int32, device=DEV)
    r = torch.arange(stride, device=DEV)
    kc = torch.zeros((B, 1, 1, stride, 128), dtype=torch.bfloat16, device=DEV)
    kc[..., 0] = r.to(torch.bfloat16)
    kc[..., 1] = torch.arange(B, device=DEV).to(torch.bfloat16)[:, None, None, None]
    vc = kc.clone()
    k0 = kc.clone()
    acc.run(logits, ids, mask, dn, seq, seq_len, at, ac, an, prefix, fin, batch=B, rows_per_slot=rps, max_length=ml)
    ops.kv_compact(kc, vc, an, ac, prefix, batch=B)
    torch.cuda.synchronize()
    assert ac.tolist() == [10, 0, 0, 7]
    assert seq_len.tolist() == [30, 21, 22, 30] and prefix.tolist() == [29, 20, 21, 29]
    assert fin.tolist() == [1, 1, 0, 1]              # slots 0 and 3 reached max_length
    for s_ in (0, 3):
        c = int(ac[s_])
        assert at[s_, :c].tolist() == info[s_][1:c + 1] and an[s_, :c].tolist() == list(range(c))
        assert seq[s_, lens[s_]:lens[s_] + c].tolist() == info[s_][1:c + 1]
    assert torch.equal(kc, k0) and torch.equal(vc, k0)  # chains are contiguous: nothing moves


def test_multinomial_accept_draws_from_softmax():
    """do_sample (pretrained_model.py:835-837: softmax of the processed scores, then multinomial): the Gumbel-max
    draws of k_row_argmax must follow softmax(penalised logits) - chi-square over 6400 draws (64 rows x 100 steps, the
    step counter advancing on the device), and differ from step to step"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(3)
    V, R = 24, 64
    base = (torch.randn((V,), device=DEV) * 1.5).to(torch.bfloat16)
    logits = base[None].repeat(R, 1).contiguous()
    for penalty in (1.0, 1.3):
        acc = ops.Accept(V, R, penalty, [2], 10 ** 6, DEV)
        ids = torch.full((R,), 5, dtype=torch.int32, device=DEV)
        mask = _mask_tensor(np.array([1 << i for i in range(R)], dtype=np.uint64) | np.uint64(1), R)  # stars: no paths
        seq = torch.zeros((512,), dtype=torch.int32, device=DEV)
        seq[:4] = torch.tensor([5, 7, 9, 5], dtype=torch.int32)
        rng = torch.tensor([1234, 0], dtype=torch.int32, device=DEV)
        counts = torch.zeros((V,), dtype=torch.float64)
        draws = []
        for step in range(100):
            seq_len = torch.tensor([4], dtype=torch.int32, device=DEV)
            prefix = torch.tensor([3], dtype=torch.int32, device=DEV)
            fin = torch.zeros((1,), dtype=torch.int32, device=DEV)
            at, ac, an = (torch.zeros((R,), dtype=torch.int32, device=DEV), torch.zeros((1,), dtype=torch.int32, device=DEV),
                          torch.zeros((R,), dtype=torch.int32, device=DEV))
            acc.run(logits, ids, mask, torch.tensor([R], dtype=torch.int32, device=DEV), seq, seq_len, at, ac, an,
                    prefix, fin, rng=rng)
            rt = acc.workspace[:R].cpu()
            draws.append(rt.tolist())
            counts += torch.bincount(rt.long(), minlength=V).double()
        assert int(rng[1]) == 100 and draws[0] != draws[1]
        sc = base.float().cpu()
        if penalty != 1.0:  # RepetitionPenaltyLogitsProcessor on the context {5, 7, 9} (+ the path token 5)
            for t in (5, 7, 9):
                v = sc[t].to(torch.bfloat16).float()
                sc[t] = (v * penalty if v < 0 else v / penalty).to(torch.bfloat16).float()
        p = torch.softmax(sc.double(), 0)
        exp = p * counts.sum()
        keep = exp > 5
        chi2 = float((((counts - exp) ** 2) / exp)[keep].sum())
        assert chi2 < 2.0 * int(keep.sum()) + 20, (penalty, chi2, int(keep.sum()))


def test_moe_router():
    """pia_moe_router vs the reference's router arithmetic (mixtral/modeling_mixtral.py:721-727): bf16 gate Linear,
    fp32 softmax, top-2, renormalise, bf16; dense [rows, E] output"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(9)
    rows, H, E = 64, 4096, 8
    y = torch.randn((rows, H), device=DEV).to(torch.bfloat16)
    g = (torch.randn((E, H), device=DEV) * 0.05).to(torch.bfloat16)
    dense = torch.full((rows, E), 5.0, dtype=torch.bfloat16, device=DEV)
    ops.moe_router(y, g, 2, dense)
    logits = torch.mm(y, g.t())
    probs = torch.softmax(logits.float(), dim=1)
    w, sel = torch.topk(probs, 2, dim=-1)
    w = (w / w.sum(dim=-1, keepdim=True)).to(torch.bfloat16)
    ref = torch.zeros((rows, E), dtype=torch.bfloat16, device=DEV).scatter_(1, sel, w)
    torch.cuda.synchronize()
    assert ((dense != 0).sum(1) == 2).all()
    assert torch.allclose(dense.float().sum(1), torch.ones(rows, device=DEV), atol=1e-2)
    srt = probs.sort(dim=1, descending=True).values
    clear = (srt[:, 1] - srt[:, 2]) > 5e-3              # rows whose 2nd / 3rd experts are not a bf16 near-tie
    assert clear.float().mean() > 0.8
    assert torch.equal((dense != 0)[clear], (ref != 0)[clear])
    assert torch.allclose(dense[clear].float(), ref[clear].float(), atol=1.5e-2)


@pytest.mark.parametrize('N,K,split', [(256, 128, 1), (12288, 4096, 1), (4096, 4096, 4), (22016, 4096, 1),
                                       (4096, 11008, 4), (32000, 4096, 1), (4096, 4096, 1), (1024, 14336, 7)])
def test_gemm_weight_streaming(N, K, split):
    """wgmma weight-streaming GEMM vs an fp32 matmul of the same bf16 operands (nn.Linear semantics,
    modeling_llama.py:254-256/:303/:185-186/:769).  Checked against an fp64 reference with the scale-aware comparator of
    tests/gemm_ref.py (one bf16 rounding plus an fp32-accumulation bound, no absolute floor)."""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(N + K)
    w = (torch.randn((N, K), device=DEV) * 0.05).to(torch.bfloat16)
    x = torch.randn((64, K), device=DEV).to(torch.bfloat16)
    g = ops.Gemm(w, x, split_k=split)
    out = g.run(64)
    torch.cuda.synchronize()
    ref, mass = gemm_ref.reference(x, w)
    if N % 128 == 0:  # the HBM-tiled weight layout gives bit-identical results (same MMA order)
        gt = ops.Gemm(ops.tile_weight(w), x, split_k=split, tiled=True)
        assert torch.equal(gt.run(64), out)
        # stream-K: equal unit ranges per SM + in-kernel fix-up; deterministic from launch to launch
        gs = ops.Gemm(ops.tile_weight(w), x, split_k=-1, tiled=True)
        o1 = gs.run(64).clone()
        o2 = gs.run(64).clone()
        torch.cuda.synchronize()
        assert torch.equal(o1, o2)
        gemm_ref.assert_close(o1, ref, mass, K, K // 64, 'stream-K')   # at most one fix-up slot per chunk
        # cluster split-K: 2 / 4 / 8 K splits of a tile reduce through DSMEM in split order; bf16 out, deterministic
        for cs in (2, 4, 8):
            if K // 64 < cs or -(-(K // 64) // (-(-(K // 64) // cs))) != cs:   # the K chunks must split into exactly cs parts
                continue
            for tiled, wt in ((True, ops.tile_weight(w)), (False, w)):
                gc = ops.Gemm(wt, x, split_k=-cs, tiled=tiled)
                assert gc.splits == 1
                c1 = gc.run(64).clone()
                c2 = gc.run(64).clone()
                torch.cuda.synchronize()
                assert torch.equal(c1, c2)
                gemm_ref.assert_close(c1, ref, mass, K, cs, f'cluster {cs}')
            oc = gc.out
            oc.fill_(7.0)
            gc.run(5)
            torch.cuda.synchronize()
            gemm_ref.assert_close(oc[:5], ref[:5], mass[:5], K, cs, f'cluster {cs}, 5 rows')
            assert float(oc[5:].float().min()) == 7.0
    if g.splits == 1:
        got = out
    else:
        assert out.shape == (g.splits, 64, N)
        got = gemm_ref.slice_sum(out)
    gemm_ref.assert_close(got, ref, mass, K, g.splits)
    # fewer live rows: rows beyond `rows` are left untouched
    if g.splits == 1:
        out.fill_(7.0)
        g.run(5)
        torch.cuda.synchronize()
        gemm_ref.assert_close(out[:5], ref[:5], mass[:5], K, 1, '5 rows')
        assert float(out[5:].float().min()) == 7.0


def test_gemm_fused_silu_epilogue_matches_unfused():
    """gate_up GEMM with the SiLU(gate)*up epilogue == plain GEMM followed by k_silu_mul, bit for bit"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(5)
    inter, K = 1024, 512
    w = (torch.randn((2 * inter, K), device=DEV) * 0.05).to(torch.bfloat16)
    x = torch.randn((64, K), device=DEV).to(torch.bfloat16)
    gu = ops.Gemm(ops.tile_weight(w), x, tiled=True).run(64)
    ref = torch.empty((64, inter), dtype=torch.bfloat16, device=DEV)
    ops.silu_mul(gu, ref)
    got = torch.zeros_like(ref)
    ops.Gemm(ops.tile_weight(ops.interleave_gate_up(w)), x, tiled=True).set_silu().run(64, out=got)
    torch.cuda.synchronize()
    assert torch.equal(got, ref)


def test_l2_prefetch_is_a_pure_hint():
    """pia_l2_prefetch: contiguous and strided (tile-interleaved) ranges, paced and unpaced; data untouched, bad
    arguments rejected"""
    from painlessinferenceacceleration_b200.common import ops
    w = torch.randn((1 << 22,), device=DEV).to(torch.bfloat16)   # 8 MB
    ref = w.clone()
    n0 = ops.launch_count()
    ops.l2_prefetch(w)
    ops.l2_prefetch(w, n_ranges=8, stride_bytes=1 << 20, range_bytes=3 * 16384, gbytes_per_s=2000.0)
    ops.l2_prefetch(w, range_bytes=4096, offset_bytes=32)
    torch.cuda.synchronize()
    assert ops.launch_count() - n0 == 3
    assert torch.equal(w, ref)
    with pytest.raises(Exception):
        ops.l2_prefetch(w, range_bytes=100)                 # not a multiple of 16
    with pytest.raises(Exception):
        ops.l2_prefetch(w, n_ranges=2, stride_bytes=16, range_bytes=64)   # overlapping ranges


def test_grouped_gemm_and_moe_combine():
    """all experts in one launch (pia_gemm_plan_create_grouped) + the routing-weighted sum in expert order
    (pia_moe_combine) vs the eager per-expert loop (mixtral/modeling_mixtral.py:734-759, dense restatement)"""
    from painlessinferenceacceleration_b200.common import ops
    torch.manual_seed(5)
    E, N, K, R = 4, 256, 320, 64
    w = (torch.randn((E, N, K), device=DEV) * 0.05).to(torch.bfloat16)
    x = torch.randn((R, E * K), device=DEV).to(torch.bfloat16)
    g = ops.Gemm.grouped(w, x)
    ye = g.run(64)
    torch.cuda.synchronize()
    assert ye.shape == (E, 64, N)
    for e in range(E):
        ref, mass = gemm_ref.reference(x[:, e * K:(e + 1) * K], w[e])
        gemm_ref.assert_close(ye[e], ref, mass, K, 1, f'expert {e}')
    dense = torch.zeros((R, E), device=DEV, dtype=torch.bfloat16)
    sel = torch.stack([torch.randperm(E, device=DEV)[:2] for _ in range(R)])
    dense.scatter_(1, sel, torch.rand((R, 2), device=DEV).to(torch.bfloat16))
    out = torch.empty((R, N), dtype=torch.bfloat16, device=DEV)
    ops.moe_combine(ye, dense, out)
    ref = torch.zeros((R, N), dtype=torch.bfloat16, device=DEV)
    for e in range(E):
        ref += ye[e] * dense[:, e:e + 1]
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
