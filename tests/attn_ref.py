# -*- coding: utf-8 -*-
"""Plain-torch restatement of k_tree_attn (csrc/tree_attn.cu) for the attention tests: the visibility rule of the
header, an exact fp64 reference, an fp32 emulation of the kernel's arithmetic, the comparator, beacon inputs and the
wrong rules (mutations) the comparator must reject.  Runs on any device; nothing here needs a GPU."""
import math

import numpy as np
import torch

LOG2E = 1.4426950408889634
WORD = (1 << 64) - 1

# ------------------------------------------------------------------------------------------------------------ trees
def tree(rng, n, max_depth=8):
    """(parent, rows) of a random DFS-pre-order tree of n <= 128 nodes, as the trie emits it: node i hangs off a node
    on the path from i - 1 to the root; rows[i] = python int with bit j set iff j is i or an ancestor of i"""
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
    return parent[:n], rows


def sibling_pair(parent):
    """(i, s): s the last node that has an earlier sibling, i its first sibling (s is hidden from row i); or None"""
    for s in range(len(parent) - 1, 0, -1):
        for i in range(1, s):
            if parent[i] == parent[s]:
                return i, s
    return None


def mask_words(trees, R, rps, device='cpu'):
    """[len(trees) * rps, R // 64] int64 mask rows: slot s's tree in rows [s * rps, s * rps + n)"""
    W = R // 64
    m = np.zeros((len(trees) * rps, W), dtype=np.uint64)
    for s_, rows in enumerate(trees):
        for i, r in enumerate(rows):
            for w in range(W):
                m[s_ * rps + i, w] = np.uint64((int(r) >> (64 * w)) & WORD)
    return torch.from_numpy(m.view(np.int64)).to(device)


# ------------------------------------------------------------------------------------------------ reference
def visibility(rows, n, P, pad):
    """[n, P + n] bool, the contract of include/pia_b200.h: prefix keys [pad, P) are visible to every row (none when
    pad >= P), draft key j is visible to row i iff bit j of rows[i] is set (bits 64..127 live in mask word 1)"""
    vis = torch.zeros((n, P + n), dtype=torch.bool)
    if pad < P:
        vis[:, pad:P] = True
    bits = [(int(rows[i]) >> j) & 1 for i in range(n) for j in range(n)]
    vis[:, P:] = torch.tensor(bits, dtype=torch.bool).view(n, n)
    return vis


def depths(rows, n, words=2):
    """tree depth of each node: popcount of its mask row - 1 (words=1: mask word 0 alone, a wrong rule)"""
    keep = WORD if words == 1 else (1 << 128) - 1
    return [bin(int(rows[i]) & keep).count('1') - 1 for i in range(n)]


def alibi_positions(rows, n, P, pad, qpos_pad=True, draft_pos='depth', depth_words=2):
    """ALiBi at tree positions (pia_tree_attn_alibi_fwd): row i sits at qpos = max(P - pad, 0) + depth(i), cached key
    j at j - pad, draft key k at max(P - pad, 0) + depth(k).  The keyword arguments state wrong rules: the pad left
    out of the cached keys' offset, a draft key at its DFS index, depth over mask word 0 only"""
    base = max(P - pad, 0)
    d = torch.tensor(depths(rows, n, depth_words), dtype=torch.float64)
    qpos = base + d
    kpre = torch.arange(P, dtype=torch.float64) - (pad if qpos_pad else 0)
    kdraft = base + (d if draft_pos == 'depth' else torch.arange(n, dtype=torch.float64))
    return qpos, torch.cat([kpre, kdraft])


def reference(q, kc, vc, rows, n, P, pad, G=None, scale_mul=1.0, slopes=None, vis=None, kv_map='div', qpos_pad=True,
              draft_pos='depth', depth_words=2):
    """exact attention in fp64: out[i, h] = softmax_j(q_i.k_j * scale_mul / sqrt(D) [+ slope_h (kpos_j - qpos_i)]) v_j
    over the visible keys j of row i; query head h reads KV head h // G.  q [>= n, Hq, D], kc / vc [Hkv, >= P + n, D].
    vis / kv_map='mod' / qpos_pad / draft_pos / depth_words replace a rule by a wrong one (see `mutations`).
    Returns [n, Hq, D] float64."""
    Hq, D = q.shape[1], q.shape[2]
    Hkv, L = kc.shape[0], P + n
    G = G or Hq // Hkv
    dev = q.device
    idx = torch.tensor([h // G if kv_map == 'div' else h % Hkv for h in range(Hq)], device=dev)
    k = kc[idx, :L].double()
    v = vc[idx, :L].double()
    s = torch.einsum('ihd,hjd->hij', q[:n].double(), k) * (scale_mul / math.sqrt(D))
    if slopes is not None:
        qpos, kpos = alibi_positions(rows, n, P, pad, qpos_pad, draft_pos, depth_words)
        s = s + slopes.double().to(dev)[:, None, None] * (kpos.to(dev)[None, None, :] - qpos.to(dev)[None, :, None])
    if vis is None:
        vis = visibility(rows, n, P, pad)
    s = s.masked_fill(~vis.to(dev)[None], float('-inf'))
    return torch.einsum('hij,hjd->ihd', torch.softmax(s, -1), v)


# ------------------------------------------------------------------------------------------------ comparator
TOL = 2.0 ** -6


def scores(got, ref):
    """|got - ref| / (2^-6 (|ref| + rms_d(ref))) per element, rms_d = the RMS of ref over the head dim of that
    (row, head).  The comparator accepts when every score is <= 1.  Where the bound comes from:

    The kernel computes p_j = exp(s_j - m) in fp32 and rounds it to bf16 before both the PV product and the row sum
    l = sum_j p^_j, so its output, before the final rounding, is the exact average of v under the perturbed weights
    p^_j = p_j (1 + e_j), |e_j| <= 2^-9 (bf16 keeps 8 significant bits).  Written with the exact weights w_j:

        o^ - o = sum_j w_j e_j (v_j - o) / (1 + sum_j w_j e_j).

    The e_j are rounding errors of unrelated numbers: mean ~0, spread 2^-9 / sqrt(3), so the sum is a random walk of
    size 2^-9 / sqrt(3) * sqrt(sum_j w_j^2 (v_j - o)^2).  When a few keys carry the weight (peaked softmax, beacon
    inputs), v_j ~ o for them and the term is a few 2^-9 |o|.  When the weight is spread over N_eff keys of
    unrelated values (flat softmax, random inputs), it is 2^-9 / sqrt(3) * sigma_v / sqrt(N_eff), and the output
    itself is an average of N_eff such values, of size sigma_v / sqrt(N_eff) ~ rms_d(ref).  The final bf16 rounding
    adds <= 2^-9 |o|.  So the error is a few 2^-9 (|ref| + rms_d(ref)); the maximum over 10^5 - 10^6 elements
    (a ~5 sigma event) stays below 2^-7 (ALiBi / scale / fp32 sums / ex2.approx / the split merge are ~2^-20
    relative and do not count), and 2^-6 keeps 2x headroom.  test_gpu_attn_power checks the bound on an emulation of
    the kernel's arithmetic (`emulate`) and on the kernel itself."""
    got, ref = got.double(), ref.double().to(got.device)
    rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    den = TOL * (ref.abs() + rms)
    diff = (got - ref).abs()
    return torch.where(den > 0, diff / den.clamp_min(1e-300), torch.where(diff > 0, float('inf'), 0.0))


def worst(got, ref):
    return float(scores(got, ref).max())


def assert_close(got, ref, msg=''):
    """the comparator: every element within 2^-6 (|ref| + rms_d(ref)) of the reference (see `scores`)"""
    w = worst(got, ref)
    assert w <= 1.0, f'{msg} worst score {w:.3g} (fraction of the tolerance used)'
    return w


# ------------------------------------------------------------------------------------------------ kernel emulation
def scale_log2(scale_mul, D):
    """the host's fp32 scale: scale_mul * log2(e) / sqrtf(D)"""
    return float(np.float32(np.float32(scale_mul) * np.float32(LOG2E)) / np.sqrt(np.float32(D)))


def emulate(q, kc, vc, rows, n, P, pad, scale_mul=1.0, slopes=None, n_split=1):
    """the kernel's arithmetic in torch: fp32 scores of the bf16 operands, log2 domain, 128-key tiles in n_split
    contiguous ranges with an online softmax each (p = bf16(exp2(t - m)), l = sum of the rounded p, PV in fp32), the
    ranges merged in fp32 (weights exp2(m_i - M)), one bf16 rounding of the normalised output"""
    Hq, D = q.shape[1], q.shape[2]
    Hkv, L = kc.shape[0], P + n
    G = Hq // Hkv
    idx = torch.tensor([h // G for h in range(Hq)], device=q.device)
    k, v = kc[idx, :L].float(), vc[idx, :L].float()
    t = torch.einsum('ihd,hjd->hij', q[:n].float(), k) * scale_log2(scale_mul, D)
    if slopes is not None:
        qpos, kpos = alibi_positions(rows, n, P, pad)
        sl2 = slopes.float().cpu() * np.float32(LOG2E)
        t = t + (sl2[:, None, None] * (kpos[None, None, :] - qpos[None, :, None]).float()).to(t.device)
    t = t.masked_fill(~visibility(rows, n, P, pad).to(t.device)[None], float('-inf'))
    T = (L + 127) // 128
    tps = (T + n_split - 1) // n_split
    parts = []
    for sp in range(n_split):
        m = torch.full((Hq, n), float('-inf'), device=t.device)
        l = torch.zeros((Hq, n), device=t.device)
        o = torch.zeros((Hq, n, D), device=t.device)
        for tl in range(sp * tps, min(sp * tps + tps, T)):
            tt = t[..., 128 * tl:min(L, 128 * tl + 128)]
            m_new = torch.maximum(m, tt.amax(-1))
            m_use = torch.where(m_new == float('-inf'), 0.0, m_new)
            alpha = torch.where(m == float('-inf'), 0.0, torch.exp2(m - m_use))
            p = torch.exp2(tt - m_use[..., None]).to(torch.bfloat16).float()
            l = l * alpha + p.sum(-1)
            o = o * alpha[..., None] + torch.einsum('hij,hjd->hid', p, v[:, 128 * tl:128 * tl + p.shape[-1]])
            m = m_new
        parts.append((m, l, o))
    if n_split == 1:
        m, l, o = parts[0]
    else:
        M = torch.stack([pm for pm, _, _ in parts]).amax(0)
        l = torch.zeros_like(M)
        o = torch.zeros_like(parts[0][2])
        for pm, pl, po in parts:
            w = torch.where(pm == float('-inf'), 0.0, torch.exp2(pm - M))
            l = l + pl * w
            o = o + po * w[..., None]
    inv = torch.where(l > 0, 1.0 / l, 0.0)
    return (o * inv[..., None]).to(torch.bfloat16).permute(1, 0, 2)


# ------------------------------------------------------------------------------------------------ beacon inputs
Q0 = 4.0          # every query row's component along head dim 0 (the beacon direction)
BEACON_NATS = 7.0
SENTINEL_NATS = 16.0
SENTINEL_V = 256.0


def key_amp(nats, D, scale_mul):
    """the dim-0 value of a key that scores `nats` above a dim-0-free key for every query row"""
    return nats * math.sqrt(D) / (Q0 * scale_mul)


def sentinel_kv(D, scale_mul, shape_prefix=(), device='cpu'):
    """a key that would dominate any row that saw it and a +-256 value: finite, so 0 * v = 0 for a hidden key"""
    k = torch.zeros(shape_prefix + (D,), device=device)
    k[..., 0] = key_amp(SENTINEL_NATS, D, scale_mul)
    v = SENTINEL_V * (1 - 2 * (torch.arange(D, device=device) % 2)).float().expand(shape_prefix + (D,))
    return k.to(torch.bfloat16), v.to(torch.bfloat16)


def beacon_keys(parent, n, P, pad, split_edges=()):
    """(beacons, sentinels): key indices in [0, P + n + 2).  Beacons: the first visible key (pad) and P - 1, the keys
    on both sides of every 128-key tile boundary, `split_edges` (first and last key of each KV split), the first node
    at each depth (an ancestor of the deeper nodes) and L - 1.  A chosen prefix key below pad becomes a sentinel, as
    do pad - 1, keys L and L + 1, and the sibling s of `sibling_pair` (hidden from its sibling's row)"""
    L = P + n
    cand = {pad, P - 1, L - 1} | set(split_edges)
    for b in range(128, L, 128):
        cand |= {b - 1, b}
    seen = set()
    d = [0] * n
    for i in range(1, n):
        d[i] = d[parent[i]] + 1
    for i in range(n):
        if d[i] not in seen:
            seen.add(d[i])
            cand.add(P + i)
    beacons, sentinels = set(), {L, L + 1}
    for x in cand:
        if 0 <= x < L:
            (sentinels if x < min(pad, P) else beacons).add(x)
    if 0 <= pad - 1 < P:
        sentinels.add(pad - 1)
    sib = sibling_pair(parent)
    if sib is not None:
        sentinels.add(P + sib[1])
    return sorted(beacons - sentinels), sorted(sentinels)


def beacon_data(parent, n, P, pad, Hq, Hkv, D, n_keys, scale_mul=1.0, split_edges=(), gen=None):
    """q [n, Hq, D], k / v [Hkv, n_keys, D] bf16 (n_keys >= P + n + 2): every query row has Q0 along dim 0, a beacon
    key scores ~7 nats above the background and carries a one-hot value in a dimension of its own (cycling over
    1..D-1), a sentinel key scores 16 nats above the background and carries +-256.  Background keys have nothing
    along dim 0 and small random values elsewhere."""
    beacons, sentinels = beacon_keys(parent, n, P, pad, split_edges)
    q = 0.3 * torch.randn((n, Hq, D), generator=gen)
    q[..., 0] = Q0
    k = 0.7 * torch.randn((Hkv, n_keys, D), generator=gen)
    k[..., 0] = 0.0
    v = 0.7 * torch.randn((Hkv, n_keys, D), generator=gen)
    for c, x in enumerate(beacons):
        k[:, x, 0] = key_amp(BEACON_NATS, D, scale_mul)
        v[:, x] = 0.0
        v[:, x, 1 + c % (D - 1)] = 1.0
    ks, vs = sentinel_kv(D, scale_mul)
    for x in sentinels:
        if x < n_keys:
            k[:, x], v[:, x] = ks.float(), vs.float()
    return q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ wrong rules
SINGLE_KEY = ('key P-1 hidden', 'sibling leaked', 'boundary key hidden')


def mutations(parent, rows, n, P, pad, Hq, Hkv, scale_mul=1.0, alibi=False):
    """name -> keyword arguments of `reference` that replace one rule by a wrong one, for the wrong rules that change
    something on this case"""
    base = visibility(rows, n, P, pad)
    out = {}

    def vis(f):
        v = base.clone()
        f(v)
        return {'vis': v}

    if pad > 0 and P > 0:
        out['pad ignored'] = vis(lambda v: v[:, :P].fill_(True))
    if 0 < pad <= P:
        out['pad off by one'] = vis(lambda v: v[:, pad - 1].fill_(True))
    if pad < P:
        out['key P-1 hidden'] = vis(lambda v: v[:, P - 1].fill_(False))
    inner = [b for b in range(128, P, 128) if b >= pad]
    if inner:
        out['boundary key hidden'] = vis(lambda v: v[:, inner[0]].fill_(False))
    full = [t for t in range(P // 128) if 128 * t >= pad]
    if full:
        out['first full prefix tile dropped'] = vis(lambda v: v[:, 128 * full[0]:128 * full[0] + 128].fill_(False))
        out['last full prefix tile dropped'] = vis(lambda v: v[:, 128 * full[-1]:128 * full[-1] + 128].fill_(False))
    chain = torch.tril(torch.ones((n, n), dtype=torch.bool))
    if not torch.equal(chain, base[:, P:]):
        out['tree replaced by the causal chain'] = vis(lambda v: v[:, P:].copy_(chain))
    if n > 1:
        out['ancestors hidden'] = vis(lambda v: v[:, P:].copy_(torch.eye(n, dtype=torch.bool)))
    sib = sibling_pair(parent)
    if sib is not None:
        out['sibling leaked'] = vis(lambda v: v[sib[0], P + sib[1]].fill_(True))
    if Hq != Hkv and Hkv > 1:
        out['GQA map h % Hkv'] = {'kv_map': 'mod'}
    out['scale_mul x1.05'] = {'scale_mul': scale_mul * 1.05}
    if alibi:
        if 0 < pad < P:
            out['ALiBi qpos without the pad'] = {'qpos_pad': False}
        if depths(rows, n) != list(range(n)):
            out['ALiBi draft key at its DFS index'] = {'draft_pos': 'dfs'}
        if n > 64:
            out['ALiBi depth over mask word 0 only'] = {'depth_words': 1}
    return out
