# -*- coding: utf-8 -*-
"""Accept-step tests that can fail (csrc/accept.cu: k_row_argmax, k_accept_walk, k_kv_compact) against the plain
restatement of tests/accept_ref.py.

CPU half: the case table run through accept_ref gives the answers it was built for, and every wrong kernel of
accept_ref.MUTATIONS changes at least one expected output of the GPU case table.

GPU half (pytest.mark.gpu):
  * the repetition penalty bit for bit over every finite bf16 score at six penalties: two rows per value
    [pen(x), x] and [x, pen(x)] with x's token in the context pick token 0 only if the kernel's penalised x equals
    accept_ref.penalise(x) exactly; the host path (transformers' RepetitionPenaltyLogitsProcessor on CUDA, which the
    loop runs whenever a caller passes logits processors) picks the same tokens;
  * first-index, NaN-greatest arg-max at real vocabularies (second chunks per thread past 8192, odd row strides,
    ties across threads and warps, +-0, +-inf, NaN), with and without a penalty;
  * every draft node's pick on random pre-order trees of 1-128 nodes (both mask words) against the processor applied to
    the reference's update_input_ids, including the > 48 KB shared-memory bitmap;
  * the walk (tokens, nodes, count, sequence, lengths, finished) and the KV compaction bit for bit."""
import ctypes as C
import functools
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import accept_ref as ar

DEV = 'cuda:0'
BIG = ar.BIG
PROBE_P = (1.04, 1.1, 1.2, 1.3, 1.92, 0.85)
TIE_V = (24, 8191, 8192, 8193, 32000, 50257, 65024, 151936, 250880)
TIE_P = 1.2
W = 8 * 32            # tokens one warp of k_row_argmax covers per pass (8 per thread)
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ case table
def finite_bf16():
    x = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return x[torch.isfinite(x.float())]


@functools.lru_cache(maxsize=None)
def probe_case(p):
    """two rows per finite bf16 x with r = penalise(x, p): [r, x] with token 1 in the context and [x, r] with token 0
    in it.  The first picks 0 only if pen(x) <= r, the second only if pen(x) >= r: both pick 0 iff pen(x) == r."""
    x = finite_bf16()
    r = ar.penalise(x, p)
    logits = torch.stack([torch.stack([r, x], 1), torch.stack([x, r], 1)], 1).reshape(-1, 2)
    ctx = torch.tensor([[1], [0]]).repeat(x.numel(), 1)
    return logits, ctx


def _tie_rows(V, p):
    """(row, penalised tokens, intended pick or None) for one vocabulary"""
    g = torch.Generator().manual_seed(V + int(p * 100))
    rows = []

    def base():
        return torch.randn((V,), generator=g).clamp(-3, 3)

    def spots(pos, val=8.0):
        x = base()
        x[list(pos)] = val
        return x

    groups = [(0,), (V - 1,), (3, 5), (8 * 5 + 1, 8 * 2 + 7), (W * 3 + 2, W + 5), (W * 31 + 4, W * 7),
              (8 * 1023 + 7, 8 * 500), (8 * 100, 8192 + 3), (8192 + 1, 8000), (8192 + 5, V - 1), (V - 2, V - 1),
              (8191, V - 1), (1, 8 * 1023, 8192 * 2 + 1), (W * 4 + 7, W * 4 + 6, V - 3)]
    seen = set()
    for pos in groups:
        pos = tuple(sorted(set(pos)))
        if max(pos) >= V or min(pos) < 0 or pos in seen:
            continue
        seen.add(pos)
        if p == 1.0:
            rows.append((spots(pos), [], pos[0]))
        else:   # the first maximum is penalised below 8: the next one wins (a lone maximum: the row decides)
            rows.append((spots(pos), [pos[0]], pos[1] if len(pos) > 1 else None))
    a, b = min(W * 2 + 3, V - 2), min(8192 + 1, V - 1)
    ninf = float('-inf')
    for i, j in ((a, b), (b, a), (0, V - 1)):
        x = torch.full((V,), ninf)
        x[i], x[j] = -0.0, 0.0
        rows.append((x, [i], min(i, j)))                       # -0.0 == +0.0, penalised or not
    x = spots([a], float('inf'))
    rows.append((x, [a], a))
    x = spots([a, b], float('inf'))
    rows.append((x, [b], min(a, b)))
    rows.append((torch.full((V,), ninf), [V - 1], 0))           # a row of -inf gives 0
    x = base()
    x[b] = float('nan')
    rows.append((x, [b], b))
    x = spots([0], float('inf'))
    x[a], x[b] = float('nan'), float('nan')
    rows.append((x, [a, 0], min(a, b)))                       # the first NaN beats +inf
    x = spots([0])
    x[V - 1] = float('nan')
    rows.append((x, [], V - 1))
    if p != 1.0:
        # a penalised score that lands exactly on another one: the lower index wins
        for y in (2.40625, 1.8515625, -2.0):
            y = torch.tensor([y]).to(torch.bfloat16)
            r = float(ar.penalise(y, p).float())
            for i, j in ((a, b), (b, a)):
                x = torch.full((V,), ninf)
                x[i], x[j] = float(y.float()), r
                rows.append((x, [i], min(i, j)))
    return rows


@functools.lru_cache(maxsize=None)
def tie_case(V, p):
    """logits [R, V] bf16, ctx [R, L] (each row's penalised tokens padded with a duplicate; a row without any gets a
    token where its score is far below the maximum), intended picks"""
    rows = _tie_rows(V, p)
    logits = torch.stack([r[0] for r in rows]).to(torch.bfloat16)
    L = max(max(len(r[1]) for r in rows), 1)
    ctx = []
    for x, t, _ in rows:
        t = list(t) or [int(torch.argmin(torch.nan_to_num(x, nan=0.0)))]
        ctx.append(t + [t[0]] * (L - len(t)))
    return logits, torch.tensor(ctx, dtype=torch.long), [r[2] for r in rows]


def pre_order_tree(rng, n, max_depth=32, force=None):
    """parent list and ancestor rows (bit a of rows[j]: a is j or an ancestor of j) of a random DFS-pre-order tree;
    force {node: parent} pins parents (a parent must lie on the current rightmost path)"""
    force = force or {}
    parent, depth = [-1], [0]
    for i in range(1, n):
        path = [i - 1]
        while parent[path[-1]] >= 0:
            path.append(parent[path[-1]])
        cands = [q for q in path if depth[q] < max_depth]
        q = force[i] if force.get(i) in path else cands[int(rng.integers(0, len(cands)))]
        parent.append(q)
        depth.append(depth[q] + 1)
    rows = [1]
    for i in range(1, n):
        rows.append(rows[parent[i]] | (1 << i))
    return parent, rows


def tree_ids(rng, parent, V, pool):
    """node tokens: siblings distinct (the trie's children are dict keys), many taken from the context pool"""
    ids = [int(pool[-1])]
    for j in range(1, len(parent)):
        used = {ids[k] for k in range(1, j) if parent[k] == parent[j]}
        while True:
            t = int(rng.choice(pool)) if rng.random() < 0.5 else int(rng.integers(3, V - 8))
            if t not in used:
                break
        ids.append(t)
    return ids


def context(rng, V, length, pads):
    """left pads (id 0), duplicates, token V - 1"""
    pool = rng.integers(3, V - 8, size=12)
    c = [0] * pads + [int(rng.choice(pool)) for _ in range(length - pads)]
    c[pads + 1] = V - 1
    return c


def path_to(parent, j):
    q = []
    while j >= 0:
        q.append(j)
        j = parent[j]
    return q[::-1]


def _slot(n, ids, rows, ctx, logits, fin0=0, why=None):
    return SimpleNamespace(n=n, ids=ids, rows=rows, ctx=ctx, logits=logits, fin0=fin0, why=why or {})


def _background(g, rps, V):
    return torch.randn((rps, V), generator=g).clamp(-3, 3)


def penalty_slot(rng, g, V, rps, n, pads, p):
    """a random tree whose rows are decided by the penalty set: per row either a token off the node's path (a sibling
    or a descendant) is top-1 by a margin penalising it would flip, or a token of the set (node k's own, an
    ancestor's, the pad id 0, V - 1) is top-1 and loses to the runner-up once penalised.  why[k]: the intended pick."""
    parent, rows = pre_order_tree(rng, n)
    ctx = context(rng, V, int(rng.integers(20, 200)), pads)
    ids = tree_ids(rng, parent, V, np.array(ctx[pads:]))
    ctx[-1] = ids[0]
    x = _background(g, rps, V)
    why = {}
    assert p > 1.0
    for k in range(n):
        S = set(ar.penalty_tokens(ctx, ids, rows, k))
        on_path = {a for a in range(n) if (rows[k] >> a) & 1}
        off = [s for s in range(1, n) if s not in on_path and ids[s] not in S]
        own = [ids[k]] if k >= 1 and ids[k] not in set(ctx) | {ids[a] for a in on_path if a not in (0, k)} else []
        anc = [ids[a] for a in on_path if a not in (0, k)]
        kind = k % 5
        u = int(rng.integers(3, V))
        while u in S:
            u = int(rng.integers(3, V))
        if kind == 0 and off:
            top = ids[off[int(rng.integers(0, len(off)))]]
            if top == u:
                continue
            x[k, top], x[k, u] = 8.0, 7.5
            why[k] = top
            continue
        top = {1: own, 2: [0] if pads else [], 3: anc, 4: [V - 1]}.get(kind) or own or [V - 1]
        x[k, top[0]], x[k, u] = 8.0, 7.5
        why[k] = u
    return _slot(n, ids, rows, ctx, x.to(torch.bfloat16), why=why)


def vote_slot(rng, g, V, rps, n, len0, target, parent=None, eos_on_path=None, last=None, fin0=0, pads=0):
    """a tree whose rows along root -> target vote for the next node's token (30.0), the target row for `last`:
    the walk accepts exactly that path.  eos_on_path: (position, token) placed on the path's token list."""
    if parent is None:
        parent, rows = pre_order_tree(rng, n, max_depth=8)
    else:
        rows = [1]
        for i in range(1, n):
            rows.append(rows[parent[i]] | (1 << i))
    ctx = context(rng, V, len0, pads)
    ids = tree_ids(rng, parent, V, np.array(ctx[pads:]))
    route = path_to(parent, target) if n else []
    if eos_on_path is not None:
        i, e = eos_on_path
        ids[route[i]] = e
    if n:
        ctx[-1] = ids[0]
    x = _background(g, rps, V)
    for a, b in zip(route, route[1:]):
        x[a, ids[b]] = 30.0
    if n:
        kids = {ids[j] for j in range(1, n) if parent[j] == target}
        t = last if last is not None else int(rng.integers(3, V - 8))
        while t in kids:
            t += 1
        x[target, t] = 30.0
    return _slot(n, ids, rows, ctx, x.to(torch.bfloat16), fin0=fin0, why={'route': route})


def _launch(kind, batch, rps, V, p, slots, eos=(), stride=256, max_length=BIG, device_max_length=None,
            bound_walk=False):
    return SimpleNamespace(kind=kind, batch=batch, rps=rps, V=V, p=p, slots=slots, eos=list(eos), stride=stride,
                           max_length=max_length, device_max_length=device_max_length, bound_walk=bound_walk)


@functools.lru_cache(maxsize=None)
def tree_launches():
    """penalty sets on real trees: 1 x 128 at V = 250880 and 50257, 4 x 32, 2 x 64, and V = 400 000 (bitmap > 48 KB)"""
    out = []
    for seed, (batch, rps, V, ns, pads) in enumerate([(1, 128, 250880, [128], [5]), (1, 128, 50257, [97], [0]),
                                                      (4, 32, 32000, [32, 17, 1, 32], [3, 0, 1, 0]),
                                                      (2, 64, 151936, [64, 40], [0, 2]),
                                                      (1, 16, 400000, [16], [4])]):
        rng = np.random.default_rng(100 + seed)
        g = torch.Generator().manual_seed(100 + seed)
        slots = [penalty_slot(rng, g, V, rps, n, pd, 1.2) for n, pd in zip(ns, pads)]
        out.append(_launch('tree', batch, rps, V, 1.2, slots, eos=[2], stride=512))
    return out


def eos8(V):
    return [2] + [V - j for j in range(2, 9)]


@functools.lru_cache(maxsize=None)
def walk_launches(p):
    V = 32000
    out = []
    rng = np.random.default_rng(7)
    g = torch.Generator().manual_seed(7)
    # 128 nodes; the accepted path runs through nodes 62 .. 72 (mask word 0 -> word 1)
    force = {i: i - 1 for i in range(62, 73)}
    parent, _ = pre_order_tree(rng, 128, max_depth=8, force=force)
    out.append(_launch('walk', 1, 128, V, p, [vote_slot(rng, g, V, 128, 128, 40, 72, parent=parent)], eos=[2]))
    # a chain of depth 33 (branch_length 32) accepted whole; EOS (one of 8 ids) mid-path, the walk goes on
    chain = [-1] + list(range(32))
    s0 = vote_slot(rng, g, V, 64, 33, 30, 32, parent=chain)
    parent, _ = pre_order_tree(rng, 64, max_depth=8)
    deep = max(range(64), key=lambda j: len(path_to(parent, j)))
    s1 = vote_slot(rng, g, V, 64, 64, 25, deep, parent=parent, eos_on_path=(2, V - 5))
    out.append(_launch('walk', 2, 64, V, p, [s0, s1], eos=eos8(V)))
    # bound_walk with a device max_length, no EOS ids: a finished slot, an idle slot, a capped walk that also runs
    # into seq_stride, and a walk through token 2 (not an EOS here)
    chain = [-1] + list(range(31))
    parent, _ = pre_order_tree(rng, 32, max_depth=8)
    deep = max(range(32), key=lambda j: len(path_to(parent, j)))
    slots = [vote_slot(rng, g, V, 32, 20, 12, 5, fin0=1), vote_slot(rng, g, V, 32, 0, 9, 0),
             vote_slot(rng, g, V, 32, 32, 50, 31, parent=chain, pads=3),
             vote_slot(rng, g, V, 32, 32, 10, deep, parent=parent, eos_on_path=(1, 2))]
    out.append(_launch('walk', 4, 32, V, p, slots, eos=[], stride=64, device_max_length=70, bound_walk=True))
    # unbounded walk past seq_stride
    slots = [vote_slot(rng, g, V, 32, 12, 60, 11, parent=[-1] + list(range(11))),
             vote_slot(rng, g, V, 32, 32, 5, 31, parent=[-1] + list(range(31)), last=2),
             vote_slot(rng, g, V, 32, 1, 64, 0), vote_slot(rng, g, V, 32, 30, 33, 20)]
    out.append(_launch('walk', 4, 32, V, p, slots, eos=[2], stride=64, max_length=90))
    return out


def all_launches():
    return tree_launches() + walk_launches(1.0) + walk_launches(1.2)


COMPACT = [(50, [0]), (37, [0, 2, 3, 5, 30, 63, 64, 66, 100]), (0, []), (120, [0, 1, 2, 3, 9, 40, 70]),
           (60, [0, 1, 2, 4, 8, 16, 32, 64, 65, 66, 67, 127])]


@functools.lru_cache(maxsize=None)
def compact_cache(D):
    """[batch, layers + 1, kv heads, S, D] finite random bf16 bit patterns (exact in any copy); the last layer of each
    slot lies outside the layers handed to the kernel"""
    g = torch.Generator().manual_seed(D)
    shape = (len(COMPACT), 4, 2, 208, D)
    v = torch.randint(0, 0x7F00, shape, generator=g, dtype=torch.int32)
    s = torch.randint(0, 2, shape, generator=g, dtype=torch.int32)
    return (v - s * 0x8000).to(torch.int16)


# ------------------------------------------------------------------------------------------------ expected outputs
def expect_launch(f, L):
    """what the device holds after pia_accept on launch L under the rules f"""
    B, stride = L.batch, L.stride
    seq = torch.full((B * stride + 8,), -7, dtype=torch.int32)
    e = SimpleNamespace(picks={}, count=[], tokens=[], nodes=[], seq=seq, seq_len=[], prefix=[], fin=[])
    ml = L.device_max_length if L.device_max_length is not None else L.max_length
    for s, sl in enumerate(L.slots):
        len0 = len(sl.ctx)
        seq[s * stride:s * stride + len0] = torch.tensor(sl.ctx, dtype=torch.int32)
        picks = [ar.pick(f, sl.logits[k], f.penalty_tokens(sl.ctx, sl.ids, sl.rows, k), L.p) for k in range(sl.n)]
        e.picks.update({s * L.rps + k: t for k, t in enumerate(picks)})
        if sl.n == 0 or sl.fin0:
            toks, nodes, fin = [], [], bool(sl.fin0)
        else:
            toks, nodes, fin = f.walk(sl.ids, sl.rows, picks, L.eos, len0, ml, L.bound_walk)
        for i, t in enumerate(toks):
            if len0 + i < stride:
                seq[s * stride + len0 + i] = t
        e.count.append(len(toks))
        e.tokens.append(toks)
        e.nodes.append(nodes)
        e.seq_len.append(len0 + len(toks))
        e.prefix.append(len0 - 1 + len(toks))
        e.fin.append(int(fin))
    return e


def expect_compact(f, D):
    x = compact_cache(D).clone()
    for s, (p_old, nodes) in enumerate(COMPACT):
        if len(nodes) >= 1:
            for lyr in range(x.shape[1] - 1):
                for h in range(x.shape[2]):
                    x[s, lyr, h] = f.compact(x[s, lyr, h], p_old, nodes)
    return x


def _launch_outputs(e):
    return (sorted(e.picks.items()), e.count, e.tokens, e.nodes, e.seq.tolist(), e.seq_len, e.prefix, e.fin)


# ------------------------------------------------------------------------------------------------ CPU half
@pytest.mark.parametrize('p,n_diff', [(1.04, 254), (1.1, 0), (1.2, 508), (1.3, 0), (1.5, 0), (1.92, 253)])
def test_penalty_probe_separates_true_division_from_the_reciprocal(p, n_diff):
    """the positive scores where bf16(x / p) and bf16(x * fl32(1/p)) differ by an ulp: the probe holds every one"""
    x = finite_bf16()
    a = ar.penalise(x, p)
    b = ar.MUTATIONS['true division on the positive branch'].penalise(x, p)
    diff = (a.view(torch.int16) != b.view(torch.int16)) & (x.float() > 0)
    assert int(diff.sum()) == n_diff
    assert torch.equal(a[x.float() < 0], b[x.float() < 0])
    if p == 1.2:
        assert {1.8515625, 3.703125, 7.40625, 14.8125, 15.5625} <= set(x[diff].float().tolist())


def test_reciprocal_is_taken_in_double():
    """1 / fl32(p) and fl32(1 / p) differ at 1.92 (by one fp32 ulp, moving 760 positive bf16 scores); CUDA PyTorch
    uses the latter, and so does the accept config (ops.Accept)"""
    x = finite_bf16()
    single = (x.float() * (torch.tensor(1.0) / torch.tensor(1.92, dtype=torch.float32))).to(torch.bfloat16)
    assert float(ar.reciprocal(1.92)) != float(torch.tensor(1.0) / torch.tensor(1.92, dtype=torch.float32))
    assert int((single.view(torch.int16) != ar.penalise(x, 1.92).view(torch.int16))[x.float() > 0].sum()) == 760
    for p in PROBE_P:
        assert float(ar.reciprocal(p)) == float(C.c_float(1.0 / p).value)


@pytest.mark.parametrize('p', PROBE_P)
def test_probe_rows_pick_token_zero(p):
    logits, ctx = probe_case(p)
    assert logits.shape[0] == 2 * 65280
    assert not ar.pick_rows(ar.REF, logits, ctx, p).any()


@pytest.mark.parametrize('V', TIE_V)
def test_tie_rows_give_the_intended_first_index(V):
    for p in (1.0, TIE_P):
        logits, ctx, want = tie_case(V, p)
        got = ar.pick_rows(ar.REF, logits, ctx, p)
        pen = logits.clone()
        if p != 1.0:
            pen.scatter_(1, ctx, ar.penalise(pen.gather(1, ctx), p))
        assert torch.equal(got, torch.argmax(pen.float(), -1))        # torch.argmax on the CPU: a second opinion
        for i, w in enumerate(want):
            if w is not None:
                assert int(got[i]) == w, (V, p, i)


def _parent_walk(ids, rows, row_tok, eos, len0, max_length, bound_walk):
    """the walk in parent form (nearest ancestor = highest bit below j): an independent restatement of the reference's
    leaf-branch loop for trees whose siblings carry distinct tokens"""
    parent = [-1] + [(rows[j] & ((1 << j) - 1)).bit_length() - 1 for j in range(1, len(ids))]
    cap = max_length - len0 if bound_walk else BIG
    cur, toks, nodes = 0, [], []
    while True:
        toks.append(row_tok[cur])
        nodes.append(cur)
        nxt = [j for j in range(1, len(ids)) if parent[j] == cur and ids[j] == toks[-1]]
        if not nxt or len(toks) >= cap:
            break
        cur = nxt[0]
    return toks, nodes, any(t in eos for t in toks) or len0 + len(toks) >= max_length


def test_walk_restatement():
    # root 0 -> {1 -> {2, 3}, 4 -> 5}; picks walk 0 -> 1 -> 3, node 3's pick ends it
    parent = [-1, 0, 1, 1, 0, 4]
    rows = [1]
    for i in range(1, 6):
        rows.append(rows[parent[i]] | (1 << i))
    ids = [9, 11, 12, 13, 14, 15]
    picks = [11, 13, 0, 2, 0, 0]
    assert ar.walk(ids, rows, picks, eos=[2]) == ([11, 13, 2], [0, 1, 3], True)
    assert ar.walk(ids, rows, picks, eos=[]) == ([11, 13, 2], [0, 1, 3], False)
    assert ar.walk(ids, rows, picks, eos=[], len0=10, max_length=12, bound_walk=True) == ([11, 13], [0, 1], True)
    assert ar.walk(ids, rows, picks, eos=[], len0=10, max_length=13) == ([11, 13, 2], [0, 1, 3], True)
    assert ar.walk(ids[:1], rows[:1], picks[:1]) == ([11], [0], False)
    rng = np.random.default_rng(3)
    for trial in range(200):
        n = int(rng.integers(1, 129))
        parent, rows = pre_order_tree(rng, n, max_depth=int(rng.integers(1, 33)))
        ids = tree_ids(rng, parent, 1000, np.arange(3, 9))
        picks = []
        for k in range(n):
            kids = [j for j in range(1, n) if parent[j] == k]
            picks.append(ids[int(rng.choice(kids))] if kids and rng.random() < 0.8 else int(rng.integers(3, 12)))
        kw = dict(eos=[5], len0=int(rng.integers(1, 50)), max_length=60, bound_walk=bool(trial & 1))
        assert ar.walk(ids, rows, picks, **kw) == _parent_walk(ids, rows, picks, **kw)


def test_compact_restatement():
    rows = torch.arange(40).view(10, 4)
    out = ar.compact(rows, 2, [0, 2, 3, 6])
    assert out[:, 0].tolist() == [0, 4, 8, 16, 20, 32, 24, 28, 32, 36]
    assert torch.equal(ar.compact(rows, 2, [0]), rows) and torch.equal(ar.compact(rows, 2, [0, 1, 2]), rows)


def test_case_table_reaches_what_it_was_built_for():
    for L in all_launches():
        assert L.batch * L.rps <= 128
        e = expect_launch(ar.REF, L)
        for s, sl in enumerate(L.slots):
            assert len(sl.ctx) <= L.stride
            for k, w in sl.why.items():
                if k != 'route':
                    assert e.picks[s * L.rps + k] == w, (L.kind, L.V, s, k)
            if 'route' in sl.why and sl.n and not sl.fin0:
                route = sl.why['route']
                assert e.nodes[s] == route[:e.count[s]]
    assert max(sl.n for L in tree_launches() for sl in L.slots) == 128
    assert max(L.V for L in tree_launches()) == 400000            # the penalty bitmap needs > 48 KB
    w = walk_launches(1.2)
    e = [expect_launch(ar.REF, L) for L in w]
    assert e[0].nodes[0][-11:] == list(range(62, 73))               # 63 -> 64 on the accepted path
    assert e[1].count[0] == 33 == w[1].slots[0].n                   # every node accepted
    assert (w[1].V - 5 in e[1].tokens[1][:-1]) and e[1].fin[1] == 1  # EOS (the 5th id) mid-path: the walk goes on
    assert e[1].fin[0] == 0
    assert e[2].count == [0, 0, 20, len(w[2].slots[3].why['route'])] and e[2].fin == [1, 0, 1, 0]
    assert 2 in e[2].tokens[3]
    assert e[3].count[0] == 12 and e[3].seq_len[0] == 72 > w[3].stride


def test_every_mutation_changes_an_expected_output():
    rows = {('probe', p): probe_case(p) + (p,) for p in PROBE_P}
    rows.update({('tie', V, p): tie_case(V, p)[:2] + (p,) for V in TIE_V for p in (1.0, TIE_P)})
    ref_rows = {k: ar.pick_rows(ar.REF, *c) for k, c in rows.items()}
    ref_launch = [_launch_outputs(expect_launch(ar.REF, L)) for L in all_launches()]
    ref_kv = {D: expect_compact(ar.REF, D) for D in (64, 128)}
    caught = {}
    for name, f in ar.MUTATIONS.items():
        hits = [k for k, c in rows.items() if not torch.equal(ar.pick_rows(f, *c), ref_rows[k])]
        hits += [i for i, L in enumerate(all_launches()) if _launch_outputs(expect_launch(f, L)) != ref_launch[i]]
        hits += [D for D in ref_kv if not torch.equal(expect_compact(f, D), ref_kv[D])]
        caught[name] = hits
    assert all(caught.values()), {k: v for k, v in caught.items() if not v}


# ------------------------------------------------------------------------------------------------ GPU half
def run_rows(logits, ctx, p):
    """every row its own request slot (n = 1, rows_per_slot 1, 128 slots per launch, max_nodes 128) whose context is
    ctx[row]; no sync between launches.  Returns the accepted token of every row."""
    from painlessinferenceacceleration_b200.common import ops
    R, V = logits.shape
    L = ctx.shape[1]
    acc = ops.Accept(V, 128, p, [], BIG, DEV)
    lg = logits.to(DEV)
    seq = torch.zeros((R, L + 1), dtype=torch.int32, device=DEV)
    seq[:, :L] = ctx.to(DEV)
    ids = seq[:, L - 1].contiguous()
    mask = torch.zeros((128, 2), dtype=torch.int64, device=DEV)
    n = torch.ones((128,), dtype=torch.int32, device=DEV)
    seq_len = torch.full((R,), L, dtype=torch.int32, device=DEV)
    prefix = seq_len - 1
    fin = torch.zeros((R,), dtype=torch.int32, device=DEV)
    at = torch.full((R, 128), -1, dtype=torch.int32, device=DEV)
    an = torch.full((R, 128), -1, dtype=torch.int32, device=DEV)
    ac = torch.zeros((R,), dtype=torch.int32, device=DEV)
    for r0 in range(0, R, 128):
        b = min(128, R - r0)
        sl = slice(r0, r0 + b)
        acc.run(lg[sl], ids[sl], mask[:b], n[:b], seq[sl], seq_len[sl], at[sl], ac[sl], an[sl], prefix[sl], fin[sl],
                batch=b, rows_per_slot=1)
    torch.cuda.synchronize()
    assert bool((ac == 1).all()) and bool((an[:, 0] == 0).all())
    return at[:, 0].long().cpu()


@gpu
@pytest.mark.parametrize('p', PROBE_P)
def test_cuda_torch_divides_a_bf16_tensor_by_the_fp32_reciprocal(p):
    """the rule accept_ref.penalise states, measured: PyTorch's CUDA bf16 tensor / Python scalar multiplies by 1 / p
    taken in double and rounded to fp32, and so does the processor"""
    from transformers import RepetitionPenaltyLogitsProcessor
    x = finite_bf16()
    got = (x.to(DEV) / p).cpu()
    want = (x.float() * ar.reciprocal(p)).to(torch.bfloat16)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    ids = torch.arange(x.numel(), device=DEV)[None]
    got = RepetitionPenaltyLogitsProcessor(p)(ids, x.to(DEV)[None])[0].cpu()
    assert torch.equal(got.view(torch.int16), ar.penalise(x, p).view(torch.int16))


@gpu
@pytest.mark.parametrize('p', PROBE_P)
def test_penalty_bit_for_bit_over_every_bf16_score(p):
    logits, ctx = probe_case(p)
    got = run_rows(logits, ctx, p)
    bad = torch.nonzero(got).flatten()
    assert bad.numel() == 0, ('penalised x != accept_ref.penalise(x) for x =',
                              logits[bad[:8]].float().tolist())


@gpu
@pytest.mark.parametrize('p', PROBE_P)
def test_host_path_equals_device_path(p):
    """LookaheadPreTrainedModel._host_pick with transformers' processor (the loop's path for callers with logits
    processors) and pia_accept with n = 1 pick the same token from every probe row"""
    from transformers import RepetitionPenaltyLogitsProcessor
    from painlessinferenceacceleration_b200.common.pretrained_model import LookaheadPreTrainedModel
    logits, ctx = probe_case(p)
    proc = RepetitionPenaltyLogitsProcessor(penalty=p)
    lg, ids = logits.to(DEV), ctx.to(DEV)
    host = torch.argmax(proc(ids, lg), -1).cpu()          # _host_pick's body over all rows at once
    dev = run_rows(logits, ctx, p)
    assert torch.equal(host, dev)
    # _host_pick itself, row by row, where true division would pick otherwise, plus every 4096th row
    wrong = ar.pick_rows(ar.MUTATIONS['true division on the positive branch'], logits, ctx, p)
    sel = torch.nonzero(wrong).flatten().tolist()[:512] + list(range(0, logits.shape[0], 4096))
    for i in sel:
        assert LookaheadPreTrainedModel._host_pick([proc], ids[i:i + 1], lg[i:i + 1], False) == int(dev[i]), i


@gpu
@pytest.mark.parametrize('V', TIE_V)
@pytest.mark.parametrize('p', [1.0, TIE_P])
def test_first_index_argmax(V, p):
    logits, ctx, _ = tie_case(V, p)
    got = run_rows(logits, ctx, p)
    assert got.tolist() == ar.pick_rows(ar.REF, logits, ctx, p).tolist()


def _mask(L):
    m = np.zeros((L.batch * L.rps, 2), dtype=np.uint64)
    for s, sl in enumerate(L.slots):
        for k in range(sl.n):
            m[s * L.rps + k] = [sl.rows[k] & (2 ** 64 - 1), sl.rows[k] >> 64]
    return torch.from_numpy(m.view(np.int64)).to(DEV)


def run_launch(L):
    from painlessinferenceacceleration_b200.common import ops
    B, rps, V = L.batch, L.rps, L.V
    logits = torch.zeros((B * rps, V), dtype=torch.bfloat16)
    ids = torch.zeros((B * rps,), dtype=torch.int32)
    for s, sl in enumerate(L.slots):
        logits[s * rps:(s + 1) * rps] = sl.logits
        ids[s * rps:s * rps + sl.n] = torch.tensor(sl.ids, dtype=torch.int32)
    buf = torch.full((B * L.stride + 8,), -7, dtype=torch.int32, device=DEV)
    seq = buf[:B * L.stride].view(B, L.stride)
    for s, sl in enumerate(L.slots):
        seq[s, :len(sl.ctx)] = torch.tensor(sl.ctx, dtype=torch.int32)
    i32 = dict(dtype=torch.int32, device=DEV)
    seq_len = torch.tensor([len(sl.ctx) for sl in L.slots], **i32)
    prefix = seq_len - 1
    fin = torch.tensor([sl.fin0 for sl in L.slots], **i32)
    n = torch.tensor([sl.n for sl in L.slots], **i32)
    at = torch.full((B, 128), -1, **i32)
    an = torch.full((B, 128), -1, **i32)
    ac = torch.full((B,), -1, **i32)
    acc = ops.Accept(V, 128, L.p, L.eos, L.max_length, DEV, bound_walk=L.bound_walk)
    ml = None if L.device_max_length is None else torch.tensor([L.device_max_length], **i32)
    acc.run(logits.to(DEV), ids.to(DEV), _mask(L), n, seq, seq_len, at, ac, an, prefix, fin, batch=B,
            rows_per_slot=rps, max_length=ml)
    torch.cuda.synchronize()
    picks = acc.workspace[:B * rps].tolist()       # k_row_argmax's pick of every draft row
    c = ac.tolist()
    return SimpleNamespace(picks={r: picks[r] for r in range(B * rps) if r % rps < L.slots[r // rps].n}, count=c,
                           tokens=[at[s, :c[s]].tolist() for s in range(B)],
                           nodes=[an[s, :c[s]].tolist() for s in range(B)], seq=buf.cpu(), seq_len=seq_len.tolist(),
                           prefix=prefix.tolist(), fin=fin.tolist())


def _hf_picks(L):
    """the reference's loop body per draft node: the processor on update_input_ids (context + the tokens accepted
    before the node = the path's tokens), then torch.argmax, on CUDA"""
    from transformers import RepetitionPenaltyLogitsProcessor
    proc = RepetitionPenaltyLogitsProcessor(penalty=L.p) if L.p != 1.0 else None
    out = {}
    for s, sl in enumerate(L.slots):
        lg = sl.logits.to(DEV)
        for k in range(sl.n):
            path = [sl.ids[a] for a in range(1, k + 1) if (sl.rows[k] >> a) & 1]
            u = torch.tensor([sl.ctx + path], dtype=torch.long, device=DEV)
            sc = lg[k:k + 1] if proc is None else proc(u, lg[k:k + 1])
            out[s * L.rps + k] = int(torch.argmax(sc, -1)[0])
    return out


def _check_launch(L):
    got = run_launch(L)
    want = expect_launch(ar.REF, L)
    assert got.picks == want.picks
    if L.p != 1.0:
        assert got.picks == _hf_picks(L)
    assert got.count == want.count and got.tokens == want.tokens and got.nodes == want.nodes
    assert got.seq.tolist() == want.seq.tolist()          # nothing written past a slot's seq_stride
    assert got.seq_len == want.seq_len and got.prefix == want.prefix and got.fin == want.fin


@gpu
@pytest.mark.parametrize('i', range(len(tree_launches())))
def test_penalty_set_on_real_trees(i):
    _check_launch(tree_launches()[i])


@gpu
@pytest.mark.parametrize('p', [1.0, 1.2])
@pytest.mark.parametrize('i', range(4))
def test_walk(p, i):
    _check_launch(walk_launches(p)[i])


@gpu
@pytest.mark.parametrize('D', [64, 128])
def test_kv_compaction_bit_for_bit(D):
    from painlessinferenceacceleration_b200 import _lib
    from painlessinferenceacceleration_b200.common.ops import _s
    x = compact_cache(D)
    B, Lp1, H, S, _ = x.shape
    kc = x.to(DEV).view(torch.bfloat16)
    vc = torch.flip(x, [3]).to(DEV).view(torch.bfloat16)
    i32 = dict(dtype=torch.int32, device=DEV)
    nodes = torch.ones((B, 128), **i32)               # past count: entries that would move rows if they were read
    for s, (_, nd) in enumerate(COMPACT):
        nodes[s, :len(nd)] = torch.tensor(nd, dtype=torch.int32)
    count = torch.tensor([len(nd) for _, nd in COMPACT], **i32)
    prefix = torch.tensor([p + len(nd) for p, nd in COMPACT], **i32)
    lib = _lib.load()
    _lib.check(lib.pia_kv_compact(kc.data_ptr(), vc.data_ptr(), Lp1 - 1, H, S, D, B, Lp1 * H * S * D,
                                  nodes.data_ptr(), 128, count.data_ptr(), prefix.data_ptr(), _s()))
    torch.cuda.synchronize()
    assert torch.equal(kc.view(torch.int16).cpu(), expect_compact(ar.REF, D))
    want_v = torch.flip(x, [3])
    for s, (p_old, nd) in enumerate(COMPACT):
        if nd:
            for lyr in range(Lp1 - 1):
                for h in range(H):
                    want_v[s, lyr, h] = ar.compact(want_v[s, lyr, h], p_old, nd)
    assert torch.equal(vc.view(torch.int16).cpu(), want_v)


@gpu
def test_vocab_too_large_for_the_penalty_bitmap_is_refused():
    from painlessinferenceacceleration_b200.common import ops
    V = 200 * 1024 * 8 + 32            # one bitmap word past the 200 KB of dynamic shared memory
    i32 = dict(dtype=torch.int32, device=DEV)
    logits = torch.zeros((1, V), dtype=torch.bfloat16, device=DEV)
    acc = ops.Accept(V, 128, 1.2, [2], BIG, DEV)
    z = lambda *s: torch.zeros(s, **i32)  # noqa: E731
    with pytest.raises(AssertionError, match='penalty bitmap'):
        acc.run(logits, z(1), torch.zeros((1, 2), dtype=torch.int64, device=DEV), z(1) + 1, z(1, 4), z(1) + 1,
                z(1, 128), z(1), z(1, 128), z(1), z(1), batch=1, rows_per_slot=1)
