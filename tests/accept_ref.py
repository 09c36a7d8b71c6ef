# -*- coding: utf-8 -*-
"""Plain restatement of the accept step (csrc/accept.cu: k_row_argmax, k_accept_walk, k_kv_compact) for the accept
tests, written from the reference's loop rather than from the kernels (pretrained_model.py:806-860, 894-907 and
transformers' RepetitionPenaltyLogitsProcessor), plus the wrong kernels (mutations) the checks must reject.  Runs on
any device; nothing here needs a GPU."""
from types import SimpleNamespace

import torch

BIG = 1 << 30


# ------------------------------------------------------------------------------------------------ one row
def reciprocal(p):
    """the fp32 factor PyTorch's CUDA true division of a tensor by the Python scalar p multiplies by
    (div_true_kernel_cuda): 1 / p taken in double, rounded once to fp32 - not 1 / fl32(p), which differs at p = 1.92"""
    return torch.tensor(1.0 / p, dtype=torch.float32)


def penalise(x, p):
    """RepetitionPenaltyLogitsProcessor on CUDA bf16 scores: score * p below zero, else score / p, which PyTorch
    computes as score * reciprocal(p).  So bf16(fl32(x) * fl32(p)) for x < 0, else bf16(fl32(x) * reciprocal(p)).
    x: bf16 tensor, p: the Python float the processor holds."""
    xf = x.float()
    return torch.where(xf < 0, xf * torch.tensor(p, dtype=torch.float32), xf * reciprocal(p)).to(torch.bfloat16)


def argmax(x):
    """torch.argmax over the last dim: the first maximal index; NaN is greater than everything (the first NaN wins);
    a row of -inf gives 0"""
    x = x.float()
    nan = torch.isnan(x)
    m = torch.where(nan, float('-inf'), x).amax(-1, keepdim=True)
    hit = torch.where(nan.any(-1, keepdim=True), nan, x == m)
    idx = torch.arange(x.shape[-1]).expand_as(x)
    return torch.where(hit, idx, x.shape[-1]).amin(-1)


def penalty_tokens(ctx, ids, rows, k):
    """the token set draft node k's scores are penalised on: update_input_ids of the reference's loop = the context
    (left pads and duplicates included; its last token is the root's) + the tokens accepted before node k, i.e. the
    tokens of nodes 1..k that are ancestors of node k or node k itself (bit a of rows[k]).  Siblings and descendants
    are not in it."""
    return list(ctx) + [ids[a] for a in range(1, k + 1) if (rows[k] >> a) & 1]


def pick(f, logits, tokens, p):
    """one row's (penalised) arg-max: logits [V] bf16, tokens the penalised set (each token once, however often it
    appears)"""
    x = logits.clone()
    if p != 1.0 and len(tokens):
        t = torch.tensor(sorted(set(tokens)), dtype=torch.long)
        x[t] = f.penalise(x[t], p)
    return int(f.argmax(x))


def pick_rows(f, logits, ctx, p):
    """pick() for many rows at once: logits [R, V] bf16, ctx [R, L] long (a row's set padded with its own duplicates)"""
    x = logits.clone()
    if p != 1.0:
        x.scatter_(1, ctx, f.penalise(x.gather(1, ctx), p))
    return f.argmax(x)


# ------------------------------------------------------------------------------------------------ the walk
def walk(ids, rows, row_tok, eos=(), len0=0, max_length=BIG, bound_walk=False):
    """the reference's accept loop (pretrained_model.py:806-860) over a draft of n = len(ids) nodes in DFS pre-order
    (node 0 = the root, the context's last token); rows[j] has bit a set for every ancestor a of node j and for j;
    row_tok[j] is node j's pick.  bound_walk: the batched loop never accepts past max_length - len0
    (pretrained_model_batch.py:862).  Returns (accepted tokens, their logit indices = draft nodes, finished)."""
    cap = max_length - len0 if bound_walk else BIG
    return _walk(ids, rows, row_tok, eos, len0, max_length, cap)


def _walk(ids, rows, row_tok, eos, len0, max_length, cap):
    n = len(ids)
    toks, nodes = [], []
    if n == 1:                                   # no draft (:783-798)
        toks, nodes = [row_tok[0]], [0]
    else:
        # draft_masks = masks[1:, 1:]; a row is a leaf when the next row is not deeper (:806-820)
        paths = [[a for a in range(1, n) if (rows[j] >> a) & 1] for j in range(1, n)]
        depth = [len(q) for q in paths]
        leaves = [i - 1 for i in range(1, len(depth)) if depth[i] <= depth[i - 1]] + [len(depth) - 1]
        branches = [paths[i] for i in leaves]
        for i in range(-1, max(depth)):
            node = 0 if i == -1 else branches[0][i]
            t = row_tok[node]
            toks.append(t)
            nodes.append(node)
            if i == max(depth) - 1 or len(toks) >= cap:
                break
            branches = [b for b in branches if len(b) > i + 1 and ids[b[i + 1]] == t]
            if not branches:
                break
    fin = any(t in eos for t in toks) or len0 + len(toks) >= max_length   # :1225-1231
    return toks, nodes, fin


# ------------------------------------------------------------------------------------------------ the cache
def compact(rows, p_old, nodes):
    """KV rows of one (layer, head) after the accept step: rows [S, D]; the root sits at row p_old, draft node j at
    p_old + j.  The reference keeps concat(rows[:ctx], rows[kv_idx]) (:904-905) with ctx = p_old + 1 and
    kv_idx = p_old + nodes[1:]; every row past that is left as it was."""
    out = rows.clone()
    kept = torch.cat([rows[:p_old + 1], rows[[p_old + j for j in nodes[1:]]]], 0)
    out[:kept.shape[0]] = kept
    return out


# ------------------------------------------------------------------------------------------------ wrong kernels
def _pen_true_division(x, p):
    xf, pf = x.float(), torch.tensor(p, dtype=torch.float32)
    return torch.where(xf < 0, xf * pf, xf / pf).to(torch.bfloat16)


def _pen_single_reciprocal(x, p):
    xf, pf = x.float(), torch.tensor(p, dtype=torch.float32)
    return torch.where(xf < 0, xf * pf, xf * (torch.tensor(1.0) / pf)).to(torch.bfloat16)


def _pen_signs_swapped(x, p):
    xf = x.float()
    return torch.where(xf < 0, xf * reciprocal(p), xf * torch.tensor(p, dtype=torch.float32)).to(torch.bfloat16)


def _argmax_last(x):
    x = x.float()
    nan = torch.isnan(x)
    m = torch.where(nan, float('-inf'), x).amax(-1, keepdim=True)
    hit = torch.where(nan.any(-1, keepdim=True), nan, x == m)
    return torch.where(hit, torch.arange(x.shape[-1]).expand_as(x), -1).amax(-1)


def _argmax_nan_ignored(x):
    x = x.float()
    m = torch.where(torch.isnan(x), float('-inf'), x).amax(-1, keepdim=True)
    i = torch.where(x == m, torch.arange(x.shape[-1]).expand_as(x), x.shape[-1]).amin(-1)
    return torch.where(m[..., 0] == float('-inf'), 0, i)


def _own_token_left_out(ctx, ids, rows, k):
    return list(ctx) + [ids[a] for a in range(1, k) if (rows[k] >> a) & 1]


def _every_draft_token(ctx, ids, rows, k):
    return list(ctx) + list(ids[1:])


def _walk_parent_word0(ids, rows, row_tok, eos=(), len0=0, max_length=BIG, bound_walk=False):
    # a parent search that only reads mask word 0: node j >= 64 takes its deepest ancestor below 64 as its parent
    def parent(j):
        m = rows[j] & (((1 << min(j, 64)) - 1))
        return m.bit_length() - 1
    cap = max_length - len0 if bound_walk else BIG
    cur, toks, nodes = 0, [], []
    while True:
        toks.append(row_tok[cur])
        nodes.append(cur)
        nxt = [j for j in range(1, len(ids)) if parent(j) == cur and ids[j] == toks[-1]]
        if not nxt or len(toks) >= len(ids) or len(toks) >= cap:
            break
        cur = nxt[0]
    return toks, nodes, any(t in eos for t in toks) or len0 + len(toks) >= max_length


def _walk_stops_at_eos(ids, rows, row_tok, eos=(), len0=0, max_length=BIG, bound_walk=False):
    toks, nodes, fin = walk(ids, rows, row_tok, eos, len0, max_length, bound_walk)
    c = next((i + 1 for i, t in enumerate(toks) if t in eos), len(toks))
    return toks[:c], nodes[:c], fin


def _walk_bound_off_by_one(ids, rows, row_tok, eos=(), len0=0, max_length=BIG, bound_walk=False):
    return _walk(ids, rows, row_tok, eos, len0, max_length, max_length - len0 + 1 if bound_walk else BIG)


def _compact_descending(rows, p_old, nodes):
    out = rows.clone()
    for k in range(len(nodes) - 1, 0, -1):
        out[p_old + k] = out[p_old + nodes[k]]
    return out


def _compact_reads_k(rows, p_old, nodes):
    out = rows.clone()
    for k in range(1, len(nodes)):
        out[p_old + k] = out[p_old + k]
    return out


REF = SimpleNamespace(penalise=penalise, argmax=argmax, penalty_tokens=penalty_tokens, walk=walk, compact=compact)

MUTATIONS = {name: SimpleNamespace(**dict(vars(REF), **over)) for name, over in {
    'true division on the positive branch': dict(penalise=_pen_true_division),
    'reciprocal of the fp32 penalty': dict(penalise=_pen_single_reciprocal),
    'last index wins a tie': dict(argmax=_argmax_last),
    'NaN ignored': dict(argmax=_argmax_nan_ignored),
    'sign branches swapped': dict(penalise=_pen_signs_swapped),
    "node k's own token not penalised": dict(penalty_tokens=_own_token_left_out),
    'every draft token penalised': dict(penalty_tokens=_every_draft_token),
    'parent searched in mask word 0 only': dict(walk=_walk_parent_word0),
    'walk stops at the first EOS': dict(walk=_walk_stops_at_eos),
    'bound_walk cap off by one': dict(walk=_walk_bound_off_by_one),
    'compaction in descending k': dict(compact=_compact_descending),
    'compaction reads p_old + k': dict(compact=_compact_reads_k),
}.items()}
