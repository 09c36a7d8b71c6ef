# -*- coding: utf-8 -*-
"""Plain-torch restatement of k_moe_router and k_moe_combine (csrc/fused_ops.cu) for the MoE tests: an fp64 reference
of the router, a comparator that tolerates only real ties, the reference's sparse combine loop, an fp32 emulation of
each kernel and the wrong kernels (mutations) the checks must reject.  Runs on any device; nothing here needs a GPU.

The reference block (mixtral/modeling_mixtral.py:716-759):
  logits = bf16(y @ gate^T)                       a bf16 Linear: fp32 accumulation, one rounding
  p = softmax(logits, fp32); top-k; w = p_sel / sum(p_sel); w = bf16(w)
  final = zeros(bf16); for e in expert order: final.index_add_(0, tokens of e, bf16(w_bf16 * ye_e))
The kernels write the weights densely ([rows, E], +0 for the experts a token did not select) and sum over all experts,
skipping those whose weight is 0."""
import itertools

import torch

from tests.norm_ref import U, bf16_rne

LANES = 32                  # k_moe_router: one warp per expert dot product
ABS = 2.0 ** -149           # fp32 subnormal spacing: the absolute error of an fp32 op in the subnormal range
BF16 = torch.bfloat16


# ------------------------------------------------------------------------------------------------ router reference
def logits64(y, gate):
    """(fp64 logits [rows, E], mass sum_i |y_i w_i|) of bf16 y [rows, H] and gate [E, H]"""
    yd, gd = y.double(), gate.double()
    return yd @ gd.t(), yd.abs() @ gd.abs().t()


def logit_depth(hidden):
    """the longest chain of fp32 additions in k_moe_router's dot product: each lane adds its 8 * ceil(H / 256)
    products serially, then 5 shuffle levels"""
    return 8 * -(-hidden // 256) - 1 + 5


def logit_budget(mass, hidden):
    """absolute bound of the fp32 dot product's error, doubled to cover cuBLAS's unknown order in the eager reference"""
    return 2.0 * logit_depth(hidden) * U * mass


def _stable_desc(p):
    """indices by decreasing p, lowest index first among equal values"""
    return torch.sort(p, dim=-1, descending=True, stable=True).indices


def softmax64(lg):
    m = lg.max(-1, keepdim=True).values
    ex = torch.exp(lg - m)
    return ex / ex.sum(-1, keepdim=True)


def router_ref(y, gate, k):
    """the fp64 reference: bf16 logits, fp64 softmax, top-k (largest first, lowest index among exactly equal logits),
    fp64 renormalisation, one bf16 rounding.  -> (dense weights [rows, E] as fp64 bf16 values, selection mask)"""
    L, _ = logits64(y, gate)
    lg = bf16_rne(L)
    p = softmax64(lg)
    order = _stable_desc(p)
    sel = torch.zeros_like(p, dtype=torch.bool).scatter_(1, order[:, :k], True)
    ps = torch.where(sel, p, torch.zeros_like(p))
    w = ps / ps.sum(-1, keepdim=True)
    return torch.where(sel, bf16_rne(w), torch.zeros_like(w)), sel


# ------------------------------------------------------------------------------------------------ router comparator
def _p_rel(lg):
    """relative error bound of the kernel's fp32 p_j = expf(l_j - max) / den, per element: the subtraction (u |d|,
    which moves exp by that much relative), expf's 2 ulp (4 u), the E - 1 additions of the denominator over the terms'
    own errors, the division (u)"""
    E = lg.shape[-1]
    d = (lg - lg.max(-1, keepdim=True).values).abs()
    ex = torch.exp(-d)
    r_ex = (4.0 + d) * U
    r_den = (ex * r_ex).sum(-1, keepdim=True) / ex.sum(-1, keepdim=True) + (E - 1) * U
    return r_ex + r_den + U


def weight_budget(lg, p, sel):
    """(relative, absolute) bound of w_e = p_e / sum_S p: p_e's own bound, the k - 1 additions of the sum over the
    selected p's bounds, the division; doubled, as norm_ref.rms_budget is, to cover eager torch's order too.  The
    absolute part covers subnormal p (expf 2 ulp, two divisions, the 1 / sum <= E amplification)"""
    E = lg.shape[-1]
    k = int(sel.sum(-1).max())
    r_p = _p_rel(lg)
    ps = torch.where(sel, p, torch.zeros_like(p))
    r_sum = (ps * r_p).sum(-1, keepdim=True) / ps.sum(-1, keepdim=True) + (k - 1) * U
    rel = 2.0 * (r_p + r_sum + U)
    return rel, 2.0 * (4.0 * E + 1.0) * ABS


def _near(p, lg, r_p, order, k):
    """whether a row's top-k set is open: some selected p and some unselected p with different logits lie within
    the doubled bound of each other (exactly equal logits give exactly equal p; the lowest index wins those)"""
    E = p.shape[-1]
    if k >= E:
        return torch.zeros(p.shape[0], dtype=torch.bool, device=p.device)
    sel = torch.zeros_like(p, dtype=torch.bool).scatter_(1, order[:, :k], True)
    tol = 2.0 * (r_p[:, :, None] + r_p[:, None, :]) * torch.maximum(p[:, :, None], p[:, None, :])
    close = (p[:, :, None] - p[:, None, :]).abs() <= tol
    pair = sel[:, :, None] & ~sel[:, None, :] & (lg[:, :, None] != lg[:, None, :]) & close
    return pair.flatten(1).any(-1)


def _weights_ok(got, lg, p, sel):
    """rows whose got equals a weight vector the selection `sel` admits: each selected weight either bf16 neighbour
    of the fp64 value within the budget, each unselected one +0 exactly"""
    rel, ab = weight_budget(lg, p, sel)
    ps = torch.where(sel, p, torch.zeros_like(p))
    w = ps / ps.sum(-1, keepdim=True)
    e = rel * w + ab
    lo, hi = bf16_rne(w - e), bf16_rne(w + e)
    g = got.double()
    pos_zero = got.view(torch.int16) == 0
    ok = torch.where(sel, (g == lo) | (g == hi), pos_zero)
    return ok.all(-1)


def _selections(p, lg, r_p, k):
    """the top-k sets a kernel may pick for one row (1-D p): fixed members, plus choices from the near-tie group at
    the k-th place; within a class of exactly equal logits the lowest indices are taken first"""
    E = p.numel()
    order = _stable_desc(p[None])[0]
    if k >= E:
        return [torch.ones(E, dtype=torch.bool, device=p.device)]
    group = torch.zeros(E, dtype=torch.bool, device=p.device)
    for b in (order[k - 1], order[k]):
        group |= (p - p[b]).abs() <= 2.0 * (r_p + r_p[b]) * torch.maximum(p, p[b])
    rank = torch.empty_like(order)
    rank[order] = torch.arange(E, device=p.device)
    fixed = (rank < k) & ~group
    need = k - int(fixed.sum())
    classes = {}
    for j in torch.nonzero(group).flatten().tolist():
        classes.setdefault(float(lg[j]), []).append(j)
    members = list(classes.values())
    out = []
    for counts in itertools.product(*[range(len(m) + 1) for m in members]):
        if sum(counts) != need:
            continue
        s = fixed.clone()
        for m, c in zip(members, counts):
            s[m[:c]] = True
        out.append(s)
    return out


def router_check(got, y, gate, k, exact=False, max_vectors=4096):
    """compare the kernel's dense weights got [rows, E] with the fp64 reference; -> dict(bad=rows outside the accepted
    set, open_logit=rows with an ambiguous logit, open_select=rows with an open top-k set, n=rows, open=the mask of
    the rows with either, needed=the mask of the rows that differ from the fp64 reference's own answer, router_ref's,
    and so needed the tie allowance).  The logit budget is a worst-case bound: on random inputs most rows have a
    logit within it of a rounding midpoint, so `open` is large there while `needed` stays small.
    exact: every partial sum of the dot products is exact in fp32 (tests' exact-logit inputs), so the logits are
    bf16_rne of the fp64 value with no ambiguity"""
    L, mass = logits64(y, gate)
    hidden = y.shape[-1]
    got = got.to(L.device)
    if exact:
        lo = hi = bf16_rne(L)
    else:
        e = logit_budget(mass, hidden)
        lo, hi = bf16_rne(L - e), bf16_rne(L + e)
    amb_logit = lo != hi
    lg = bf16_rne(L)
    p = softmax64(lg)
    r_p = _p_rel(lg)
    order = _stable_desc(p)
    open_sel = _near(p, lg, r_p, order, k)
    sel = torch.zeros_like(p, dtype=torch.bool).scatter_(1, order[:, :k], True)
    ok = _weights_ok(got, lg, p, sel)
    hard = amb_logit.any(-1) | open_sel
    for t in torch.nonzero(hard & ~ok).flatten().tolist():
        ok[t] = _row_ok(got[t], lg[t], lo[t], hi[t], k, max_vectors)
    ps = torch.where(sel, p, torch.zeros_like(p))
    principal = torch.where(sel, bf16_rne(ps / ps.sum(-1, keepdim=True)), torch.zeros_like(p))
    return dict(bad=int((~ok).sum()), open_logit=int(amb_logit.any(-1).sum()), open_select=int(open_sel.sum()),
                n=got.shape[0], open=hard, needed=~(got.double() == principal).all(-1))


def _row_ok(g, lg, lo, hi, k, max_vectors):
    """one row through every admissible logit vector and every admissible top-k set of it"""
    amb = torch.nonzero(lo != hi).flatten().tolist()
    assert 2 ** len(amb) <= max_vectors, f'{len(amb)} ambiguous logits in one row'
    for bits in itertools.product((0, 1), repeat=len(amb)):
        v = lg.clone()
        for j, b in zip(amb, bits):
            v[j] = hi[j] if b else lo[j]
        p = softmax64(v[None])[0]
        r_p = _p_rel(v[None])[0]
        for s in _selections(p, v, r_p, k):
            if bool(_weights_ok(g[None], v[None], p[None], s[None])[0]):
                return True
    return False


# ------------------------------------------------------------------------------------------------ router emulation
def emulate_logits(y, gate, mut=None):
    """k_moe_router's fp32 dot products in its order: lane l sums vectors l, l + 32, ... (8 products each) serially,
    then an xor-shuffle butterfly; one bf16 rounding (none under the mutation 'fp32_logits').  The products of bf16
    values are exact in fp32, so a fused multiply-add rounds the same"""
    rows, H = y.shape
    E = gate.shape[0]
    c = -(-H // (LANES * 8))
    yp = torch.zeros((rows, c * LANES * 8))
    gp = torch.zeros((E, c * LANES * 8))
    yp[:, :H], gp[:, :H] = y.float(), gate.float()
    yv = yp.view(rows, 1, c, LANES, 8)
    gv = gp.view(1, E, c, LANES, 8)
    acc = torch.zeros((rows, E, LANES))
    for v in range(c):
        for j in range(8):
            acc = acc + yv[:, :, v, :, j] * gv[:, :, v, :, j]
    idx = torch.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, :, idx ^ o]
    lg = acc[:, :, 0]
    return lg if mut == 'fp32_logits' else lg.to(BF16).float()


def _bf(t):
    return t.to(BF16).float()


def emulate_router(y, gate, k, mut=None, fp32_weights=False):
    """k_moe_router in fp32 on the CPU -> dense bf16 weights [rows, E] (or, fp32_weights, the renormalised fp32 weights
    before the cast).  mut: a name of ROUTER_MUTATIONS"""
    lg = emulate_logits(y, gate, mut)
    rows, E = lg.shape
    mx = lg.max(-1, keepdim=True).values
    ex = torch.exp(lg - mx)
    if mut == 'bf16_exp':
        ex = _bf(ex)
    den = torch.zeros((rows,))
    for e in range(E):
        den = den + ex[:, e]
    p = ex / den[:, None]
    if mut == 'prob_bf16':
        p = _bf(p)
    chosen = torch.zeros((rows, E), dtype=torch.bool)
    s = torch.zeros((rows,))
    rank = torch.arange(E, 0, -1) if mut != 'highest_index_wins_ties' else torch.arange(1, E + 1)
    for _ in range(k - 1 if mut == 'top_k_minus_1' else k):
        q = -p if mut == 'smallest_k' else p
        q = torch.where(chosen, torch.full_like(q, -float('inf')), q)
        m = q.max(-1, keepdim=True).values
        best = ((q == m) * rank).argmax(-1)
        chosen[torch.arange(rows), best] = True
        s = s + p[torch.arange(rows), best]
    w = p if mut == 'no_renormalisation' else p / s[:, None]
    w = torch.where(chosen, w, torch.zeros_like(w))
    if fp32_weights:
        return w
    if mut == 'truncate_weights':
        return (w.view(torch.int32) & ~0xFFFF).view(torch.float32).to(BF16)
    return w.to(BF16)


ROUTER_MUTATIONS = ('no_renormalisation', 'prob_bf16', 'highest_index_wins_ties', 'smallest_k', 'fp32_logits',
                    'bf16_exp', 'truncate_weights', 'top_k_minus_1')


# ------------------------------------------------------------------------------------------------ combine
def combine_ref(ye, dense):
    """the reference's sparse loop (mixtral/modeling_mixtral.py:729-757) on dense weights [rows, E]: final = zeros
    (bf16); for each expert in index order, only the tokens that selected it (weight != 0):
    final.index_add_(0, tok, bf16(w_bf16 * ye[e, tok])).  Runs with the device's own index_add_"""
    E, _, H = ye.shape
    rows = dense.shape[0]
    final = torch.zeros((rows, H), dtype=BF16, device=ye.device)
    for e in range(E):
        tok = torch.nonzero(dense[:, e] != 0).flatten()
        if tok.numel() == 0:
            continue
        final.index_add_(0, tok, dense[tok, e, None] * ye[e, tok])
    return final


def combine_transformers(ye, w32):
    """transformers 5.5's MixtralExperts: the same loop with the fp32 routing weights, bf16(ye * w_fp32): one rounding
    fewer than the reference.  Used only to show that the two formulas differ"""
    E, _, H = ye.shape
    rows = w32.shape[0]
    final = torch.zeros((rows, H), dtype=BF16, device=ye.device)
    for e in range(E):
        tok = torch.nonzero(w32[:, e] != 0).flatten()
        if tok.numel() == 0:
            continue
        final.index_add_(0, tok, (ye[e, tok] * w32[tok, e, None]).to(BF16))
    return final


def emulate_combine(ye, dense, mut=None):
    """k_moe_combine densely over all experts: acc = +0; for e in index order, skipping w == 0:
    acc = bf16(acc + bf16(ye[e] * w)).  mut: a name of COMBINE_MUTATIONS"""
    E = ye.shape[0]
    rows = dense.shape[0]
    y = ye[:, :rows].float()
    w = dense.float()
    acc = torch.zeros(y.shape[1:], device=ye.device)
    experts = range(E - 1, -1, -1) if mut == 'reverse_order' else range(E)
    if mut == 'weight_after_sum':   # the selected outputs summed first, the sum scaled once by the total weight
        for e in experts:
            acc = torch.where(w[:, e:e + 1] != 0, _bf(acc + y[e]), acc)
        return (acc * w.sum(-1, keepdim=True)).to(BF16)
    for e in experts:
        we = w[:, e:e + 1]
        prod = y[e] * we if mut == 'product_unrounded' else _bf(y[e] * we)
        s = acc + prod if mut == 'fp32_accumulate' else _bf(acc + prod)
        acc = s if mut == 'no_zero_skip' else torch.where(we != 0, s, acc)
    return acc.to(BF16)


COMBINE_MUTATIONS = ('reverse_order', 'fp32_accumulate', 'product_unrounded', 'weight_after_sum', 'no_zero_skip')


# ------------------------------------------------------------------------------------------------ test inputs
def exact_router_inputs(rows, hidden, E, seed, device='cpu'):
    """(y, gate) bf16 whose dot products are exact in fp32 in any order: y in {-1, 0, 1}, gate entries multiples of
    2^-5 (sparse, |w| <= 1/4, plus two reserved columns of +-64 and +-45), so every partial sum is a multiple of 2^-5
    below 2^19.  By construction:
      * gate rows 1 and E - 1 are equal (E >= 3), and so are 2 and E - 2 (E >= 5): exactly equal logits in every row;
      * rows t % 6 == 0 are all zero: every logit 0;
      * rows t % 6 == 1 see column H - 1 (gate +64 for expert 0, -64 for the others): expert 0 dominates by >= 120, the
        others' weights underflow to 0;
      * rows t % 6 == 2 see column H - 1 negated and nothing else: expert 0 is 128 below the others, all equal;
      * rows t % 6 == 3 see column H - 2 (+45 / -45) and nothing else: a gap of 90, where fp32 exp is subnormal and the
        second weight a bf16 subnormal;
      * the other rows are random, with negative and zero logits.
    The reserved columns are the last two, so a kernel that drops the width tail past the 256-lane stride loses them"""
    g = torch.Generator().manual_seed(seed)
    gate = torch.zeros((E, hidden))
    free = max(hidden - 2, 0)
    nnz = min(free, 24)
    for e in range(E):
        cols = torch.randperm(free, generator=g)[:nnz]
        gate[e, cols] = torch.randint(-8, 9, (nnz,), generator=g).float() * 2.0 ** -5
    gate[:, hidden - 1] = -64.0
    gate[0, hidden - 1] = 64.0
    gate[:, hidden - 2] = -45.0
    gate[0, hidden - 2] = 45.0
    if E >= 3:
        gate[E - 1] = gate[1]
    if E >= 5:
        gate[E - 2] = gate[2]
    y = torch.randint(-1, 2, (rows, hidden), generator=g).float()
    y[:, hidden - 2:] = 0
    kind = torch.arange(rows) % 6
    y[kind == 0] = 0
    y[kind == 1, hidden - 1] = 1
    y[kind == 2] = 0
    y[kind == 2, hidden - 1] = -1
    y[kind == 3] = 0
    y[kind == 3, hidden - 2] = 1
    return y.to(BF16).to(device), gate.to(BF16).to(device)


def random_router_inputs(rows, hidden, E, seed, std=0.02, device='cpu'):
    """(y, gate) bf16: y ~ N(0, 1), gate ~ N(0, std^2), Mixtral-like logits of a few units"""
    g = torch.Generator().manual_seed(seed)
    y = torch.randn((rows, hidden), generator=g)
    gate = torch.randn((E, hidden), generator=g) * std
    return y.to(BF16).to(device), gate.to(BF16).to(device)


def expert_outputs(E, rows_cap, hidden, seed, device='cpu'):
    """ye [E, rows_cap, hidden] bf16 ~ N(0, 1) with a spread of magnitudes (x 2^-20 .. 2^12 per row) so that the
    rounding of the products and the order of the sum show"""
    g = torch.Generator().manual_seed(seed)
    ye = torch.randn((E, rows_cap, hidden), generator=g)
    ye = ye * torch.exp2(torch.randint(-20, 13, (E, rows_cap, 1), generator=g).float())
    return ye.to(BF16).to(device)
