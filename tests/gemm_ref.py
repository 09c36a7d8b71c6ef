# -*- coding: utf-8 -*-
"""Plain-torch restatement of the weight-streaming GEMMs (csrc/gemm_ws.cu: k_gemm_ws, k_gemm_stream, k_gemm_sk,
k_gemm_fp8, k_gemm_w4) for the GEMM tests: the plan rules of pia_gemm_plan_create* and pia_gemm_run down to the kernel
instance launched, exact-integer operands (int4: codes, zero points and power-of-two scales whose dequantised weight
is exact), an fp64 reference with a scale-aware comparator, the one-hot routing probe, an fp32 emulation of the
kernels' summation order and the wrong kernels (mutations) the checks must reject.  Runs on any device; nothing here
needs a GPU."""
from collections import namedtuple

import torch

BMW, TOK = 128, 64          # weight rows per CTA tile, token rows per CTA
MASS_LIMIT = 2 ** 11        # exact-integer operands keep sum_k |x_k| |w_k| below this


def _ceil(a, b):
    return (a + b - 1) // b


# ------------------------------------------------------------------------------------------------ plan rules
# kind: 'ws' (k_gemm_ws), 'stream' (k_gemm_stream), 'sk' (k_gemm_sk, stream-K), 'fp8' (k_gemm_fp8), 'w4' (k_gemm_w4).
# bk: k per pipeline stage (chunk).  cps / n_split: chunks per split and splits; cluster: 0 or the cluster size (the
# splits of a tile reduce on chip); nstage: the kernel instance's stage count; sk_grid: stream-K CTAs; wg: consumer
# warpgroups (64-row slices) per k_gemm_stream tile; tiled: the bf16 weight's HBM layout; group / f16: the int4 scale
# group (k per scale) and scale dtype.
Plan = namedtuple('Plan', 'kind N K bk n_chunks cps n_split cluster nstage groups tiles sk_grid wg tiled group f16')
W4_BK = 256                 # k per k_gemm_w4 stage: 128 bytes of codes per weight row


def _split(n_chunks, split_k, want_cluster):
    split = min(max(want_cluster or split_k, 1), n_chunks)
    cps = _ceil(n_chunks, split)
    n_split = _ceil(n_chunks, cps)
    if want_cluster and n_split != want_cluster:
        raise ValueError(f'{n_chunks} chunks are too short for {want_cluster} cluster splits')
    return cps, n_split


def plan(N, K, split_k=1, tiled=False, fp8=False, groups=1, bias=False, n_sm=132, silu=False, w4=False, group=128,
         f16=False):
    """what pia_gemm_plan_create / _grouped / _create_fp8 / _grouped_fp8 / _create_w4 / _grouped_w4 (+ set_silu)
    choose on a device with n_sm SMs, and which kernel pia_gemm_run launches; raises ValueError where the library
    refuses the plan"""
    want_cluster = -split_k if split_k in (-2, -4, -8) else 0
    if w4:
        if N % BMW or K % 128:
            raise ValueError('the int4 GEMM needs N % 128 == 0 and K % 128 == 0')
        if group <= 0 or group % 128 or K % group:
            raise ValueError(f'group size {group}: a multiple of 128 that divides K = {K}')
        if split_k < 1 and not want_cluster:
            raise ValueError('int4 plans take split_k >= 1 or a cluster split')
        if groups > 1 and (split_k != 1 or bias):
            raise ValueError('a grouped int4 plan has one K split and no bias')
        n_chunks = _ceil(K, W4_BK)
        cps, n_split = _split(n_chunks, split_k, want_cluster)
        if bias and n_split > 1 and not want_cluster:
            raise ValueError('a bias needs split_k == 1 or a cluster split')
        if silu and (groups > 1 or n_split > 1 or bias):
            raise ValueError('the SiLU*up epilogue needs one group, split_k == 1 and no bias')
        tiles = N // BMW
        nstage = 4 if tiles * n_split * groups <= n_sm else 2
        return Plan('w4', N, K, W4_BK, n_chunks, cps, n_split, want_cluster, nstage, groups, tiles, 0, 0, True,
                    group, bool(f16))
    if fp8:
        if N % BMW or K % 128:
            raise ValueError('the fp8 GEMM needs N % 128 == 0 and K % 128 == 0')
        if split_k < 1 and not want_cluster:
            raise ValueError('fp8 plans take split_k >= 1 or a cluster split')
        if groups > 1 and split_k != 1:
            raise ValueError('a grouped fp8 plan has one K split')
        n_chunks = K // 128
        cps, n_split = _split(n_chunks, split_k, want_cluster)
        if bias and n_split > 1 and not want_cluster:
            raise ValueError('a bias needs split_k == 1 or a cluster split')
        tiles = N // BMW
        nstage = 6 if tiles * n_split * groups <= n_sm else 3
        return Plan('fp8', N, K, 128, n_chunks, cps, n_split, want_cluster, nstage, groups, tiles, 0, 0, True, 0,
                    False)
    if K % 64:
        raise ValueError('K must be a multiple of 64')
    n_chunks = K // 64
    if groups > 1:
        if N % BMW:
            raise ValueError('grouped GEMM needs N % 128 == 0')
        tiles = N // BMW
        return Plan('ws', N, K, 64, n_chunks, n_chunks, 1, 0, 8 if tiles * groups <= n_sm else 4, groups, tiles, 0,
                    0, False, 0, False)
    if split_k < -1 and not want_cluster:
        raise ValueError('cluster split-K supports 2, 4 or 8 CTAs')
    cps, n_split = _split(n_chunks, split_k, want_cluster)
    if tiled and N % BMW:
        raise ValueError('a tiled weight needs N % 128 == 0')
    tiles = _ceil(N, BMW)
    nstage = 8 if tiles * n_split <= n_sm else 4
    if split_k == -1:
        if not tiled:
            raise ValueError('stream-K needs the tiled weight layout')
        units = (N // BMW) * n_chunks
        return Plan('sk', N, K, 64, n_chunks, n_chunks, 1, 0, 8, 1, N // BMW, min(units, n_sm), 0, True, 0, False)
    if silu and (n_split > 1 or N % BMW):
        raise ValueError('the SiLU*up epilogue needs split_k == 1 and N % 128 == 0')
    if n_split == 1 and not want_cluster and not silu:
        # k_gemm_stream: 64-row tiles while they fit in one wave at 3 CTAs per SM, else 128-row tiles; 4 stages
        wg = 1 if _ceil(N, 64) <= 3 * n_sm else 2
        return Plan('stream', N, K, 64, n_chunks, cps, 1, 0, 4, 1, _ceil(N, 64 * wg), 0, wg, bool(tiled), 0, False)
    return Plan('ws', N, K, 64, n_chunks, cps, n_split, want_cluster, nstage, 1, tiles, 0, 0, bool(tiled), 0, False)


def instance(p):
    """the kernel template instance pia_gemm_run launches for plan p, spelled as in csrc/gemm_ws.cu without spaces
    and with every template argument given"""
    if p.kind == 'sk':
        return 'k_gemm_sk'
    if p.kind == 'stream':
        return f'k_gemm_stream<{p.wg},{p.nstage}>'
    if p.kind == 'w4':
        return f'k_gemm_w4<{p.nstage},{str(p.f16).lower()},{str(p.groups > 1).lower()}>'
    return f'k_gemm_{p.kind}<{p.nstage}>'


def splits_reported(p):
    """pia_gemm_plan_splits: 1 for a cluster (bf16 output) or stream-K plan, else the fp32 slice count"""
    return 1 if p.cluster else p.n_split


def split_ranges(p):
    """[(c0, c1)] chunk range of every K split, as the kernels clip the last one"""
    return [(s * p.cps, min((s + 1) * p.cps, p.n_chunks)) for s in range(p.n_split)]


# stream-K partition (k_gemm_sk): (tile, chunk) units cut into G contiguous ranges [sk_begin(b), sk_begin(b + 1))
def sk_begin(b, U, G):
    return b * U // G


def sk_cta_of(x, U, G):
    b = x * G // U
    while b + 1 < G and sk_begin(b + 1, U, G) <= x:
        b += 1
    while b > 0 and sk_begin(b, U, G) > x:
        b -= 1
    return b


def sk_segments(tile, n_chunks, U, G):
    """[(cta, c0, c1)]: the chunk ranges of one tile in CTA order; the first CTA owns the tile, the others fill
    contributor slots 0, 1, ... in that order"""
    ts, segs = tile * n_chunks, []
    for b in range(sk_cta_of(ts, U, G), sk_cta_of(ts + n_chunks - 1, U, G) + 1):
        lo, hi = max(sk_begin(b, U, G), ts), min(sk_begin(b + 1, U, G), ts + n_chunks)
        segs.append((b, lo - ts, hi - ts))
    return segs


def sk_slots_old(n_tiles, n_chunks, G):
    """the fix-up slot count the plan used to allocate: ceil(n_chunks / ceil(U / G)) + 1"""
    per = _ceil(n_tiles * n_chunks, G)
    return _ceil(n_chunks, per) + 1


def sk_slots_needed(n_tiles, n_chunks, G):
    """contributor slots the kernel writes: the most CTAs after a tile's owner that hold some of its chunks"""
    U = n_tiles * n_chunks
    return max([1] + [sk_cta_of(t * n_chunks + n_chunks - 1, U, G) - sk_cta_of(t * n_chunks, U, G)
                      for t in range(n_tiles)])


# ------------------------------------------------------------------------------------------------ operands
def exact_operands(rows, N, K, gen, groups=1, fp8=False, bias=False, device='cpu'):
    """integer operands whose every partial sum is exact: x [rows, groups * K] bf16 with |x| <= 3 on a random support
    of at most 160 columns per row and group, w [groups, N, K] with |w| <= 4 (bf16, or e4m3 codes for fp8), so that
    sum_k |x_k| |w_k| <= 160 * 12 < 2^11.  Then every partial sum, in any order and in any accumulator of at least 12
    bits, is an exact integer, and the kernel's output must be bf16_rne(exact) bit for bit.  Even rows of x and rows
    n % 4 < 2 of w are non-negative, so that about a quarter of the outputs exceed 256 and their bf16 rounding is not
    trivial.  fp8: scale [groups * N] powers of two 2^-2 .. 2^2 varying from row to row (the product stays exact),
    bias [N] integers in [-64, 64] or None.  Returns (x, w, scale, bias); w is float8_e4m3fn for fp8, scale / bias None
    for bf16."""
    x = torch.zeros((rows, groups * K))
    support = min(K, 160)
    for g in range(groups):
        for t in range(rows):
            cols = torch.randperm(K, generator=gen)[:support] + g * K
            lo = 1 if t % 2 == 0 else -3
            x[t, cols] = torch.randint(lo, 4, (support,), generator=gen).float()
    w = torch.randint(-4, 5, (groups, N, K), generator=gen).float()
    pos = (torch.arange(N) % 4) < 2
    w[:, pos] = w[:, pos].abs()
    scale = b = None
    if fp8:
        scale = torch.pow(2.0, (torch.randint(0, 5, (groups * N,), generator=gen) - 2).float())
        scale[1::2] = torch.where(scale[1::2] == scale[0::2], scale[1::2] * 2, scale[1::2])  # n and n ^ 1 differ
        if bias:
            b = torch.randint(-64, 65, (N,), generator=gen).float()
        wq = w.to(torch.float8_e4m3fn)
        assert torch.equal(wq.float(), w)
        w = wq
    else:
        w = w.to(torch.bfloat16)
    x = x.to(torch.bfloat16)
    for g in range(groups):
        mass = x[:, g * K:(g + 1) * K].double().abs() @ w[g].double().abs().t()
        assert float(mass.max()) < MASS_LIMIT
    mv = lambda t: None if t is None else t.to(device)  # noqa: E731
    return mv(x), mv(w), mv(scale), mv(b)


W4 = namedtuple('W4', 'u s z group')   # int4 weights: codes u [G, N, K], scales s [G, N, K / group], zero points z


def dequant_w4(q, mut=None):
    """the weight k_gemm_w4 multiplies with, bf16 [G, N, K]: W[n, k] = bf16(dtype_s(s[g, n] * (u[n, k] - z[g, n]))),
    g = the scale group of k's 128-k half; u - z is exact in the scale's dtype, the product rounds once to it.  mut: a
    key of MUTATIONS that changes which scale a weight takes or how the product rounds."""
    u, s, z, gs = q
    G, N, K = u.shape
    k = torch.arange(K, device=u.device)
    gi = (k // 128) * 128 // gs
    if mut == "a half takes its chunk's first group's scale and zero point":
        gi = (k // W4_BK) * W4_BK // gs
    if mut == 'rows r and r + 8 swap scales':
        s = s[:, torch.arange(N, device=u.device) ^ 8]
    if mut == "a grouped plan reads expert 0's table columns":
        s, z = s[:1].expand_as(s), z[:1].expand_as(z)
    d = u.to(s.dtype) - z[:, :, gi].to(s.dtype)
    if mut == 'the fp16 product is not rounded to fp16 before bf16':
        return (d.float() * s[:, :, gi].float()).to(torch.bfloat16)
    return (d * s[:, :, gi]).to(torch.bfloat16)


def dense(w):
    """the bf16 / e4m3 / float weight [G, N, K] a plan multiplies with: int4 codes dequantised"""
    return dequant_w4(w) if isinstance(w, W4) else w


def exact_operands_w4(rows, N, K, group, gen, groups=1, f16=False, bias=False, device='cpu'):
    """int4 exact-integer operands: x as exact_operands gives it, codes u 0..15, zero points covering 0..16 and
    power-of-two scales 2^-4 .. 2^-2 that differ between adjacent scale groups and between rows n, n ^ 1 and n ^ 8,
    so that the dequantised weight is s (u - z) exactly (|W| <= 4 on a 2^-4 grid, in bf16 and fp16 alike) and
    sum_k |x_k| |W_k| < MASS_LIMIT: every partial sum is exact in fp32 and the output is bf16_rne(exact).  Rows
    n % 4 < 2 have u >= z.  fp16: rows n % 16 == 5 take the 11-bit scale 2^e (1 + 3 * 2^-10) and u - z in {0, 3}, whose
    product rounds to fp16 on a tie and then to bf16 on a tie: W = 3 * 2^e exactly, but 3 * 2^e (1 + 2^-6) when the
    product goes straight to bf16.  Returns (x, W4(u, s, z, group), None, bias)."""
    x, _, _, _ = exact_operands(rows, N, K, gen, groups=groups)
    ng = K // group
    n = torch.arange(N)[:, None]
    j = torch.arange(ng)[None, :]
    r16 = torch.randint(0, 3, (groups, N // 16 + 1, 1), generator=gen)[:, n.squeeze(1) // 16]
    e = -4 + ((n & 1) + 2 * ((n >> 3) & 1) + j + r16) % 3                         # [groups, N, ng]
    z = torch.randint(0, 17, (groups, N, ng), generator=gen)
    pos = (torch.arange(N) % 4) < 2
    z[:, pos] = torch.randint(0, 9, z[:, pos].shape, generator=gen)
    zn = z[0, ~pos].reshape(-1)
    zn[:17] = torch.arange(17)                                                    # every zero point appears
    z[0, ~pos] = zn.view(-1, ng)
    zk = z.repeat_interleave(group, 2)
    u = torch.randint(0, 16, (groups, N, K), generator=gen)
    lo = torch.rand((groups, N, K), generator=gen)
    u[:, pos] = (zk[:, pos] + (lo[:, pos] * (16 - zk[:, pos])).long()).clamp_max(15)   # u >= z where z <= 15
    sdt = torch.float16 if f16 else torch.bfloat16
    s = torch.pow(2.0, e.double())
    if f16:
        odd = (torch.arange(N) % 16) == 5
        s[:, odd] *= 1 + 3 * 2.0 ** -10
        zo = torch.randint(0, 13, z[:, odd].shape, generator=gen)
        z[:, odd] = zo
        u[:, odd] = zo.repeat_interleave(group, 2) + 3 * torch.randint(0, 2, u[:, odd].shape, generator=gen)
    q = W4(u.to(torch.uint8), s.to(sdt), z.to(torch.uint8), group)
    assert torch.equal(q.s.double(), s)
    w = dequant_w4(q).double()
    assert torch.equal(w * 16, (w * 16).round()) and float(w.abs().max()) <= 4
    if f16:
        assert not torch.equal(dequant_w4(q, 'the fp16 product is not rounded to fp16 before bf16').double(), w)
    for g in range(groups):
        mass = x[:, g * K:(g + 1) * K].double().abs() @ w[g].abs().t()
        assert float(mass.max()) < MASS_LIMIT
    b = torch.randint(-64, 65, (N,), generator=gen).float() if bias else None
    mv = lambda t: None if t is None else t.to(device)  # noqa: E731
    return mv(x), W4(*(mv(t) for t in q[:3]), group), None, mv(b)


def onehot_x(K, c, rows=TOK, device='cpu'):
    """the routing probe: row t one-hot at k = 64 c + t (rows past K stay zero), so out[t, n] == W[n, 64 c + t]
    exactly; c = 0 .. K / 64 - 1 visits every (n, k) pair once"""
    x = torch.zeros((rows, K), dtype=torch.bfloat16, device=device)
    t = torch.arange(min(TOK, K - 64 * c), device=device)
    x[t, 64 * c + t] = 1.0
    return x


# ------------------------------------------------------------------------------------------------ reference
def reference(x, w, scale=None, bias=None):
    """(ref, mass) in fp64 for one group: ref = x @ (w * scale)^T (+ bias), mass = |x| @ |w * scale|^T (+ |bias|).
    x [rows, K], w [N, K] bf16 / e4m3 / float (or int4 W4 codes of one group), scale [N] or None, bias [N] or None"""
    w = dense(w)
    wd = w.double() if w.dtype != torch.float8_e4m3fn else w.float().double()
    if scale is not None:
        wd = wd * scale.double()[:, None]
    xd = x.double()
    ref, mass = xd @ wd.t(), xd.abs() @ wd.abs().t()
    if bias is not None:
        ref, mass = ref + bias.double(), mass + bias.double().abs()
    return ref, mass


def bf16_exact(ref):
    """the expected output of exact-integer operands: bf16_rne of the exact value (which fp32 holds exactly); a zero
    is +0, as an accumulator that starts at +0 leaves it"""
    assert torch.equal(ref.float().double(), ref)
    return (ref.float() + 0.0).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ comparator
REL = 2.0 ** -8


def gamma(K, n_split=1):
    """the accumulation term of the comparator, per unit of sum_k |x_k| |w_k|: (K / 16 + n_split + 3) 2^-22"""
    return (K / 16 + n_split + 3) * 2.0 ** -22


def scores(got, ref, mass, K, n_split=1):
    """|got - ref| / (2^-8 |ref| + gamma sum_k |x_k| |w_k|) per element; the comparator accepts when every score is
    <= 1.  No absolute floor.  Where the two terms come from:

    The kernel's value before the output rounding, c, is an fp32 accumulation.  Each wgmma.m64n64k16 adds one 16-term
    block of exact bf16 x bf16 products into the fp32 accumulator; whatever the tensor core's internal alignment and
    truncation, that costs at most 2 ulp of the largest magnitude involved, and every partial sum and block is bounded
    by M = sum_k |x_k| |w_k|, so one step errs by <= 2 * 2^-23 M = 2^-22 M.  There are K / 16 steps; the split-K /
    cluster / stream-K partial sums add at most n_split fp32 roundings, the fp8 scale and the bias two more (2^-24 M
    each), so |c - ref| <= (K / 16 + n_split + 2) 2^-22 M.  The output is bf16_rne(c): bf16 keeps 8 significant bits,
    so |bf16(c) - c| <= 2^-8 |c| <= 2^-8 (|ref| + |c - ref|).  Together
        |got - ref| <= 2^-8 |ref| + (1 + 2^-8) (K / 16 + n_split + 2) 2^-22 M <= 2^-8 |ref| + gamma M.
    The first term is tight: just above a power of two, half a bf16 ulp is 2^-8 |ref|, so a correct kernel scores up
    to ~0.99 on some element of a large output.  The second is a worst case (the accumulation errors are a random
    walk), and it is the only slack a wrong kernel gets: a 16-k block or a slice missing, a wrong scale, or
    round-toward-zero (up to a whole ulp, score ~2) move elements past 1.  fp32 slices summed by the caller count as
    splits and one bf16 rounding."""
    got, ref, mass = got.double(), ref.double().to(got.device), mass.double().to(got.device)
    den = REL * ref.abs() + gamma(K, n_split) * mass
    diff = (got - ref).abs()
    return torch.where(den > 0, diff / den.clamp_min(1e-300), torch.where(diff > 0, float('inf'), 0.0))


def worst(got, ref, mass, K, n_split=1):
    return float(scores(got, ref, mass, K, n_split).max())


def assert_close(got, ref, mass, K, n_split=1, msg=''):
    """the comparator: every element within 2^-8 |ref| + gamma(K, n_split) sum_k |x_k| |w_k| (see `scores`)"""
    w = worst(got, ref, mass, K, n_split)
    assert w <= 1.0, f'{msg} worst score {w:.3g} (fraction of the tolerance used)'
    return w


def old_close(got, ref):
    """the fixed tolerance the GEMM tests used before the comparator"""
    return torch.allclose(got.double(), ref.double(), atol=2e-2, rtol=1.6e-2)


# ------------------------------------------------------------------------------------------------ kernel emulation
MUTATIONS = {
    'one 16-k step dropped': lambda p: True,
    'last (short) split dropped': lambda p: p.n_split > 1 and not p.cluster,
    'cluster write-out quad tokens swapped': lambda p: p.cluster > 0,
    "adjacent row's fp8 scale": lambda p: p.kind == 'fp8',
    'bias added per split': lambda p: p.kind in ('fp8', 'w4') and p.cluster > 0,
    'cluster partials rounded to bf16 before the sum': lambda p: p.cluster > 0,
    'round toward zero (__float2bfloat16_rz)': lambda p: p.cluster > 0 or p.n_split == 1,
    'grouped GEMM reads the wrong X column offset': lambda p: p.groups > 1,
    "a half takes its chunk's first group's scale and zero point": lambda p: p.kind == 'w4' and p.group % W4_BK != 0,
    'rows r and r + 8 swap scales': lambda p: p.kind == 'w4',
    'the fp16 product is not rounded to fp16 before bf16': lambda p: p.kind == 'w4' and p.f16,
    'the half chunk is dropped': lambda p: p.kind == 'w4' and p.K % W4_BK == 128,
    "a grouped plan reads expert 0's table columns": lambda p: p.kind == 'w4' and p.groups > 1,
    'a 64-row k_gemm_stream tile reads the other half of its 128-row block':
        lambda p: p.kind == 'stream' and p.wg == 1 and p.tiled,
}
W4_MUTATIONS = {"a half takes its chunk's first group's scale and zero point", 'rows r and r + 8 swap scales',
                'the fp16 product is not rounded to fp16 before bf16', "a grouped plan reads expert 0's table columns"}


def _bf16(v, rz=False):
    if not rz:
        return v.to(torch.bfloat16)
    return (v.contiguous().view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


def _acc(P, b0, b1, skip=None):
    """fp32 accumulation of the 16-k block products P[b0:b1] in order, starting from +0"""
    acc = torch.zeros(P.shape[1:], dtype=torch.float32, device=P.device)
    for b in range(b0, b1):
        if b != skip:
            acc = acc + P[b]
    return acc


def emulate(p, x, w, scale=None, bias=None, mut=None):
    """the kernel's arithmetic in torch: each 16-k block product exact, rounded to fp32 and added to an fp32
    accumulator that starts at 0 for every (tile, split) / stream-K segment; fp8: the partial times s[n] in fp32;
    int4: the dequantised weight, 256-k chunks of which the last is a 128-k half when K % 256 == 128; cluster:
    partials summed in split order, then + bias, one bf16 rounding; slices: the fp32 partials; stream-K: the owner's
    segment plus the contributor slots in order; k_gemm_stream: k_gemm_ws's split-1 sums.  x [rows, groups * K], w
    [groups, N, K] (bf16 / e4m3 / float, or W4 codes), scale [groups * N], bias [N].  mut: a key of MUTATIONS.  Returns
    bf16 [rows, N] (or [groups, rows, N]), or fp32 slices [n_split, rows, N]."""
    rows, K, N = x.shape[0], p.K, p.N
    if isinstance(w, W4):
        w = dequant_w4(w, mut if mut in W4_MUTATIONS else None)
        if mut == 'the half chunk is dropped':
            w = w.clone()
            w[:, :, K - 128:] = 0
    if mut == 'a 64-row k_gemm_stream tile reads the other half of its 128-row block':
        w = w[:, torch.arange(N, device=w.device) ^ 64]
    outs = []
    for g in range(p.groups):
        x0 = g * K + (64 if mut == 'grouped GEMM reads the wrong X column offset' else 0)
        xg = torch.zeros((rows, K), dtype=torch.float64, device=x.device)
        xs = x[:, x0:min(x0 + K, x.shape[1])].double()
        xg[:, :xs.shape[1]] = xs
        wg = w[g].float().double()
        nb = K // 16
        P = torch.einsum('tbk,nbk->btn', xg.view(rows, nb, 16), wg.view(N, nb, 16)).float()
        bpc = p.bk // 16
        skip = 1 if mut == 'one 16-k step dropped' else None
        if p.kind == 'sk':
            U, out = p.tiles * p.n_chunks, torch.empty((rows, N), dtype=torch.float32, device=x.device)
            for t in range(p.tiles):
                segs = [_acc(P[:, :, t * BMW:(t + 1) * BMW], c0 * bpc, c1 * bpc, skip)
                        for _, c0, c1 in sk_segments(t, p.n_chunks, U, p.sk_grid)]
                acc = segs[0]
                for s in segs[1:]:
                    acc = acc + s
                out[:, t * BMW:(t + 1) * BMW] = acc
            outs.append(_bf16(out, mut == 'round toward zero (__float2bfloat16_rz)'))
            continue
        parts = [_acc(P, c0 * bpc, min(c1 * bpc, nb), skip) for c0, c1 in split_ranges(p)]
        if scale is not None:
            sc = scale[g * N:(g + 1) * N].float().to(x.device)
            if mut == "adjacent row's fp8 scale":
                sc = sc[torch.arange(N, device=x.device) ^ 1]
            parts = [q * sc for q in parts]
        bs = torch.zeros(N, device=x.device) if bias is None else bias.float().to(x.device)
        if p.n_split > 1 and not p.cluster:
            if mut == 'last (short) split dropped':
                parts[-1] = torch.zeros_like(parts[-1])
            outs.append(torch.stack(parts))
            continue
        if mut == 'cluster partials rounded to bf16 before the sum':
            parts = [q.to(torch.bfloat16).float() for q in parts]
        if mut == 'bias added per split':
            parts = [q + bs for q in parts]
        a = parts[0]
        for q in parts[1:]:
            a = a + q
        if mut != 'bias added per split':
            a = a + bs
        o = _bf16(a, mut == 'round toward zero (__float2bfloat16_rz)')
        if mut == 'cluster write-out quad tokens swapped':
            perm = torch.arange(rows)
            for t0 in range(0, rows - 1, 4):
                perm[t0], perm[t0 + 1] = t0 + 1, t0
            o = o[perm.to(o.device)]
        outs.append(o)
    return outs[0] if p.groups == 1 else torch.stack(outs)


def slice_sum(slices):
    """what pia_rmsnorm_partials feeds on: the fp32 slices summed in slice order, one bf16 rounding"""
    a = slices[0].float()
    for s in slices[1:]:
        a = a + s.float()
    return a.to(torch.bfloat16)


def exact_slices(p, x, w, scale=None):
    """the fp32 slices exact-integer operands must produce bit for bit: the exact partial sum of every split's k range
    (times s[n] for fp8; the dequantised weight for int4), [n_split, rows, N]"""
    out = []
    for c0, c1 in split_ranges(p):
        k0, k1 = c0 * p.bk, min(c1 * p.bk, p.K)
        r, _ = reference(x[:, k0:k1], dense(w)[0][:, k0:k1], None if scale is None else scale[:p.N])
        out.append(r)
    return torch.stack(out)


def mutation_names(p):
    return [m for m, applies in MUTATIONS.items() if applies(p)]


def describe(p):
    """a short path label: the kernel instance, split mode, layout / groups"""
    if p.kind == 'sk':
        return f'k_gemm_sk units/CTAs={p.tiles * p.n_chunks}/{p.sk_grid}'
    if p.kind == 'stream':
        return f'{instance(p)} split1 {"tiled" if p.tiled else "row-major"}'
    mode = f'cluster{p.cluster}' if p.cluster else ('split1' if p.n_split == 1 else f'slices{p.n_split}')
    out = f'{instance(p)} {mode}' + (f' groups={p.groups}' if p.groups > 1 else '')
    return out + (f' group={p.group}{" fp16" if p.f16 else " bf16"} scales' if p.kind == 'w4' else '')
