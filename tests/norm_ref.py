# -*- coding: utf-8 -*-
"""Plain-torch restatement of k_rmsnorm and k_silu_mul (csrc/fused_ops.cu) for the norm tests: an fp64 reference of
both RMSNorm rounding modes and of SiLU*up, a comparator that tolerates only real ties, the exact split-K slice sum,
an fp32 emulation of each kernel's operations and the wrong kernels (mutations) the checks must reject.  Runs on any
device; nothing here needs a GPU.

RMSNorm rounding modes (pia_rmsnorm's `rounding`):
  ONCE:  y = bf16(w * x_hat)        llama/modeling_llama.py:90, chatglm/modeling_chatglm.py:187, chatglm3/...:196
  TWICE: y = bf16(w * bf16(x_hat))  mistral/modeling_mistral.py:90, mixtral/...:165, qwen2/...:96, the Baichuan
                                    members (h.to(weight.dtype), then weight * h), transformers' Glm(4)RMSNorm
with x_hat = x * rsqrt(mean(x^2) + eps) and x = bf16(x + residual) when there is a residual."""
import math

import torch

ONCE, TWICE = 0, 1
U = 2.0 ** -24              # fp32 unit roundoff
THREADS, WARPS = 512, 16    # k_rmsnorm's CTA
MAX_HIDDEN = 16384
FLT_MAX = float(torch.finfo(torch.float32).max)
BF16_OVERFLOW = 2.0 ** 128  # the first value past the bf16 grid (it rounds to inf)


# ------------------------------------------------------------------------------------------------ bf16 rounding
def bf16_rne(z):
    """z (any float tensor) rounded to the nearest bf16 value, ties to even, computed exactly in fp64 (no detour
    through fp32, which could round twice); returned as fp64"""
    z = z.double()
    out = z.clone()
    fin = torch.isfinite(z) & (z != 0)
    v = z[fin]
    _, e = torch.frexp(v)                              # |v| in [2^(e-1), 2^e): 8 significant bits -> ulp 2^(e-8)
    k = torch.clamp(e - 8, min=-133)                   # bf16 subnormals: spacing 2^-133
    r = torch.ldexp(torch.round(torch.ldexp(v, -k)), k)   # torch.round rounds half to even
    r = torch.where(r.abs() >= BF16_OVERFLOW, torch.sign(r) * math.inf, r)
    out[fin] = r
    return out


def bf(t):
    """fp32 -> bf16 -> fp32, as __float2bfloat16_rn and eager torch's casts do"""
    return t.float().to(torch.bfloat16).float()


# ------------------------------------------------------------------------------------------------ inputs of the norm
def slice_sum(parts):
    """what pia_rmsnorm_partials normalises: the fp32 slices summed in slice order, ((p0 + p1) + p2) + ..., then one
    bf16 rounding (bit exact: IEEE fp32 addition in a fixed order)"""
    acc = parts[0].float().clone()
    for s in range(1, parts.shape[0]):
        acc = acc + parts[s].float()
    return acc.to(torch.bfloat16)


def residual_sum(x, r):
    """bf16(x + r), the fp32 sum of two bf16 values rounded once, as the kernel and eager bf16 torch compute it"""
    return x if r is None else (x.float() + r.float()).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ error budget
def summation_depth(hidden):
    """the longest chain of fp32 additions in k_rmsnorm's sum of squares: each thread adds its 8 * ceil(nvec / 512)
    squares serially, then 5 shuffle levels, then the 16 warp sums serially"""
    per_thread = 8 * -(-(hidden // 8) // THREADS)
    return (per_thread - 1) + 5 + (WARPS - 1)


def rms_budget(hidden):
    """relative error bound of the fp32 evaluation of x_hat (and of w * x_hat), in units derived from the operations:
      * the squares of bf16 values are exact in fp32; the sum of d additions of non-negative terms is off by at most
        d u relative (d = summation_depth);
      * mean = tot / hidden: u (eager torch multiplies by an fp32 1/hidden instead: 2 u, taken);
      * + eps: u;  so the argument of rsqrt is within (d + 3) u, which moves rsqrt by (d + 3) u / 2;
      * rsqrtf: at most 2 ulp = 4 u;
      * x * inv: u;  w * x_hat (one-rounding mode): u.
    The total, ((d + 3) / 2 + 6) u, is doubled so that eager torch's summation order, whose depth is of the same size,
    is covered too: where torch and the kernel disagree, the fp64 value must be within this budget of a tie."""
    d = summation_depth(hidden)
    return 2.0 * ((d + 3) / 2.0 + 6.0) * U


def rmsnorm_ref(x, w, eps, r=None, parts=None):
    """fp64 reference: (residual sum s as bf16, x_hat = s * rsqrt(mean(s^2) + eps) in fp64).  eps is the fp32 value the
    kernel (and eager torch's fp32 add) uses"""
    a = slice_sum(parts) if parts is not None else x
    s = residual_sum(a, r)
    s64 = s.double()
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    inv = 1.0 / torch.sqrt((s64 * s64).mean(-1, keepdim=True) + eps32)
    return s, s64 * inv


def rms_accept(xh, w, rounding, hidden):
    """(lo, hi, ambiguous) for every element: the kernel's y must equal lo or hi; lo == hi except within the budget of
    a bf16 rounding boundary.  ONCE: the rounded value is w * x_hat.  TWICE: x_hat is rounded first (either neighbour
    where it is within budget of a boundary), then w * bf16(x_hat) is exact in fp32 and rounds deterministically."""
    rel = rms_budget(hidden)
    w64 = w.double()
    if rounding == ONCE:
        z = w64 * xh
        e = rel * z.abs()
        lo, hi = bf16_rne(z - e), bf16_rne(z + e)
    else:
        e = rel * xh.abs()
        c_lo, c_hi = bf16_rne(xh - e), bf16_rne(xh + e)
        lo, hi = bf16_rne(w64 * c_lo), bf16_rne(w64 * c_hi)
    return lo, hi, lo != hi


def rms_check(got, xh, w, rounding, hidden):
    """(number of elements outside the accepted set, number of ambiguous elements).  The ambiguous ones come in clumps:
    in a row every x with the same 8-bit significand lands at the same place relative to the bf16 grid after the
    multiply by the row's one inv, so a share is only meaningful over many rows"""
    lo, hi, amb = rms_accept(xh, w, rounding, hidden)
    g = got.double()
    bad = ~((g == lo) | (g == hi))
    return int(bad.sum()), int(amb.sum())


# ------------------------------------------------------------------------------------------------ SiLU * up
LN_FLT_MAX = math.log(FLT_MAX)


def silu_ref(g):
    """fp64 g / (1 + exp(-g)) as the fp32 op sequence evaluates it: where exp(-g) overflows fp32 (g < -88.72) the
    denominator is inf and the quotient -0"""
    g64 = g.double()
    s = g64 / (1.0 + torch.exp(-g64))
    return torch.where(torch.isfinite(g64) & (-g64 > LN_FLT_MAX), torch.zeros_like(s) * -1.0, s)


def silu_budget():
    """relative error of the fp32 SiLU: expf is within 2 ulp (4 u), 1 + e adds u, the division u: 6 u, doubled; plus an
    absolute 2^-149 for quotients in the fp32 subnormal range"""
    return 12.0 * U, 2.0 ** -149


def silu_accept(g, u):
    """(lo, hi, ambiguous): y = bf16(bf16(silu(g)) * u); the first rounding may go either way within the budget, the
    product of two bf16 values is exact and rounds once"""
    s = silu_ref(g)
    rel, ab = silu_budget()
    e = torch.where(torch.isfinite(s), rel * s.abs() + ab, torch.zeros_like(s))
    c_lo, c_hi = bf16_rne(s - e), bf16_rne(s + e)
    u64 = u.double()
    lo, hi = bf16_rne(c_lo * u64), bf16_rne(c_hi * u64)
    return lo, hi, (lo != hi) & ~(torch.isnan(lo) & torch.isnan(hi))


def silu_check(got, g, u):
    lo, hi, amb = silu_accept(g, u)
    gd = got.double()
    ok = (gd == lo) | (gd == hi) | (torch.isnan(gd) & torch.isnan(lo) & torch.isnan(hi))
    return int((~ok).sum()), float(amb.double().mean())


# ------------------------------------------------------------------------------------------------ fp32 emulations
def _sum_of_squares(s):
    """k_rmsnorm's fp32 sum of squares, in its order: per thread serially over vectors t, t + 512, ... (8 elements
    each), an xor-shuffle butterfly within each warp, then the 16 warp sums serially"""
    rows, hidden = s.shape
    nvec = hidden // 8
    k = -(-nvec // THREADS)
    f = s.float() ** 2                                  # exact for bf16 values: 8 significant bits
    pad = torch.zeros((rows, k * THREADS * 8), dtype=torch.float32)
    pad[:, :hidden] = f
    per = pad.view(rows, k, THREADS, 8).permute(0, 2, 1, 3).reshape(rows, THREADS, k * 8)
    acc = torch.zeros((rows, THREADS), dtype=torch.float32)
    for i in range(k * 8):
        acc = acc + per[:, :, i]
    lanes = acc.view(rows, WARPS, 32)
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, :, idx ^ o]
    tot = torch.zeros((rows,), dtype=torch.float32)
    for wi in range(WARPS):
        tot = tot + lanes[:, wi, 0]
    return tot


def emulate_rmsnorm(x, w, eps, rounding, r=None, parts=None, mut=None):
    """the kernel's arithmetic in fp32 on the CPU -> (residual_out, y) as bf16.  mut: a name of RMS_MUTATIONS"""
    if parts is not None:
        a = slice_sum(parts.flip(0) if mut == 'slices_reversed' else parts)
    else:
        a = x
    s = residual_sum(a, r)
    sq = s
    if mut == 'residual_unrounded' and r is not None:
        sq = a.float() + r.float()
    hidden = s.shape[-1]
    tot = _sum_of_squares(sq)
    n = float(hidden - 1) if mut == 'mean_over_hidden_minus_1' else float(hidden)
    mean = tot / torch.tensor(n, dtype=torch.float32)
    eps32 = torch.tensor(eps, dtype=torch.float32)
    if mut == 'no_eps':
        inv = torch.rsqrt(mean)
    elif mut == 'eps_after_sqrt':
        inv = 1.0 / (torch.sqrt(mean) + eps32)
    else:
        inv = torch.rsqrt(mean + eps32)
    src = s
    if mut == 'inplace_reread' and r is not None and hidden > 2 * THREADS * 8:
        # the old second pass for vectors past 2 per thread: x + residual_in again, after residual_out (== residual_in)
        # already holds the sum
        src = s.clone()
        src[:, 2 * THREADS * 8:] = (a[:, 2 * THREADS * 8:].float() + s[:, 2 * THREADS * 8:].float()).to(torch.bfloat16)
    xh = src.float() * inv[:, None]
    rnd = rounding if mut != 'other_rounding' else 1 - rounding
    y = w.float() * (bf(xh) if rnd == TWICE else xh)
    return s, y.to(torch.bfloat16)


RMS_MUTATIONS = ('other_rounding', 'residual_unrounded', 'no_eps', 'eps_after_sqrt', 'mean_over_hidden_minus_1',
                 'slices_reversed', 'inplace_reread')


def emulate_silu(gu, mut=None):
    """k_silu_mul in fp32 on the CPU: gu [rows, 2 * inter] (gate | up) -> bf16 [rows, inter]"""
    inter = gu.shape[-1] // 2
    g, u = gu[:, :inter].float(), gu[:, inter:].float()
    if mut == 'gate_up_swapped':
        g, u = u, g
    s = g / (1.0 + torch.exp(-g))
    if mut != 'silu_unrounded':
        s = bf(s)
    return (s * u).to(torch.bfloat16)


SILU_MUTATIONS = ('silu_unrounded', 'gate_up_swapped')


# ------------------------------------------------------------------------------------------------ LayerNorm
# k_layernorm (pia_layernorm): BLOOM's and OPT's LayerNorm with weight and bias, after the bf16 residual add.  One CTA
# per row of blockDim = min(512, nvec rounded up to a warp) threads (nvec = hidden / 8 vectors); thread t owns vectors
# t, t + blockDim, ...  Both passes (the sum, then the sum of squared deviations) add in the same order: per thread
# serially over its vectors' 8 elements each, then 5 xor-shuffle levels, then the blockDim / 32 warp sums serially.
# Ptxas (CUDA 12.9, sm_90a) contracts `ss += d * d` into an FFMA chain and `x_hat * w + b` into one FFMA
# (x_hat = (f - mean) * rstd is an FMUL of its own); mean and variance are IEEE divisions by hidden, rstd is rsqrtf.
LN_MAX_HIDDEN = 16384


def ln_threads(hidden):
    """k_layernorm's blockDim at this width"""
    nvec = hidden // 8
    return THREADS if nvec >= THREADS else -(-nvec // 32) * 32


def ln_depth(hidden):
    """the longest chain of fp32 additions in either pass: 8 * ceil(nvec / blockDim) - 1 per thread (the first add is
    to 0), 5 shuffle levels, blockDim / 32 - 1 warp sums"""
    threads = ln_threads(hidden)
    return 8 * -(-(hidden // 8) // threads) - 1 + 5 + threads // 32 - 1


def _eps32(eps):
    return float(torch.tensor(eps, dtype=torch.float32))


def layernorm_ref(x, w, b, eps, r=None):
    """fp64 reference -> (s, x_hat, z, sum_scale, var): s = bf16(x + r) (or x), mu and the biased variance of s in
    fp64, x_hat = (s - mu) / sqrt(var + eps32) with eps the fp32 value the kernel receives, z = x_hat * w + b.
    sum_scale = mean |s| scales the rounding error of an fp32 mean; it is 0 for a constant row, whose mean is exact in
    any order (k equal bf16 values sum exactly in fp32 for k <= 2^16, and k c / k = c)"""
    s = residual_sum(x, r)
    s64 = s.double()
    mu = s64.mean(-1, keepdim=True)
    var = ((s64 - mu) ** 2).mean(-1, keepdim=True)
    xh = (s64 - mu) / torch.sqrt(var + _eps32(eps))
    const = (s64 == s64[..., :1]).all(-1, keepdim=True)
    scale = torch.where(const, torch.zeros_like(mu), s64.abs().mean(-1, keepdim=True))
    return s, xh, xh * w.double() + b.double(), scale, var


def ln_budget(xh, w, b, sum_scale, var, eps, hidden):
    """absolute error bound of the kernel's fp32 z = x_hat * w + b per element, before its one bf16 rounding, with
    d = ln_depth(hidden) and u the fp32 unit roundoff:
      * the mean: the sum of d additions is off by at most d u sum|s|, the division by hidden adds u |mu|, so
        |mean - mu| <= dmu = (d + 1) u mean|s| (sum_scale).  In f - mean this is an absolute error, which for an offset row (a
        large |mu| next to a small spread) is many ulps of f - mean; it reaches z as |w| dmu rstd;
      * the variance: f - mean rounds once (u per deviation, 2 u per square); the FFMA chain of non-negative squares
        adds d u; using mean instead of mu adds exactly dmu^2 to the mean square; / hidden u, + eps u.  The argument of
        rsqrt is within (d + 5) u + dmu^2 / (var + eps) relative (the chain's first step rounds d * d too: d + 1
        roundings), which moves rsqrt by half of that;
      * rsqrtf: at most 2 ulp = 4 u;  x_hat = (f - mean) * rstd: u;  so x_hat * w is within
        R = ((d + 5) / 2 + 6) u + dmu^2 / (2 (var + eps)) of itself, relative;
      * the final expression: one FFMA rounds once, u |z|; without contraction fl(fl(x_hat w) + b) rounds twice.  Both
        are within 2 u (|x_hat w| + |b|): relative to the addends, not to z, because where x_hat w and b cancel the
        fp32 result is only as exact as the addends' ulp.
    The total is doubled so that torch's LayerNorm (CUDA: Welford per thread, merged across the block), whose order
    differs but whose depth is of the same size, is covered too"""
    d = ln_depth(hidden)
    dmu = (d + 1) * U * sum_scale
    a = (xh * w.double()).abs()
    rel = ((d + 5) / 2.0 + 6.0) * U + dmu ** 2 / (2.0 * (var + _eps32(eps)))
    rstd = 1.0 / torch.sqrt(var + _eps32(eps))
    return 2.0 * (a * rel + w.double().abs() * dmu * rstd + 2.0 * U * (a + b.double().abs()))


def ln_accept(x, w, b, eps, r=None):
    """(lo, hi, ambiguous) for every element: the kernel's y must lie in [lo, hi] on the bf16 grid, the roundings of
    the ends of z's error interval; lo == hi except within the budget of a rounding boundary.  Where x_hat * w and b
    do not cancel, lo and hi are neighbours at most, so y is lo or hi"""
    _, xh, z, am, var = layernorm_ref(x, w, b, eps, r)
    e = ln_budget(xh, w, b, am, var, eps, x.shape[-1])
    lo, hi = bf16_rne(z - e), bf16_rne(z + e)
    return lo, hi, lo != hi


def ln_check(got, x, w, b, eps, r=None):
    """(number of elements outside the accepted set, number of ambiguous elements)"""
    lo, hi, amb = ln_accept(x, w, b, eps, r)
    g = got.double()
    bad = ~((g >= lo) & (g <= hi))
    return int(bad.sum()), int(amb.sum())


def _ln_block_sum(v, hidden, sq=None):
    """k_layernorm's block_sum of per-element fp32 terms v [rows, hidden] in its order.  sq: the deviations d whose
    squares the FFMA chain adds (each step rounds d * d + acc once, emulated in fp64 then rounded to fp32: exact except
    for a double rounding at a tie, which the comparator's budget dwarfs)"""
    src = v if sq is None else sq
    rows = src.shape[0]
    threads = ln_threads(hidden)
    k = -(-(hidden // 8) // threads)
    pad = torch.zeros((rows, k * threads * 8), dtype=torch.float32)
    pad[:, :hidden] = src
    per = pad.view(rows, k, threads, 8).permute(0, 2, 1, 3).reshape(rows, threads, k * 8)
    acc = torch.zeros((rows, threads), dtype=torch.float32)
    for i in range(k * 8):
        if sq is None:
            acc = acc + per[:, :, i]
        else:
            t = per[:, :, i].double()
            acc = (t * t + acc.double()).float()
    lanes = acc.view(rows, threads // 32, 32)
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, :, idx ^ o]
    tot = torch.zeros((rows,), dtype=torch.float32)
    for wi in range(threads // 32):
        tot = tot + lanes[:, wi, 0]
    return tot


def _ln_out(xh, w, b):
    """bf16(fma(x_hat, w, b)): x_hat * w (fp32 times bf16) is exact in fp64, so is its sum with b unless the two are
    far apart in magnitude"""
    return (xh.double() * w.double() + b.double()).float().to(torch.bfloat16)


def _ln_stats(f, hidden, eps, mut):
    n = hidden
    threads = ln_threads(hidden)
    if mut == 'mean_over_padded_width' and (hidden // 8) % 32:
        n = threads * 8
    n32 = torch.tensor(float(n), dtype=torch.float32)
    mean = _ln_block_sum(f, hidden) / n32
    eps32 = torch.tensor(eps, dtype=torch.float32)
    if mut == 'one_pass_variance':
        var = _ln_block_sum(None, hidden, sq=f) / n32 - mean * mean
    else:
        dev = f - mean[:, None]
        ss = _ln_block_sum(None, hidden, sq=dev)
        var = ss / (torch.tensor(float(n - 1), dtype=torch.float32) if mut == 'unbiased_variance' else n32)
    if mut == 'no_eps':
        rstd = torch.rsqrt(var)
    elif mut == 'eps_after_sqrt':
        rstd = 1.0 / (torch.sqrt(var) + eps32)
    else:
        rstd = torch.rsqrt(var + eps32)
    return mean, rstd


def emulate_layernorm(x, w, b, eps, r=None, mut=None, inplace=False, y_is_residual=False):
    """k_layernorm's arithmetic in fp32 on the CPU -> (residual sum as bf16, y as bf16).  inplace: residual_out is
    residual_in; y_is_residual: y is residual_in (OPT-350m's last post-LN call).  mut: a name of LN_MUTATIONS; the
    aliasing mutations only change a call that has their aliasing"""
    hidden = x.shape[-1]
    s = residual_sum(x, r)
    if mut == 'y_before_residual_read' and y_is_residual and r is not None:
        # the residual is read where y already holds the row's output
        _, y0 = emulate_layernorm(x, w, b, eps, r)
        s_seen = residual_sum(x, y0)
        _, y = emulate_layernorm(x, w, b, eps, y0)
        return s_seen, y
    f = s.float()
    if mut == 'residual_unrounded' and r is not None:
        mean, rstd = _ln_stats(x.float() + r.float(), hidden, eps, None)
    elif mut == 'stats_without_residual' and r is not None:
        mean, rstd = _ln_stats(x.float(), hidden, eps, None)
    else:
        mean, rstd = _ln_stats(f, hidden, eps, mut)
    src = f
    threads = ln_threads(hidden)
    if mut == 'inplace_reread' and inplace and r is not None and hidden > 2 * threads * 8:
        # the output pass re-forms x + residual_in for vectors past 2 per thread, after residual_out (== residual_in)
        # already holds the sum
        src = f.clone()
        tail = slice(2 * threads * 8, None)
        src[:, tail] = (x[:, tail].float() + s[:, tail].float()).to(torch.bfloat16).float()
    xh = (src - mean[:, None]) * rstd[:, None]
    if mut == 'xhat_rounded':
        y = _ln_out(bf(xh), w, b)
    elif mut == 'two_roundings':
        y = (bf(xh * w.float()) + b.float()).to(torch.bfloat16)
    elif mut == 'bias_dropped':
        y = (xh * w.float()).to(torch.bfloat16)
    else:
        y = _ln_out(xh, w, b)
    return s, y


LN_MUTATIONS = ('no_eps', 'eps_after_sqrt', 'unbiased_variance', 'one_pass_variance', 'xhat_rounded', 'two_roundings',
                'bias_dropped', 'residual_unrounded', 'stats_without_residual', 'mean_over_padded_width',
                'inplace_reread', 'y_before_residual_read')
