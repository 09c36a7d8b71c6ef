# -*- coding: utf-8 -*-
"""Thin typed wrappers over the C ABI (include/pia_b200.h) for torch tensors: raw device pointers + the current
torch stream, nothing else. Every call is asynchronous and CUDA-graph capturable."""
import ctypes as C
import math

import torch

from .. import _lib as L


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return t.data_ptr() if t is not None else None


ROUND_ONCE, ROUND_TWICE = L.RMSNORM_ROUND_ONCE, L.RMSNORM_ROUND_TWICE


def rmsnorm(x, residual_in, weight, eps, residual_out, y, *, rounding=ROUND_ONCE):
    """y = RMSNorm(x (+ residual_in)), the residual sum to residual_out (pia_rmsnorm).  rounding: ROUND_ONCE,
    bf16(w * x_hat) (Llama, ChatGLM), or ROUND_TWICE, bf16(w * bf16(x_hat)) (Mistral, Mixtral, Qwen2, Baichuan, GLM)"""
    rows, hidden = x.shape
    L.check(L.load().pia_rmsnorm(_p(x), _p(residual_in), _p(weight), float(eps), int(rounding), rows, hidden,
                                 _p(residual_out), _p(y), _s()))


def rmsnorm_partials(parts, residual_in, weight, eps, residual_out, y, *, rounding=ROUND_ONCE):
    """parts: fp32 [n_parts, 64, hidden] split-K slices of a Gemm; rounding as rmsnorm"""
    n_parts, prow, hidden = parts.shape
    rows = y.shape[0]
    L.check(L.load().pia_rmsnorm_partials(_p(parts), n_parts, prow * hidden, _p(residual_in), _p(weight), float(eps),
                                          int(rounding), rows, hidden, _p(residual_out), _p(y), _s()))


def layernorm(x, residual_in, weight, bias, eps, residual_out, y):
    """y = LayerNorm(x (+ residual_in)) with weight and bias; the residual sum goes to residual_out (pia_layernorm)"""
    rows, hidden = x.shape
    L.check(L.load().pia_layernorm(_p(x), _p(residual_in), _p(weight), _p(bias), float(eps), rows, hidden,
                                   _p(residual_out), _p(y), _s()))


def bloom_gelu(x, out=None):
    """BLOOM's tanh-GELU with eager bf16 rounding (pia_bloom_gelu); out=None: in place"""
    out = x if out is None else out
    assert x.is_contiguous() and out.is_contiguous() and out.numel() == x.numel()
    L.check(L.load().pia_bloom_gelu(_p(x), x.numel(), _p(out), _s()))
    return out


def tile_weight(w):
    """[N, K] -> [N/128, K/64, 128, 64] contiguous: one 16 KB block per (128-row tile, 64-wide k chunk), the unit the
    GEMM kernel's TMA box moves, so each CTA reads one contiguous slab of HBM"""
    N, K = w.shape
    assert N % 128 == 0 and K % 64 == 0
    t = w.view(N // 128, 128, K // 64, 64).permute(0, 2, 1, 3).contiguous()
    t.pia_shape = (N, K)
    return t


def interleave_gate_up(w_gate_up):
    """[gate (I rows); up (I rows)] -> per 128-row tile: 64 gate rows then the 64 up rows of the same columns, the
    layout the fused SiLU*up epilogue of the GEMM expects"""
    two_i, K = w_gate_up.shape
    inter = two_i // 2
    assert inter % 64 == 0
    g = w_gate_up[:inter].view(inter // 64, 64, K)
    u = w_gate_up[inter:].view(inter // 64, 64, K)
    return torch.cat([g, u], dim=1).reshape(two_i, K).contiguous()


FP8_MAX = 448.0
# position p of every 16-byte k group of a tiled fp8 weight holds k = _FP8_KPERM[p]: thread c of a wgmma A fragment
# finds its codes for k {2c, 2c+1} and {2c+8, 2c+9} in one 32-bit word
_FP8_KPERM = (0, 1, 8, 9, 2, 3, 10, 11, 4, 5, 12, 13, 6, 7, 14, 15)


def quantize_fp8(w):
    """per-output-row symmetric e4m3 of a weight [..., N, K]: s[n] = amax(|W[n, :]|) / 448 (1 for an all-zero row),
    q = RNE(clamp(W / s, +-448)); the dequantised weight is float(q) * s[n].  Returns (q float8_e4m3fn, s fp32 [..., N]);
    computed in fp32 on w's device, a slab of rows at a time."""
    q = torch.empty(w.shape, dtype=torch.float8_e4m3fn, device=w.device)
    s = torch.empty(w.shape[:-1], dtype=torch.float32, device=w.device)
    w2, q2, s2 = w.reshape(-1, w.shape[-1]), q.view(-1, w.shape[-1]), s.view(-1)
    step = max(1, (1 << 26) // max(w.shape[-1], 1))
    for r in range(0, w2.shape[0], step):
        x = w2[r:r + step].float()
        amax = x.abs().amax(dim=1)
        sc = torch.where(amax > 0, amax / FP8_MAX, torch.ones_like(amax))
        q2[r:r + step] = (x / sc[:, None]).clamp_(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
        s2[r:r + step] = sc
    return q, s


def tile_weight_fp8(q):
    """e4m3 [..., N, K] -> uint8 [..., N/128, K/128, 128, 128] contiguous (the fp8 GEMM's HBM layout): one 16 KB block
    per (128-row tile, 128-wide k chunk), k permuted inside every 16-byte group by _FP8_KPERM"""
    N, K = q.shape[-2:]
    if N % 128 or K % 128:
        raise ValueError(f'the fp8 GEMM needs both weight dimensions to be multiples of 128, got [{N}, {K}]')
    lead = q.shape[:-2]
    b = q.view(torch.uint8).reshape(-1, N // 128, 128, K // 128, 8, 16)
    perm = torch.tensor(_FP8_KPERM, device=q.device)
    t = b.index_select(5, perm).permute(0, 1, 3, 2, 4, 5).reshape(*lead, N // 128, K // 128, 128, 128).contiguous()
    return t


def untile_weight_fp8(t):
    """inverse of tile_weight_fp8: uint8 [..., N/128, K/128, 128, 128] -> e4m3 [..., N, K]"""
    nt, kt = t.shape[-4:-2]
    lead = t.shape[:-4]
    inv = torch.empty(16, dtype=torch.long)
    inv[torch.tensor(_FP8_KPERM)] = torch.arange(16)
    b = t.reshape(-1, nt, kt, 128, 8, 16).index_select(5, inv.to(t.device))
    return b.permute(0, 1, 3, 2, 4, 5).reshape(*lead, nt * 128, kt * 128).contiguous().view(torch.float8_e4m3fn)


# position p (a nibble, low half of its byte first) of every 16-byte group of a tiled int4 weight holds k =
# _W4_KPERM[p] of the group's 32: word c (bytes 4c..4c+3) is thread c's, its nibble j holds k 2c + (0, 8, 16, 24)[j % 4]
# + j // 4, so that word >> 8t and word >> (8t + 4), masked with 0x000F000F, are the k pairs of the thread's a0 and a2
# fragment registers of the group's k-step t
_W4_KPERM = tuple(2 * c + (0, 8, 16, 24)[j % 4] + j // 4 for c in range(4) for j in range(8))
W4_SCALE_DTYPES = (torch.bfloat16, torch.float16)


def dequantize_w4(u, s, z, group_size):
    """the weight the int4 GEMM multiplies with, W[n, k] = bf16(dtype_s(s[n, g] * (u[n, k] - z[n, g]))), g = k // group:
    u uint8 [N, K] codes 0..15, s [N, G] bf16 or fp16, z uint8 [N, G] zero points (the unpackers' form).  u - z is exact
    in the scale's dtype, the product is rounded once to it (as compressed-tensors' dequantisation does), then to bf16."""
    N, K = u.shape
    rep = lambda t: t.repeat_interleave(group_size, dim=1)[:, :K]
    return ((u.to(s.dtype) - rep(z).to(s.dtype)) * rep(s)).to(torch.bfloat16)


def tile_weight_w4(u):
    """int4 codes uint8 [N, K] (values 0..15) -> uint8 [N/128, ceil(K/256), 128, 128] contiguous (the int4 GEMM's HBM
    layout): one 16 KB block per (128-row tile, 256-wide k chunk), two codes per byte, nibbles permuted inside every
    16-byte group by _W4_KPERM; a K that is an odd multiple of 128 is padded with zero codes the kernel never reads"""
    N, K = u.shape
    if N % 128 or K % 128:
        raise ValueError(f'the int4 GEMM needs both weight dimensions to be multiples of 128, got [{N}, {K}]')
    if K % 256:
        u = torch.cat([u, u.new_zeros((N, 128))], dim=1)
    kc = u.shape[1] // 256
    b = u.reshape(N // 128, 128, kc, 8, 32).index_select(4, torch.tensor(_W4_KPERM, device=u.device))
    b = (b[..., 0::2] | (b[..., 1::2] << 4)).to(torch.uint8)
    return b.permute(0, 2, 1, 3, 4).reshape(N // 128, kc, 128, 128).contiguous()


def untile_weight_w4(t, K):
    """inverse of tile_weight_w4: uint8 [N/128, ceil(K/256), 128, 128] -> codes uint8 [N, K]"""
    nt, kc = t.shape[:2]
    inv = torch.empty(32, dtype=torch.long)
    inv[torch.tensor(_W4_KPERM)] = torch.arange(32)
    b = t.reshape(nt, kc, 128, 8, 16)
    nib = torch.stack([b & 15, b >> 4], dim=-1).reshape(nt, kc, 128, 8, 32).index_select(4, inv.to(t.device))
    return nib.permute(0, 2, 1, 3, 4).reshape(nt * 128, kc * 256)[:, :K].contiguous()


def _unpack_nibbles(packed, dim):
    """int32 tensor with 8 nibbles per element (nibble i at bits 4i) -> uint8 codes, the 8 nibbles of an element
    consecutive along `dim` (0 or 1)"""
    p = packed.to(torch.int32)
    nib = torch.stack([(p >> (4 * i)) & 15 for i in range(8)], dim=dim + 1)   # [..., 8] next to the packed dim
    shape = list(p.shape)
    shape[dim] *= 8
    return nib.reshape(shape).to(torch.uint8)


def unpack_compressed_tensors_w4(weight_packed, weight_scale, weight_shape=None, weight_zero_point=None):
    """compressed-tensors `pack-quantized` (num_bits 4): weight_packed int32 [N, K/8] (nibble i of column j is k = 8j + i,
    stored as the signed code + 8), weight_scale [N, G] (G = 1: channel-wise), weight_zero_point None (symmetric: z = 8)
    or int32 [ceil(N/8), G] packed along N, stored zp + 8 (an int8 [N, G] tensor of signed zero points is taken too).
    Returns the internal form (u uint8 [N, K], s [N, G] in the scale's dtype, z uint8 [N, G], group size)."""
    N = weight_packed.shape[0]
    K = int(weight_shape[1]) if weight_shape is not None else weight_packed.shape[1] * 8
    u = _unpack_nibbles(weight_packed, 1)[:, :K].contiguous()
    s = weight_scale
    if s.dim() == 1:
        s = s[:, None]
    if s.dtype not in W4_SCALE_DTYPES:
        raise ValueError(f'weight_scale dtype {s.dtype}: the int4 GEMM takes bf16 or fp16 scales')
    G = s.shape[1]
    if s.shape[0] != N or K % G:
        raise ValueError(f'weight_scale {tuple(s.shape)} does not fit a [{N}, {K}] weight')
    if weight_zero_point is None:
        z = torch.full((N, G), 8, dtype=torch.uint8, device=u.device)
    elif weight_zero_point.dtype == torch.int32:
        z = _unpack_nibbles(weight_zero_point, 0)[:N].contiguous()
    else:
        z = (weight_zero_point.to(torch.int16) + 8).to(torch.uint8).reshape(N, G)
    return u, s.contiguous(), z, K // G


def unpack_gptq_w4(qweight, qzeros, scales, g_idx=None):
    """GPTQ 4-bit, checkpoint_format v1: qweight int32 [K/8, N] packed along K (nibble i of row j is k = 8j + i),
    qzeros int32 [G, N/8] packed along N, stored z - 1, scales [G, N], g_idx [K] (must be k // group: no act-order).
    Returns the internal form (u uint8 [N, K], s [N, G], z uint8 [N, G], group size)."""
    u = _unpack_nibbles(qweight, 0).t().contiguous()
    N, K = u.shape
    G = scales.shape[0]
    if scales.shape[1] != N or K % G:
        raise ValueError(f'scales {tuple(scales.shape)} do not fit a [{N}, {K}] weight')
    if scales.dtype not in W4_SCALE_DTYPES:
        raise ValueError(f'scales dtype {scales.dtype}: the int4 GEMM takes bf16 or fp16 scales')
    gs = K // G
    if g_idx is not None and not torch.equal(g_idx.to(torch.long).cpu(), torch.arange(K) // gs):
        raise ValueError('g_idx is not k // group_size (act-order / desc_act GPTQ): not supported')
    z = ((_unpack_nibbles(qzeros, 1)[:, :N].to(torch.int16) + 1)).to(torch.uint8).t().contiguous()
    return u, scales.t().contiguous(), z, gs


class Gemm(object):
    """pia_gemm_plan_t: Y = X @ W^T for one (weight, activation buffer) pair; `out` is bf16 [rows, N] when the plan
    has one K split, else fp32 [splits, 64, N]"""

    def __init__(self, weight, x, split_k=1, tiled=False):
        """weight: [N, K] row-major, or (tiled=True) the output of tile_weight() with its logical shape in .pia_shape"""
        N, K = weight.pia_shape if tiled else weight.shape
        assert x.shape[1] == K and x.is_contiguous() and weight.is_contiguous()
        self.lib = L.load()
        self.h = L.vp()
        with torch.cuda.device(weight.device):
            L.check(self.lib.pia_gemm_plan_create(_p(weight), N, K, _p(x), x.shape[0], split_k, int(tiled),
                                                  C.byref(self.h)))
        self.splits = self.lib.pia_gemm_plan_splits(self.h)
        self.N = N
        self._keep = (weight, x)
        self.weight = weight
        if self.splits == 1:
            self.out = torch.empty((x.shape[0], N), dtype=torch.bfloat16, device=weight.device)
        else:
            self.out = torch.empty((self.splits, 64, N), dtype=torch.float32, device=weight.device)

    @classmethod
    def grouped(cls, weight, x):
        """one launch for all experts: weight [G, N, K] (stacked, contiguous), x [rows >= 64, G * K];
        out [G, 64, N] bf16 (pia_gemm_plan_create_grouped)"""
        G, N, K = weight.shape
        assert weight.is_contiguous() and x.is_contiguous() and x.shape[1] == G * K
        self = cls.__new__(cls)
        self.lib = L.load()
        self.h = L.vp()
        with torch.cuda.device(weight.device):
            L.check(self.lib.pia_gemm_plan_create_grouped(_p(weight), G, N, K, _p(x), x.shape[0], C.byref(self.h)))
        self.splits, self.N, self.weight, self._keep = 1, N, weight, (weight, x)
        self.out = torch.empty((G, 64, N), dtype=torch.bfloat16, device=weight.device)
        return self

    @classmethod
    def fp8(cls, qweight, scale, x, bias=None, split_k=1, out=None):
        """fp8 weight plan (pia_gemm_plan_create_fp8): qweight = tile_weight_fp8(q) of an [N, K] weight, scale fp32 [N]
        (same row order), bias fp32 [N] or None; runs 1..x.shape[0] rows.  out (allocated unless given): bf16
        [x_rows, N] (N/2 columns with set_silu), or fp32 [splits, x_rows, N] slices for split_k > 1"""
        nt, kt = qweight.shape[-4:-2]
        N, K = nt * 128, kt * 128
        assert qweight.dtype == torch.uint8 and qweight.is_contiguous() and qweight.dim() == 4
        assert scale.dtype == torch.float32 and scale.numel() == N and x.shape[1] == K and x.is_contiguous()
        assert bias is None or (bias.dtype == torch.float32 and bias.numel() == N and bias.is_contiguous())
        self = cls.__new__(cls)
        self.lib = L.load()
        self.h = L.vp()
        with torch.cuda.device(qweight.device):
            L.check(self.lib.pia_gemm_plan_create_fp8(_p(qweight), _p(scale), _p(bias), N, K, _p(x), x.shape[0],
                                                      split_k, C.byref(self.h)))
        self.splits = self.lib.pia_gemm_plan_splits(self.h)
        self.N, self.weight, self._keep = N, qweight, (qweight, scale, bias, x)
        if out is not None:
            self.out = out
        elif self.splits == 1:
            self.out = torch.empty((x.shape[0], N), dtype=torch.bfloat16, device=x.device)
        else:
            self.out = torch.empty((self.splits, x.shape[0], N), dtype=torch.float32, device=x.device)
        return self

    @classmethod
    def w4(cls, codes, scale_t, zero_t, group_size, x, bias=None, split_k=1, out=None):
        """int4 weight plan (pia_gemm_plan_create_w4): codes = tile_weight_w4(u) of an [N, K] weight, scale_t [K/group, N]
        bf16 or fp16 and zero_t uint8 [K/group, N] (the unpackers' s and z transposed, same row order), bias fp32 [N] or
        None; runs 1..x.shape[0] rows; out as for fp8()"""
        G, N = scale_t.shape
        K = G * group_size
        assert codes.dtype == torch.uint8 and codes.is_contiguous() and codes.dim() == 4
        assert tuple(codes.shape) == (N // 128, -(-K // 256), 128, 128)
        assert scale_t.dtype in W4_SCALE_DTYPES and scale_t.is_contiguous()
        assert zero_t.dtype == torch.uint8 and tuple(zero_t.shape) == (G, N) and zero_t.is_contiguous()
        assert x.shape[1] == K and x.is_contiguous()
        assert bias is None or (bias.dtype == torch.float32 and bias.numel() == N and bias.is_contiguous())
        self = cls.__new__(cls)
        self.lib = L.load()
        self.h = L.vp()
        with torch.cuda.device(codes.device):
            L.check(self.lib.pia_gemm_plan_create_w4(_p(codes), _p(scale_t), _p(zero_t),
                                                     int(scale_t.dtype == torch.float16), _p(bias), N, K,
                                                     int(group_size), _p(x), x.shape[0], split_k, C.byref(self.h)))
        self.splits = self.lib.pia_gemm_plan_splits(self.h)
        self.N, self.weight, self._keep = N, codes, (codes, scale_t, zero_t, bias, x)
        if out is not None:
            self.out = out
        elif self.splits == 1:
            self.out = torch.empty((x.shape[0], N), dtype=torch.bfloat16, device=x.device)
        else:
            self.out = torch.empty((self.splits, x.shape[0], N), dtype=torch.float32, device=x.device)
        return self

    @classmethod
    def grouped_fp8(cls, qweight, scale, x):
        """one launch for all experts (pia_gemm_plan_create_grouped_fp8): qweight = tile_weight_fp8 of [G, N, K],
        scale fp32 [G, N], x [rows, G * K]; out bf16 [G, x_rows, N]"""
        G, nt, kt = qweight.shape[:3]
        N, K = nt * 128, kt * 128
        assert qweight.dtype == torch.uint8 and qweight.is_contiguous() and qweight.dim() == 5
        assert scale.dtype == torch.float32 and scale.numel() == G * N and x.shape[1] == G * K and x.is_contiguous()
        self = cls.__new__(cls)
        self.lib = L.load()
        self.h = L.vp()
        with torch.cuda.device(qweight.device):
            L.check(self.lib.pia_gemm_plan_create_grouped_fp8(_p(qweight), _p(scale), G, N, K, _p(x), x.shape[0],
                                                              C.byref(self.h)))
        self.splits, self.N, self.weight, self._keep = 1, N, qweight, (qweight, scale, x)
        self.out = torch.empty((G, x.shape[0], N), dtype=torch.bfloat16, device=x.device)
        return self

    def set_pdl(self, on=True):
        L.check(self.lib.pia_gemm_plan_set_pdl(self.h, int(on)))
        return self

    def set_silu(self, on=True):
        L.check(self.lib.pia_gemm_plan_set_silu(self.h, int(on)))
        return self

    def set_relu(self, on=True):
        """fp8 plans with bf16 outputs: ReLU after the bias, before the one bf16 rounding (pia_gemm_plan_set_relu)"""
        L.check(self.lib.pia_gemm_plan_set_relu(self.h, int(on)))
        return self

    def run(self, rows=64, out=None):
        o = out if out is not None else self.out
        L.check(self.lib.pia_gemm_run(self.h, rows, _p(o), _s()))
        return o

    def __del__(self):
        try:
            if self.h:
                self.lib.pia_gemm_plan_destroy(self.h)
                self.h = None
        except Exception:
            pass


class Slots(object):
    """pia_slots_t: the request slots of one verify step.  `n`, `prefix_len`, `pad_len` are int32 DEVICE tensors of
    `batch` entries read when the kernels run (so one CUDA graph serves every length / padding); slot s owns rows
    [s * rows_per_slot, (s + 1) * rows_per_slot) of the activation and draft buffers and the KV cache that starts
    kv_slot_stride elements after slot s-1's (0: all slots share one cache, e.g. the chain chunks of a prefill pass)."""

    def __init__(self, n, prefix_len, pad_len=None, rows_per_slot=64, kv_slot_stride=0, batch=None, kv_first_slot=0):
        batch = int(batch if batch is not None else n.numel())
        assert n.dtype == torch.int32 and prefix_len.dtype == torch.int32 and n.numel() >= batch <= prefix_len.numel()
        assert pad_len is None or (pad_len.dtype == torch.int32 and pad_len.numel() >= batch)
        self.batch, self.rows_per_slot, self.kv_slot_stride = batch, int(rows_per_slot), int(kv_slot_stride)
        self.n, self.prefix_len, self.pad_len = n, prefix_len, pad_len
        self.kv_first_slot = int(kv_first_slot)
        self.c = L.Slots(batch, int(rows_per_slot), _p(n), _p(prefix_len), _p(pad_len), int(kv_slot_stride),
                         int(kv_first_slot))

    @property
    def rows(self):
        return self.batch * self.rows_per_slot

    def ref(self):
        return C.byref(self.c)


def rope_kv_append(qkv, mask, slots, n_q_heads, n_kv_heads, head_dim, cos, sin, q_out, k_layer, v_layer, max_seq,
                   rotary_dim=None, q_scale=None):
    """qkv / q_out: >= slots.rows rows; mask: [>= slots.rows, W] int64 ancestor rows; k_layer / v_layer: the layer's
    [n_kv_heads, max_seq, head_dim] planes of slot 0.  rotary_dim=None: Llama RoPE over the whole head (tables
    [max_pos, head_dim/2]); an int: GLM RoPE, interleaved pairs over the first rotary_dim dims (tables
    [max_pos, rotary_dim/2]), the rest passed through (pia_rope_interleaved_kv_append).  float32 tables (Llama layout
    only): fp32 arithmetic, one bf16 rounding (pia_rope_f32_kv_append, Baichuan2-7B).  q_scale: a bf16 [max_pos]
    table the rotated queries are multiplied by at their positions, in bf16 (Qwen's log-n scaling,
    pia_rope_f32_logn_kv_append; float32 tables only)"""
    assert qkv.shape[0] >= slots.rows and mask.shape[0] >= slots.rows
    assert cos.dtype == sin.dtype and cos.dtype in (torch.bfloat16, torch.float32)
    L_ = L.load()
    args = (_p(qkv), _p(mask), mask.shape[-1], slots.ref(), n_q_heads, n_kv_heads, head_dim, _p(cos), _p(sin),
            cos.shape[0], _p(q_out), _p(k_layer), _p(v_layer), max_seq)
    if q_scale is not None:
        if cos.dtype != torch.float32 or rotary_dim is not None:
            raise ValueError('log-n query scaling exists for the fp32 half-split (Qwen) RoPE only')
        if q_scale.dtype != torch.bfloat16 or q_scale.dim() != 1 or q_scale.shape[0] < cos.shape[0]:
            raise ValueError(f'q_scale must be bf16 [>= {cos.shape[0]}] (one entry per table position), got '
                             f'{q_scale.dtype} {tuple(q_scale.shape)}')
        L.check(L_.pia_rope_f32_logn_kv_append(*args, _p(q_scale), _s()))
    elif cos.dtype == torch.float32:
        if rotary_dim is not None:
            raise ValueError('fp32 RoPE tables exist for the half-split (Llama) layout only')
        L.check(L_.pia_rope_f32_kv_append(*args, _s()))
    elif rotary_dim is None:
        L.check(L_.pia_rope_kv_append(*args, _s()))
    else:
        L.check(L_.pia_rope_interleaved_kv_append(*args, int(rotary_dim), _s()))


def kv_append(qkv, mask, slots, n_q_heads, n_kv_heads, src_head_dim, head_dim, q_mul, q_out, k_layer, v_layer,
              max_seq):
    """the KV append without rotation (OPT, pia_kv_append_qscale): qkv [>= slots.rows, (Hq + 2 Hkv) * src_head_dim];
    q_out [rows, Hq, head_dim] gets bf16(q * q_mul), K / V go to the cache rows unchanged; columns [src_head_dim,
    head_dim) of q / K / V are written as zeros"""
    assert qkv.shape[0] >= slots.rows and mask.shape[0] >= slots.rows
    assert qkv.shape[-1] == (n_q_heads + 2 * n_kv_heads) * src_head_dim and qkv.is_contiguous()
    L.check(L.load().pia_kv_append_qscale(_p(qkv), _p(mask), mask.shape[-1], slots.ref(), n_q_heads, n_kv_heads,
                                          int(src_head_dim), int(head_dim), float(q_mul), _p(q_out), _p(k_layer),
                                          _p(v_layer), max_seq, _s()))


def learned_pos_embed(tok_table, ids, pos_table, offset, mask, slots, out):
    """out[i] = bf16(a[i] + pos_table[offset + pos_i]) at the rows' tree positions, pos_i clamped to
    [0, pos_table.shape[0] - offset); a[i] = tok_table[ids[i]], or out[i] itself when tok_table is None
    (pia_learned_pos_embed).  Rows past their slot's n are zeroed."""
    hidden = out.shape[-1]
    assert pos_table.shape[-1] == hidden and pos_table.shape[0] > offset and out.shape[0] >= slots.rows
    assert tok_table is None or (tok_table.shape[-1] == hidden and ids.shape[0] >= slots.rows)
    assert mask.shape[0] >= slots.rows
    L.check(L.load().pia_learned_pos_embed(_p(tok_table), _p(ids) if tok_table is not None else None, _p(pos_table),
                                           int(offset), pos_table.shape[0] - int(offset), _p(mask), mask.shape[-1],
                                           slots.ref(), hidden, _p(out), _s()))


def _alibi_slopes_f64(n):
    """the ALiBi slopes of n heads as python floats (baichuan_13b/modeling_baichuan.py:25-36 `_get_interleave`, the
    same numbers as BLOOM's build_alibi_tensor): the geometric series start^(i+1), start = 2^(-8/n), for a power of
    two n; otherwise that series for the largest power of two c < n, then every other slope of the 2c series"""
    def pow2(m):
        start = 2 ** (-(2 ** -(math.log2(m) - 3)))
        return [start * start ** i for i in range(m)]
    if math.log2(n).is_integer():
        return pow2(n)
    c = 2 ** math.floor(math.log2(n))
    return pow2(c) + _alibi_slopes_f64(2 * c)[0::2][:n - c]


def alibi_slopes(n_heads):
    """fp32 [n_heads] CPU tensor of the ALiBi slopes, computed in float64 and then cast"""
    if int(n_heads) < 1:
        raise ValueError(f'n_heads={n_heads}: ALiBi needs at least one head')
    return torch.tensor(_alibi_slopes_f64(int(n_heads)), dtype=torch.float64).to(torch.float32)


def silu_mul(gate_up, out):
    rows, two_inter = gate_up.shape
    L.check(L.load().pia_silu_mul(_p(gate_up), rows, two_inter // 2, _p(out), _s()))


def moe_combine(expert_out, weights, out):
    """out[t] = sum_e expert_out[e, t] * weights[t, e] in expert order, bf16 rounding per step (pia_moe_combine)"""
    E, rows_cap, hidden = expert_out.shape
    rows = weights.shape[0]
    assert weights.shape[1] == E and weights.is_contiguous() and expert_out.is_contiguous() and out.shape[0] >= rows
    L.check(L.load().pia_moe_combine(_p(expert_out), _p(weights), E, rows, rows_cap, hidden, _p(out), _s()))


def moe_router(y, gate_weight, top_k, dense_out):
    """dense routing weights [rows, E] (0 for unselected experts) of the rows of y (pia_moe_router)"""
    rows, hidden = y.shape
    E = gate_weight.shape[0]
    assert gate_weight.shape[1] == hidden and dense_out.shape[0] >= rows and dense_out.shape[1] == E
    assert y.is_contiguous() and gate_weight.is_contiguous() and dense_out.is_contiguous()
    L.check(L.load().pia_moe_router(_p(y), _p(gate_weight), rows, hidden, E, int(top_k), _p(dense_out), _s()))


def l2_prefetch(t, n_ranges=1, stride_bytes=0, range_bytes=None, gbytes_per_s=0.0, offset_bytes=0):
    """hint: pull (part of) an immutable weight tensor into L2 on the current stream (pia_l2_prefetch)"""
    if range_bytes is None:
        range_bytes = t.numel() * t.element_size() - offset_bytes
    L.check(L.load().pia_l2_prefetch(t.data_ptr() + offset_bytes, int(n_ranges), int(stride_bytes), int(range_bytes),
                                     float(gbytes_per_s), _s()))


def embed_gather(table, ids, n, out):
    rows, hidden = out.shape
    L.check(L.load().pia_embed_gather(_p(table), _p(ids), _p(n), rows, hidden, _p(out), _s()))


class AttnPlan(object):
    """pia_attn_plan_t: TMA descriptors over one model's KV cache(s) (KV splits merge on chip: no workspace).
    k_cache / v_cache: [n_layers, n_kv_heads, max_seq, head_dim], or [n_slots, ...] for the batched loop"""

    def __init__(self, k_cache, v_cache, n_q_heads, n_kv_heads, head_dim, max_nodes, kv_split_max=0):
        n_slots = k_cache.shape[0] if k_cache.dim() == 5 else 1
        n_layers, hkv, max_seq, hd = k_cache.shape[-4:]
        assert hkv == n_kv_heads and hd == head_dim and k_cache.is_contiguous() and v_cache.is_contiguous()
        self.cfg = L.AttnConfig(n_q_heads, n_kv_heads, head_dim, max_seq, max_nodes, n_layers, kv_split_max, n_slots)
        self.slot_stride = n_layers * hkv * max_seq * hd
        self.h = L.vp()
        self.lib = L.load()
        with torch.cuda.device(k_cache.device):
            L.check(self.lib.pia_attn_plan_create(C.byref(self.cfg), _p(k_cache), _p(v_cache), C.byref(self.h)))
        self._keep = (k_cache, v_cache)

    def forward(self, layer, q, mask, slots, out, scale_mul=1.0, alibi_slopes=None):
        """alibi_slopes: None, or an fp32 device tensor [n_q_heads] -> the ALiBi bias at tree positions
        (pia_tree_attn_alibi_fwd, head_dim 128)"""
        assert q.shape[0] >= slots.rows and mask.shape[0] >= slots.rows and out.shape[0] >= slots.rows
        if alibi_slopes is None:
            L.check(self.lib.pia_tree_attn_fwd(self.h, layer, _p(q), _p(mask), slots.ref(), float(scale_mul), _p(out),
                                               _s()))
            return
        assert alibi_slopes.dtype == torch.float32 and alibi_slopes.numel() == self.cfg.n_q_heads and \
            alibi_slopes.is_cuda and alibi_slopes.is_contiguous()
        L.check(self.lib.pia_tree_attn_alibi_fwd(self.h, layer, _p(q), _p(mask), slots.ref(), float(scale_mul),
                                                 _p(alibi_slopes), _p(out), _s()))

    def forward_fused(self, layer, qkv, mask, slots, cos, sin, out, scale_mul=1.0):
        """RoPE + KV append + tree attention in one launch (pia_tree_attn_fused_fwd): qkv is the fused projection
        output; needs one cache per slot"""
        assert qkv.shape[0] >= slots.rows and mask.shape[0] >= slots.rows and out.shape[0] >= slots.rows
        L.check(self.lib.pia_tree_attn_fused_fwd(self.h, layer, _p(qkv), _p(cos), _p(sin), cos.shape[0], _p(mask),
                                                 slots.ref(), float(scale_mul), _p(out), _s()))

    def close(self):
        if self.h:
            self.lib.pia_attn_plan_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Accept(object):
    """pia_accept + its config/workspace.  max_length is a device scalar (d_max_length) when given, so that one
    captured step serves every request length."""

    def __init__(self, vocab, max_nodes, repetition_penalty, eos_ids, max_length, device, bound_walk=False):
        eos = [int(e) for e in (eos_ids or []) if e is not None][:8]
        arr = (C.c_int32 * 8)(*(eos + [-1] * (8 - len(eos))))
        # the reciprocal in double, rounded once to fp32: what RepetitionPenaltyLogitsProcessor's score / penalty
        # multiplies by on CUDA
        self.cfg = L.AcceptConfig(vocab, max_nodes, float(repetition_penalty), len(eos), arr, int(max_length),
                                  int(bool(bound_walk)),
                                  1.0 / float(repetition_penalty) if repetition_penalty > 0 else 0.0)
        self.max_nodes = max_nodes
        self.lib = L.load()
        self.workspace = torch.empty((max(self.lib.pia_accept_workspace_bytes(C.byref(self.cfg)) // 4, 1),),
                                     dtype=torch.int32, device=device)

    def run(self, logits, ids, mask, n, seq, seq_len, acc_tokens, acc_count, acc_nodes, prefix_len, finished,
            batch=1, rows_per_slot=None, max_length=None, rng=None):
        """ids [batch * rows_per_slot], mask [batch * rows_per_slot, W], n / seq_len / prefix_len / finished /
        acc_count [batch], seq [batch, stride] (or 1-D for one slot), acc_tokens / acc_nodes [batch, max_nodes];
        max_length: optional int32 device scalar overriding the config's; rng: None (greedy) or an int32 device
        tensor {seed, counter} -> multinomial accept (do_sample)"""
        rps = int(rows_per_slot if rows_per_slot is not None else self.max_nodes // batch)
        stride = seq.shape[-1] if seq.dim() == 2 else seq.numel()
        L.check(self.lib.pia_accept(C.byref(self.cfg), _p(logits), _p(ids), _p(mask), mask.shape[-1], int(batch), rps,
                                    _p(n), _p(seq), _p(seq_len), int(stride), _p(max_length), _p(rng), _p(acc_tokens),
                                    _p(acc_count), _p(acc_nodes), _p(prefix_len), _p(finished), _p(self.workspace), _s()))


def kv_compact(k_cache, v_cache, acc_nodes, acc_count, prefix_len, batch=1):
    """k_cache / v_cache [n_layers, Hkv, S, D] (batch 1) or [batch_cap, n_layers, Hkv, S, D]"""
    n_layers, hkv, max_seq, hd = k_cache.shape[-4:]
    stride = n_layers * hkv * max_seq * hd if k_cache.dim() == 5 else 0
    nodes_stride = acc_nodes.shape[-1] if acc_nodes.dim() == 2 else acc_nodes.numel()
    L.check(L.load().pia_kv_compact(_p(k_cache), _p(v_cache), n_layers, hkv, max_seq, hd, int(batch), int(stride),
                                    _p(acc_nodes), int(nodes_stride), _p(acc_count), _p(prefix_len), _s()))


def launch_count():
    return int(L.load().pia_launch_count())
