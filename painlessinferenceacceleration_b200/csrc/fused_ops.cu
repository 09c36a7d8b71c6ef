// Elementwise pieces of the LOOKAHEAD verify forward (sm_90a), all HBM-bound, 16-byte vectorised:
//   k_rmsnorm           models/llama/modeling_llama.py:76-90   (+ the residual add of the decoder layer :340-352), in
//                       the rounding of the family's own norm (one or two bf16 roundings, see k_rmsnorm)
//   k_rope_kv_append    :156-169 apply_rotary_pos_emb at the tree positions of :587, and the KV-cache append
//                       that replaces the reference's per-step torch.cat (:265-268); a second instance rotates in
//                       the GLM layout (chatglm/modeling_chatglm.py:156-169, positions :815), a third one in fp32
//                       with fp32 tables (baichuan2_7b/modeling_baichuan.py:148-155), a fourth one without rotation
//                       and with OPT's pre-scaled query (opt/modeling_opt.py:175)
//   k_silu_mul          :185-186
//   k_embed_gather      :582
//   k_learned_pos_embed opt/modeling_opt.py:109-121, :663 learned positions at tree positions
//   k_layernorm         bloom/modeling_bloom.py LayerNorm with weight and bias (+ the residual add, dropout_add)
//   k_bloom_gelu        bloom/modeling_bloom.py:194-203 bloom_gelu_forward
// Rounding points follow the reference's bf16 eager arithmetic (each torch op rounds to bf16) so that
// the verify logits stay as close to the reference's as a different GEMM order allows.
#include <cuda_bf16.h>

#include "common.cuh"

namespace pia {
namespace fused {

__device__ __forceinline__ float bf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

union Pack8 { uint4 u; __nv_bfloat16 h[8]; };

// one CTA per row; hidden % 8 == 0
// x comes either as bf16 [rows, hidden] or as `n_parts` fp32 split-K slices [n_parts][part_rows][hidden] of the
// producing GEMM (summed in slice order and rounded to bf16 first, i.e. what a bf16 GEMM output would hold)
__device__ __forceinline__ Pack8 load_x8(const __nv_bfloat16 *x, const float *parts, int n_parts, long long part_stride,
                                         long long off) {
  Pack8 a;
  if (parts == nullptr) { a.u = *reinterpret_cast<const uint4 *>(x + off); return a; }
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int s = 0; s < n_parts; ++s) {
    const float4 lo = *reinterpret_cast<const float4 *>(parts + s * part_stride + off);
    const float4 hi = *reinterpret_cast<const float4 *>(parts + s * part_stride + off + 4);
    acc[0] += lo.x; acc[1] += lo.y; acc[2] += lo.z; acc[3] += lo.w;
    acc[4] += hi.x; acc[5] += hi.y; acc[6] += hi.z; acc[7] += hi.w;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) a.h[j] = __float2bfloat16_rn(acc[j]);
  return a;
}

// the whole row stays in registers: at most kRmsVec 16-byte vectors per thread, hidden <= 512 * 8 * kRmsVec = 16384.
// Thread t owns vectors t, t + 512, ...; its squares are summed serially in that order, then over the warp (5 shuffle
// levels) and over the 16 warps (serially, warp order).
// kRoundTwice selects where the normalised value x_hat = x * rsqrt(mean(x^2) + eps) is rounded:
//   false: y = bf16(w * x_hat)        (llama/modeling_llama.py:90, chatglm/modeling_chatglm.py:187)
//   true:  y = bf16(w * bf16(x_hat))  (mistral/modeling_mistral.py:90, qwen2/modeling_qwen2.py:96, Baichuan, GLM HF)
// The product of two bf16 values is exact in fp32, so the second form has one more rounding and no other difference.
constexpr int kRmsVec = 4;
constexpr int kRmsMaxHidden = 512 * 8 * kRmsVec;

template <bool kRoundTwice>
__global__ void __launch_bounds__(512) k_rmsnorm(const __nv_bfloat16 *x, const float *parts, int n_parts,
                                                 long long part_stride, const __nv_bfloat16 *res_in,
                                                 const __nv_bfloat16 *w, float eps, int hidden,
                                                 __nv_bfloat16 *res_out, __nv_bfloat16 *y) {
  __shared__ float red[16];
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int nvec = hidden >> 3;
  const long long row_off = (long long)row * hidden;
  const uint4 *rv = res_in ? reinterpret_cast<const uint4 *>(res_in + row_off) : nullptr;
  uint4 *rov = res_out ? reinterpret_cast<uint4 *>(res_out + row_off) : nullptr;
  float ss = 0.f;
  // res_in may alias res_out (the decoder layer updates its residual in place): each vector is read before it is
  // written, by the same thread, and never read again
  Pack8 keep[kRmsVec];
#pragma unroll
  for (int k = 0; k < kRmsVec; ++k) {
    const int v = tid + k * 512;
    if (v < nvec) {
      Pack8 a = load_x8(x, parts, n_parts, part_stride, row_off + v * 8);
      if (rv) {
        Pack8 r; r.u = rv[v];
#pragma unroll
        for (int j = 0; j < 8; ++j) a.h[j] = __float2bfloat16_rn(__bfloat162float(a.h[j]) + __bfloat162float(r.h[j]));
      }
      if (rov) rov[v] = a.u;
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float f = __bfloat162float(a.h[j]); ss += f * f; }
      keep[k] = a;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(FULL, ss, o);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) tot += red[i];
  const float inv = rsqrtf(tot / (float)hidden + eps);
  const uint4 *wv = reinterpret_cast<const uint4 *>(w);
  uint4 *yv = reinterpret_cast<uint4 *>(y + row_off);
#pragma unroll
  for (int k = 0; k < kRmsVec; ++k) {
    const int v = tid + k * 512;
    if (v < nvec) {
      Pack8 ww; ww.u = wv[v];
      Pack8 o;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = __bfloat162float(keep[k].h[j]) * inv;
        o.h[j] = __float2bfloat16_rn(__bfloat162float(ww.h[j]) * (kRoundTwice ? bf(xh) : xh));
      }
      yv[v] = o.u;
    }
  }
}

// grid = batch * rows_per_slot rows (pia_slots_t); thread = one (head, 8-wide d chunk) of q | k | v
// ROPE_HALF:        Llama layout, x[d] pairs with x[d +- hd/2] over the whole head, bf16 tables [max_pos, hd/2]
//                   (rotary_dim unused).
// ROPE_INTERLEAVED: GLM layout (chatglm/modeling_chatglm.py:156-169): only d < rotary_dim rotates, in pairs
//                   (2i, 2i+1) with frequency i, bf16 tables [max_pos, rotary_dim/2]; the other dims pass through.
// ROPE_HALF_F32:    Llama layout with fp32 tables [max_pos, hd/2] and fp32 arithmetic, one bf16 rounding at the end
//                   (baichuan2_7b/modeling_baichuan.py:148-155: q.float() * cos + rotate_half(q.float()) * sin).
// kLogn (ROPE_HALF_F32 only): Qwen's log-n attention scaling (qwen/modeling_qwen.py:374-380), every rotated q element
//                   times q_scale[pos] in bf16 arithmetic, bf16(float(bf16(rot)) * float(q_scale[pos])); K / V untouched.
// ROPE_NONE:        no rotation and no tables (OPT, opt/modeling_opt.py:175): q is written as bf16(float(q) * q_mul),
//                   one rounding of the bf16 projection output, K / V are appended unchanged.  The source rows hold
//                   heads of hd_src <= hd elements ([rows, (hq + 2 hkv) * hd_src]); q / K / V are written hd wide, the
//                   columns [hd_src, hd) zero.
enum { ROPE_HALF = 0, ROPE_INTERLEAVED = 1, ROPE_HALF_F32 = 2, ROPE_NONE = 3 };

// the tree position of activation row i: rowsum(attention_mask) - 1 (modeling_llama.py:587), i.e. the visible prefix
// keys [pad_len, P) of its slot + its visible draft keys - 1, clamped to [0, max_pos)
__device__ __forceinline__ int tree_pos(const unsigned long long *mask, int mask_words, int i, int P, int pad_len,
                                        int max_pos) {
  int depth = -1;
  for (int w = 0; w < mask_words; ++w) depth += __popcll(mask[(long long)i * mask_words + w]);
  int pos = (P > pad_len ? P - pad_len : 0) + depth;
  if (pos < 0) pos = 0;
  if (pos >= max_pos) pos = max_pos - 1;
  return pos;
}

template <int kLayout, bool kLogn = false>
__global__ void __launch_bounds__(256) k_rope_kv_append(const __nv_bfloat16 *qkv, const unsigned long long *mask,
                                                        int mask_words, pia_slots_t sl,
                                                        int hq, int hkv, int hd, const void *cos_t,
                                                        const void *sin_t, int max_pos, __nv_bfloat16 *q_out,
                                                        __nv_bfloat16 *kc, __nv_bfloat16 *vc, int max_seq,
                                                        int rotary_dim, const __nv_bfloat16 *q_scale, int hd_src,
                                                        float q_mul) {
  static_assert(!kLogn || kLayout == ROPE_HALF_F32, "log-n scaling is built on the fp32 layout only");
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x;                       // activation row
  const int slot = i / sl.rows_per_slot, node = i % sl.rows_per_slot;
  const int n = sl.d_n[slot], P = sl.d_prefix_len[slot];
  const int pad_len = sl.d_pad_len ? sl.d_pad_len[slot] : 0;
  if (node >= n) return;
  kc += (long long)slot * sl.kv_slot_stride;
  vc += (long long)slot * sl.kv_slot_stride;
  if constexpr (kLayout == ROPE_NONE) {
    const int cpr = hd >> 3, cache_row = P + node;
    const __nv_bfloat16 *src = qkv + (long long)i * (hq + 2 * hkv) * hd_src;
    for (int c = threadIdx.x; c < (hq + 2 * hkv) * cpr; c += blockDim.x) {
      const int head = c / cpr, d0 = (c % cpr) * 8;
      Pack8 a;
      a.u = d0 < hd_src ? *reinterpret_cast<const uint4 *>(src + head * hd_src + d0) : make_uint4(0, 0, 0, 0);
      if (head < hq) {
#pragma unroll
        for (int j = 0; j < 8; ++j) a.h[j] = __float2bfloat16_rn(__fmul_rn(__bfloat162float(a.h[j]), q_mul));
        *reinterpret_cast<uint4 *>(q_out + ((long long)i * hq + head) * hd + d0) = a.u;
      } else if (head < hq + hkv) {
        *reinterpret_cast<uint4 *>(kc + ((long long)(head - hq) * max_seq + cache_row) * hd + d0) = a.u;
      } else {
        *reinterpret_cast<uint4 *>(vc + ((long long)(head - hq - hkv) * max_seq + cache_row) * hd + d0) = a.u;
      }
    }
    return;
  }
  const int pos = tree_pos(mask, mask_words, i, P, pad_len, max_pos);
  const int half = hd >> 1, cpr = hd >> 3;  // 16-byte chunks per head row
  const int row_elems = (hq + 2 * hkv) * hd;
  const __nv_bfloat16 *src = qkv + (long long)i * row_elems;
  const int cache_row = P + node;
  const int total = (hq + 2 * hkv) * cpr;
  for (int c = threadIdx.x; c < total; c += blockDim.x) {
    const int head = c / cpr, ch = c % cpr;
    const int d0 = ch * 8;
    Pack8 a; a.u = *reinterpret_cast<const uint4 *>(src + head * hd + d0);
    if (head < hq + hkv) {  // q or k: x*cos + rotate_half(x)*sin, every product/sum rounded to bf16 like eager torch
      Pack8 o;
      const __nv_bfloat16 *cos_b = static_cast<const __nv_bfloat16 *>(cos_t);
      const __nv_bfloat16 *sin_b = static_cast<const __nv_bfloat16 *>(sin_t);
      if constexpr (kLayout == ROPE_INTERLEAVED) {
        o = a;
        if (d0 < rotary_dim) {  // 4 whole pairs (2i, 2i+1), i = d0/2 .. d0/2+3: cos/sin are one 8-byte load each
          const int rhalf = rotary_dim >> 1;
          union { uint2 u; __nv_bfloat16 h[4]; } cs, sn;
          cs.u = *reinterpret_cast<const uint2 *>(cos_b + (long long)pos * rhalf + (d0 >> 1));
          sn.u = *reinterpret_cast<const uint2 *>(sin_b + (long long)pos * rhalf + (d0 >> 1));
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float x0 = __bfloat162float(a.h[2 * j]), x1 = __bfloat162float(a.h[2 * j + 1]);
            const float c = __bfloat162float(cs.h[j]), s = __bfloat162float(sn.h[j]);
            o.h[2 * j] = __float2bfloat16_rn(bf(x0 * c) + bf(-x1 * s));
            o.h[2 * j + 1] = __float2bfloat16_rn(bf(x1 * c) + bf(x0 * s));
          }
        }
      } else if constexpr (kLayout == ROPE_HALF_F32) {
        const int dp = d0 < half ? d0 + half : d0 - half;
        Pack8 b; b.u = *reinterpret_cast<const uint4 *>(src + head * hd + dp);
        const float *cf = static_cast<const float *>(cos_t) + (long long)pos * half + d0 % half;
        const float *sf = static_cast<const float *>(sin_t) + (long long)pos * half + d0 % half;
        float c[8], s[8];
        *reinterpret_cast<float4 *>(c) = *reinterpret_cast<const float4 *>(cf);
        *reinterpret_cast<float4 *>(c + 4) = *reinterpret_cast<const float4 *>(cf + 4);
        *reinterpret_cast<float4 *>(s) = *reinterpret_cast<const float4 *>(sf);
        *reinterpret_cast<float4 *>(s + 4) = *reinterpret_cast<const float4 *>(sf + 4);
#pragma unroll
        for (int j = 0; j < 8; ++j) {  // fp32 products and sum, no FMA contraction, one rounding to bf16
          const float x = __bfloat162float(a.h[j]);
          const float r = d0 < half ? -__bfloat162float(b.h[j]) : __bfloat162float(b.h[j]);
          o.h[j] = __float2bfloat16_rn(__fadd_rn(__fmul_rn(x, c[j]), __fmul_rn(r, s[j])));
        }
        if constexpr (kLogn) {
          if (head < hq) {  // query * logn_tensor: a bf16 product of the rounded rotation and the bf16 table entry
            const float sc = __bfloat162float(q_scale[pos]);
#pragma unroll
            for (int j = 0; j < 8; ++j) o.h[j] = __float2bfloat16_rn(__fmul_rn(__bfloat162float(o.h[j]), sc));
          }
        }
      } else {
        const int dp = d0 < half ? d0 + half : d0 - half;
        Pack8 b; b.u = *reinterpret_cast<const uint4 *>(src + head * hd + dp);
        Pack8 cs, sn;
        const int f0 = d0 % half;
        cs.u = *reinterpret_cast<const uint4 *>(cos_b + (long long)pos * half + f0);
        sn.u = *reinterpret_cast<const uint4 *>(sin_b + (long long)pos * half + f0);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float x = __bfloat162float(a.h[j]);
          const float r = d0 < half ? -__bfloat162float(b.h[j]) : __bfloat162float(b.h[j]);
          o.h[j] = __float2bfloat16_rn(bf(x * __bfloat162float(cs.h[j])) + bf(r * __bfloat162float(sn.h[j])));
        }
      }
      if (head < hq) *reinterpret_cast<uint4 *>(q_out + ((long long)i * hq + head) * hd + d0) = o.u;
      else *reinterpret_cast<uint4 *>(kc + ((long long)(head - hq) * max_seq + cache_row) * hd + d0) = o.u;
    } else {
      *reinterpret_cast<uint4 *>(vc + ((long long)(head - hq - hkv) * max_seq + cache_row) * hd + d0) = a.u;
    }
  }
}

__global__ void __launch_bounds__(256) k_silu_mul(const __nv_bfloat16 *gu, int inter, __nv_bfloat16 *out) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.y;
  const int v = blockIdx.x * 256 + threadIdx.x;
  if (v * 8 >= inter) return;
  Pack8 g, u, o;
  g.u = *reinterpret_cast<const uint4 *>(gu + (long long)row * 2 * inter + v * 8);
  u.u = *reinterpret_cast<const uint4 *>(gu + (long long)row * 2 * inter + inter + v * 8);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float x = __bfloat162float(g.h[j]);
    const float s = bf(x / (1.f + expf(-x)));
    o.h[j] = __float2bfloat16_rn(s * __bfloat162float(u.h[j]));
  }
  *reinterpret_cast<uint4 *>(out + (long long)row * inter + v * 8) = o.u;
}

__global__ void __launch_bounds__(256) k_embed_gather(const __nv_bfloat16 *table, const int *ids, const int *d_n,
                                                      int hidden, __nv_bfloat16 *out) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  const int n = *d_n;
  const int nvec = hidden >> 3;
  uint4 *dst = reinterpret_cast<uint4 *>(out + (long long)row * hidden);
  if (row >= n) { for (int v = threadIdx.x; v < nvec; v += 256) dst[v] = make_uint4(0, 0, 0, 0); return; }
  const uint4 *src = reinterpret_cast<const uint4 *>(table + (long long)ids[row] * hidden);
  for (int v = threadIdx.x; v < nvec; v += 256) dst[v] = src[v];
}

// learned absolute positions at tree positions (OPT, opt/modeling_opt.py:109-121 and :663): out[i] = bf16(a[i] +
// pos_table[offset + pos(i)]), one rounding of the bf16 + bf16 sum as eager `inputs_embeds + pos_embeds`; pos(i) is
// k_rope_kv_append's tree position, clamped to [0, max_pos).  a[i] = tok[ids[i]], or out[i] itself when tok is null
// (the row already holds project_in's output).  grid = slot rows; rows past their slot's n are zero, as in
// k_embed_gather.
__global__ void __launch_bounds__(256) k_learned_pos_embed(const __nv_bfloat16 *tok, const int *ids,
                                                           const __nv_bfloat16 *pos_table, int offset, int max_pos,
                                                           const unsigned long long *mask, int mask_words,
                                                           pia_slots_t sl, int hidden, __nv_bfloat16 *out) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x;
  const int slot = i / sl.rows_per_slot, node = i % sl.rows_per_slot;
  const int nvec = hidden >> 3;
  uint4 *dst = reinterpret_cast<uint4 *>(out + (long long)i * hidden);
  if (node >= sl.d_n[slot]) { for (int v = threadIdx.x; v < nvec; v += 256) dst[v] = make_uint4(0, 0, 0, 0); return; }
  const int pos = tree_pos(mask, mask_words, i, sl.d_prefix_len[slot], sl.d_pad_len ? sl.d_pad_len[slot] : 0, max_pos);
  const uint4 *src = tok ? reinterpret_cast<const uint4 *>(tok + (long long)ids[i] * hidden) : dst;
  const uint4 *pe = reinterpret_cast<const uint4 *>(pos_table + (long long)(offset + pos) * hidden);
  for (int v = threadIdx.x; v < nvec; v += 256) {
    Pack8 a, p;
    a.u = src[v];
    p.u = pe[v];
#pragma unroll
    for (int j = 0; j < 8; ++j) a.h[j] = __float2bfloat16_rn(__bfloat162float(a.h[j]) + __bfloat162float(p.h[j]));
    dst[v] = a.u;
  }
}

// LayerNorm with weight and bias (bloom/modeling_bloom.py:346-349, :422, :428) over one row per CTA, preceded by the
// residual add of the decoder block (dropout_add, :504 / :539: a bf16 add).  blockDim = min(512, nvec rounded up to a
// warp); the row stays in registers (at most kLnVec 16-byte vectors per thread: hidden <= 512 * 8 * 4 = 16384) and the
// mean and the biased variance are two fp32 passes over them.
constexpr int kLnVec = 4;
constexpr int kLnMaxHidden = 512 * 8 * kLnVec;

__device__ __forceinline__ float block_sum(float v, float *red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float tot = 0.f;
  const int nw = blockDim.x >> 5;
  for (int i = 0; i < nw; ++i) tot += red[i];
  return tot;
}

__global__ void __launch_bounds__(512) k_layernorm(const __nv_bfloat16 *x, const __nv_bfloat16 *res_in,
                                                   const __nv_bfloat16 *w, const __nv_bfloat16 *b, float eps,
                                                   int hidden, __nv_bfloat16 *res_out, __nv_bfloat16 *y) {
  __shared__ float red[2][16];
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int nvec = hidden >> 3;
  const long long row_off = (long long)row * hidden;
  const uint4 *xv = reinterpret_cast<const uint4 *>(x + row_off);
  const uint4 *rv = res_in ? reinterpret_cast<const uint4 *>(res_in + row_off) : nullptr;
  uint4 *rov = res_out ? reinterpret_cast<uint4 *>(res_out + row_off) : nullptr;
  float f[kLnVec][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kLnVec; ++k) {
    const int v = tid + k * blockDim.x;
    if (v < nvec) {
      Pack8 a; a.u = xv[v];
      if (rv) {
        Pack8 r; r.u = rv[v];
#pragma unroll
        for (int j = 0; j < 8; ++j) a.h[j] = __float2bfloat16_rn(__bfloat162float(a.h[j]) + __bfloat162float(r.h[j]));
      }
      if (rov) rov[v] = a.u;
#pragma unroll
      for (int j = 0; j < 8; ++j) { f[k][j] = __bfloat162float(a.h[j]); s += f[k][j]; }
    }
  }
  const float mean = block_sum(s, red[0]) / (float)hidden;
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < kLnVec; ++k) {
    if (tid + k * blockDim.x < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = f[k][j] - mean; ss += d * d; }
    }
  }
  const float rstd = rsqrtf(block_sum(ss, red[1]) / (float)hidden + eps);
  const uint4 *wv = reinterpret_cast<const uint4 *>(w);
  const uint4 *bv = reinterpret_cast<const uint4 *>(b);
  uint4 *yv = reinterpret_cast<uint4 *>(y + row_off);
#pragma unroll
  for (int k = 0; k < kLnVec; ++k) {
    const int v = tid + k * blockDim.x;
    if (v < nvec) {
      Pack8 ww, bb, o;
      ww.u = wv[v];
      bb.u = bv[v];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        o.h[j] = __float2bfloat16_rn((f[k][j] - mean) * rstd * __bfloat162float(ww.h[j]) + __bfloat162float(bb.h[j]));
      yv[v] = o.u;
    }
  }
}

// BLOOM's tanh-GELU (bloom/modeling_bloom.py:194-203)
//   x * 0.5 * (1.0 + tanh(0.79788456 * x * (1 + 0.044715 * x * x)))
// evaluated as eager bf16 torch does: every op computes in fp32 with the Python scalars as fp32 and rounds to bf16.
// Eight elements per thread; n % 8 == 0 and 16-byte aligned buffers.
__device__ __forceinline__ float bloom_gelu1(float x) {
  const float a = bf(x * 0.5f);
  const float c = bf(bf(0.044715f * x) * x);
  const float t = bf(bf(0.79788456f * x) * bf(c + 1.f));
  return a * bf(bf(tanhf(t)) + 1.f);
}

__global__ void __launch_bounds__(256) k_bloom_gelu(const __nv_bfloat16 *in, long long nvec, __nv_bfloat16 *out) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (long long)gridDim.x * blockDim.x) {
    Pack8 a, o;
    a.u = reinterpret_cast<const uint4 *>(in)[v];
#pragma unroll
    for (int j = 0; j < 8; ++j) o.h[j] = __float2bfloat16_rn(bloom_gelu1(__bfloat162float(a.h[j])));
    reinterpret_cast<uint4 *>(out)[v] = o.u;
  }
}

}  // namespace fused
}  // namespace pia

using namespace pia;
using namespace pia::fused;

static int rmsnorm(const void *d_x, const float *d_parts, int n_parts, long long part_stride, const void *d_residual_in,
                   const void *d_weight, float eps, int rounding, int rows, int hidden, void *d_residual_out, void *d_y,
                   void *stream) {
  PIA_REQUIRE(d_weight && d_y && rows > 0 && hidden > 0 && hidden % 8 == 0 && hidden <= kRmsMaxHidden,
              "bad rmsnorm arguments: hidden must be a positive multiple of 8, at most 16384");
  PIA_REQUIRE(rounding == PIA_RMSNORM_ROUND_ONCE || rounding == PIA_RMSNORM_ROUND_TWICE,
              "bad rmsnorm rounding: PIA_RMSNORM_ROUND_ONCE or PIA_RMSNORM_ROUND_TWICE");
  auto kern = rounding == PIA_RMSNORM_ROUND_TWICE ? k_rmsnorm<true> : k_rmsnorm<false>;
  PIA_CUDA_CHECK(launch_kernel(kern, dim3(rows), dim3(512), 0, (cudaStream_t)stream, (const __nv_bfloat16 *)d_x,
                              d_parts, n_parts, part_stride, (const __nv_bfloat16 *)d_residual_in,
                              (const __nv_bfloat16 *)d_weight, eps, hidden, (__nv_bfloat16 *)d_residual_out,
                              (__nv_bfloat16 *)d_y));
  count_launch();
  return PIA_OK;
}

extern "C" int pia_rmsnorm(const void *d_x, const void *d_residual_in, const void *d_weight, float eps, int rounding,
                           int rows, int hidden, void *d_residual_out, void *d_y, void *stream) {
  PIA_REQUIRE(d_x, "bad rmsnorm arguments");
  return rmsnorm(d_x, nullptr, 0, 0ll, d_residual_in, d_weight, eps, rounding, rows, hidden, d_residual_out, d_y,
                 stream);
}

extern "C" int pia_rmsnorm_partials(const float *d_x_parts, int n_parts, int64_t part_stride, const void *d_residual_in,
                                    const void *d_weight, float eps, int rounding, int rows, int hidden,
                                    void *d_residual_out, void *d_y, void *stream) {
  PIA_REQUIRE(d_x_parts && n_parts >= 1, "bad rmsnorm arguments");
  return rmsnorm(nullptr, d_x_parts, n_parts, (long long)part_stride, d_residual_in, d_weight, eps, rounding, rows,
                 hidden, d_residual_out, d_y, stream);
}

template <int kLayout, bool kLogn = false>
static int rope_kv_append(const void *d_qkv, const uint64_t *d_mask, int mask_words, const pia_slots_t *slots,
                          int n_q_heads, int n_kv_heads, int head_dim, const void *d_cos, const void *d_sin, int max_pos,
                          void *d_q_out, void *d_k_cache_layer, void *d_v_cache_layer, int max_seq, int rotary_dim,
                          void *stream, const void *d_q_scale = nullptr, int hd_src = 0, float q_mul = 1.f) {
  PIA_REQUIRE(d_qkv && d_mask && slots && slots->d_n && slots->d_prefix_len && d_q_out && d_k_cache_layer &&
                  d_v_cache_layer && (kLayout == ROPE_NONE || (d_cos && d_sin)), "null argument");
  PIA_REQUIRE(slots->batch >= 1 && slots->rows_per_slot >= 1 && slots->kv_slot_stride >= 0, "bad slot table");
  PIA_REQUIRE(head_dim % 16 == 0 && mask_words >= 1 && mask_words <= 2, "bad rope arguments");
  PIA_REQUIRE(!kLogn || d_q_scale, "null argument");
  PIA_REQUIRE(kLayout != ROPE_NONE || (hd_src >= 8 && hd_src % 8 == 0 && hd_src <= head_dim),
              "bad source head width: a positive multiple of 8, at most head_dim");
  PIA_CUDA_CHECK(launch_kernel(k_rope_kv_append<kLayout, kLogn>, dim3(slots->batch * slots->rows_per_slot), dim3(256), 0,
                              (cudaStream_t)stream, (const __nv_bfloat16 *)d_qkv, (const unsigned long long *)d_mask,
                              mask_words, *slots, n_q_heads, n_kv_heads, head_dim, d_cos, d_sin, max_pos,
                              (__nv_bfloat16 *)d_q_out,
                              (__nv_bfloat16 *)d_k_cache_layer, (__nv_bfloat16 *)d_v_cache_layer, max_seq, rotary_dim,
                              (const __nv_bfloat16 *)d_q_scale, hd_src, q_mul));
  count_launch();
  return PIA_OK;
}

extern "C" int pia_kv_append_qscale(const void *d_qkv, const uint64_t *d_mask, int mask_words, const pia_slots_t *slots,
                                    int n_q_heads, int n_kv_heads, int src_head_dim, int head_dim, float q_mul,
                                    void *d_q_out, void *d_k_cache_layer, void *d_v_cache_layer, int max_seq,
                                    void *stream) {
  return rope_kv_append<ROPE_NONE>(d_qkv, d_mask, mask_words, slots, n_q_heads, n_kv_heads, head_dim, nullptr, nullptr,
                                   1, d_q_out, d_k_cache_layer, d_v_cache_layer, max_seq, head_dim, stream, nullptr,
                                   src_head_dim, q_mul);
}

extern "C" int pia_learned_pos_embed(const void *d_tok_table, const int32_t *d_ids, const void *d_pos_table,
                                     int offset, int max_pos, const uint64_t *d_mask, int mask_words,
                                     const pia_slots_t *slots, int hidden, void *d_out, void *stream) {
  PIA_REQUIRE(d_pos_table && d_mask && slots && slots->d_n && slots->d_prefix_len && d_out &&
                  (d_ids || !d_tok_table), "null argument");
  PIA_REQUIRE(slots->batch >= 1 && slots->rows_per_slot >= 1, "bad slot table");
  PIA_REQUIRE(hidden > 0 && hidden % 8 == 0 && offset >= 0 && max_pos >= 1 && mask_words >= 1 && mask_words <= 2,
              "bad position embedding arguments: hidden a positive multiple of 8, offset >= 0, max_pos >= 1");
  PIA_CUDA_CHECK(launch_kernel(k_learned_pos_embed, dim3(slots->batch * slots->rows_per_slot), dim3(256), 0,
                              (cudaStream_t)stream, (const __nv_bfloat16 *)d_tok_table, (const int *)d_ids,
                              (const __nv_bfloat16 *)d_pos_table, offset, max_pos, (const unsigned long long *)d_mask,
                              mask_words, *slots, hidden, (__nv_bfloat16 *)d_out));
  count_launch();
  return PIA_OK;
}

extern "C" int pia_rope_kv_append(const void *d_qkv, const uint64_t *d_mask, int mask_words, const pia_slots_t *slots,
                                  int n_q_heads, int n_kv_heads, int head_dim, const void *d_cos, const void *d_sin,
                                  int max_pos, void *d_q_out, void *d_k_cache_layer, void *d_v_cache_layer, int max_seq,
                                  void *stream) {
  return rope_kv_append<ROPE_HALF>(d_qkv, d_mask, mask_words, slots, n_q_heads, n_kv_heads, head_dim, d_cos, d_sin,
                                   max_pos, d_q_out, d_k_cache_layer, d_v_cache_layer, max_seq, head_dim, stream);
}

extern "C" int pia_rope_f32_kv_append(const void *d_qkv, const uint64_t *d_mask, int mask_words, const pia_slots_t *slots,
                                      int n_q_heads, int n_kv_heads, int head_dim, const void *d_cos, const void *d_sin,
                                      int max_pos, void *d_q_out, void *d_k_cache_layer, void *d_v_cache_layer,
                                      int max_seq, void *stream) {
  return rope_kv_append<ROPE_HALF_F32>(d_qkv, d_mask, mask_words, slots, n_q_heads, n_kv_heads, head_dim, d_cos, d_sin,
                                       max_pos, d_q_out, d_k_cache_layer, d_v_cache_layer, max_seq, head_dim, stream);
}

extern "C" int pia_rope_f32_logn_kv_append(const void *d_qkv, const uint64_t *d_mask, int mask_words,
                                           const pia_slots_t *slots, int n_q_heads, int n_kv_heads, int head_dim,
                                           const void *d_cos, const void *d_sin, int max_pos, void *d_q_out,
                                           void *d_k_cache_layer, void *d_v_cache_layer, int max_seq,
                                           const void *d_q_scale, void *stream) {
  return rope_kv_append<ROPE_HALF_F32, true>(d_qkv, d_mask, mask_words, slots, n_q_heads, n_kv_heads, head_dim, d_cos,
                                             d_sin, max_pos, d_q_out, d_k_cache_layer, d_v_cache_layer, max_seq,
                                             head_dim, stream, d_q_scale);
}

extern "C" int pia_rope_interleaved_kv_append(const void *d_qkv, const uint64_t *d_mask, int mask_words,
                                              const pia_slots_t *slots, int n_q_heads, int n_kv_heads, int head_dim,
                                              const void *d_cos, const void *d_sin, int max_pos, void *d_q_out,
                                              void *d_k_cache_layer, void *d_v_cache_layer, int max_seq,
                                              int rotary_dim, void *stream) {
  PIA_REQUIRE(rotary_dim >= 8 && rotary_dim % 8 == 0 && rotary_dim <= head_dim,
              "bad rotary_dim: a positive multiple of 8, at most head_dim");
  return rope_kv_append<ROPE_INTERLEAVED>(d_qkv, d_mask, mask_words, slots, n_q_heads, n_kv_heads, head_dim, d_cos, d_sin, max_pos,
                              d_q_out, d_k_cache_layer, d_v_cache_layer, max_seq, rotary_dim, stream);
}

extern "C" int pia_silu_mul(const void *d_gate_up, int rows, int inter, void *d_out, void *stream) {
  PIA_REQUIRE(d_gate_up && d_out && rows > 0 && inter > 0 && inter % 8 == 0, "bad silu_mul arguments");
  dim3 grid((inter / 8 + 255) / 256, rows);
  PIA_CUDA_CHECK(launch_kernel(k_silu_mul, grid, dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16 *)d_gate_up,
                              inter, (__nv_bfloat16 *)d_out));
  count_launch();
  return PIA_OK;
}

extern "C" int pia_layernorm(const void *d_x, const void *d_residual_in, const void *d_weight, const void *d_bias,
                             float eps, int rows, int hidden, void *d_residual_out, void *d_y, void *stream) {
  PIA_REQUIRE(d_x && d_weight && d_bias && d_y && rows > 0 && hidden > 0 && hidden % 8 == 0 && hidden <= kLnMaxHidden,
              "bad layernorm arguments: hidden must be a positive multiple of 8, at most 16384");
  const int nvec = hidden / 8;
  const int threads = nvec >= 512 ? 512 : (nvec + 31) / 32 * 32;
  PIA_CUDA_CHECK(launch_kernel(k_layernorm, dim3(rows), dim3(threads), 0, (cudaStream_t)stream,
                              (const __nv_bfloat16 *)d_x, (const __nv_bfloat16 *)d_residual_in,
                              (const __nv_bfloat16 *)d_weight, (const __nv_bfloat16 *)d_bias, eps, hidden,
                              (__nv_bfloat16 *)d_residual_out, (__nv_bfloat16 *)d_y));
  count_launch();
  return PIA_OK;
}

extern "C" int pia_bloom_gelu(const void *d_in, int64_t n, void *d_out, void *stream) {
  PIA_REQUIRE(d_in && d_out && n > 0 && n % 8 == 0 && ((uintptr_t)d_in & 15) == 0 && ((uintptr_t)d_out & 15) == 0,
              "bad bloom_gelu arguments: n must be a positive multiple of 8, buffers 16-byte aligned");
  const long long nvec = n / 8;
  const long long blocks = (nvec + 255) / 256;
  PIA_CUDA_CHECK(launch_kernel(k_bloom_gelu, dim3((unsigned)(blocks < 65536 ? blocks : 65536)), dim3(256), 0,
                              (cudaStream_t)stream, (const __nv_bfloat16 *)d_in, nvec, (__nv_bfloat16 *)d_out));
  count_launch();
  return PIA_OK;
}

// MoE combine (mixtral/modeling_mixtral.py:734-759 restated densely): out[t] = sum over experts e, in expert-index
// order, of ye[e][t] * w[t][e]; the product and every partial sum are rounded to bf16 like the eager bf16 loop
// (`final_hidden_states.index_add_`), w = 0 for the experts a token did not select.  grid = rows, thread = 8 columns.
// An expert whose weight is 0 is skipped, not added as ye * 0: the reference never evaluates an unselected expert for
// the token, so an inf or NaN in that expert's output must not reach out[t] (inf * 0 = NaN).  For finite outputs the
// skip changes no bit: the accumulator starts at +0, never becomes -0, and adding +-0 leaves it as it is.  It differs
// from the reference only for a selected expert whose bf16 weight underflowed to 0 and whose output is not finite.
__global__ void __launch_bounds__(256) k_moe_combine(const __nv_bfloat16 *ye, const __nv_bfloat16 *w, int n_exp, int rows_cap,
                                                     int hidden, __nv_bfloat16 *out) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  for (int v = threadIdx.x; v * 8 < hidden; v += blockDim.x) {
    Pack8 acc;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc.h[j] = __float2bfloat16_rn(0.f);
    for (int e = 0; e < n_exp; ++e) {
      const float we = __bfloat162float(w[(long long)t * n_exp + e]);
      if (we == 0.f) continue;
      Pack8 y;
      y.u = *reinterpret_cast<const uint4 *>(ye + ((long long)e * rows_cap + t) * hidden + v * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        acc.h[j] = __float2bfloat16_rn(__bfloat162float(acc.h[j]) + bf(__bfloat162float(y.h[j]) * we));
    }
    *reinterpret_cast<uint4 *>(out + (long long)t * hidden + v * 8) = acc.u;
  }
}

extern "C" int pia_moe_combine(const void *d_expert_out, const void *d_weights, int n_experts, int rows, int rows_cap,
                               int hidden, void *d_out, void *stream) {
  PIA_REQUIRE(d_expert_out && d_weights && d_out && n_experts > 0 && rows > 0 && rows <= rows_cap && hidden > 0 &&
                  hidden % 8 == 0, "bad combine arguments");
  PIA_CUDA_CHECK(launch_kernel(k_moe_combine, dim3(rows), dim3(256), 0, (cudaStream_t)stream,
                              (const __nv_bfloat16 *)d_expert_out, (const __nv_bfloat16 *)d_weights, n_experts, rows_cap,
                              hidden, (__nv_bfloat16 *)d_out));
  count_launch();
  return PIA_OK;
}

// MoE router (mixtral/modeling_mixtral.py:721-727): router_logits = gate(hidden) (a bf16 Linear: fp32 accumulation,
// one bf16 rounding), softmax in fp32, top-k, renormalise, cast to bf16; written DENSE: w[t][e] = routing weight or 0 for
// the experts token t did not select (what k_moe_combine and the dense-over-experts verify path consume).
// grid = rows; one warp per expert dot product (round robin), thread 0 does the 8-way softmax / top-k.
__global__ void __launch_bounds__(256) k_moe_router(const __nv_bfloat16 *y, const __nv_bfloat16 *gate_w, int hidden,
                                                    int n_exp, int top_k, __nv_bfloat16 *dense) {
  __shared__ float s_logit[64];
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __nv_bfloat16 *yr = y + (long long)t * hidden;
  for (int e = warp; e < n_exp; e += 8) {
    const __nv_bfloat16 *wr = gate_w + (long long)e * hidden;
    float acc = 0.f;
    for (int v = lane; v * 8 < hidden; v += 32) {
      Pack8 a, w;
      a.u = *reinterpret_cast<const uint4 *>(yr + v * 8);
      w.u = *reinterpret_cast<const uint4 *>(wr + v * 8);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += __bfloat162float(a.h[j]) * __bfloat162float(w.h[j]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL, acc, o);
    if (lane == 0) s_logit[e] = bf(acc);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float mx = -INFINITY;
    for (int e = 0; e < n_exp; ++e) mx = fmaxf(mx, s_logit[e]);
    float den = 0.f, p[64];
    for (int e = 0; e < n_exp; ++e) { p[e] = expf(s_logit[e] - mx); den += p[e]; }
    for (int e = 0; e < n_exp; ++e) p[e] /= den;
    unsigned long long chosen = 0ull;
    float sum = 0.f;
    for (int k = 0; k < top_k; ++k) {   // largest first, lowest index on ties
      int best = -1;
      for (int e = 0; e < n_exp; ++e)
        if (!((chosen >> e) & 1ull) && (best < 0 || p[e] > p[best])) best = e;
      chosen |= 1ull << best;
      sum += p[best];
    }
    for (int e = 0; e < n_exp; ++e)
      dense[(long long)t * n_exp + e] = __float2bfloat16_rn(((chosen >> e) & 1ull) ? p[e] / sum : 0.f);
  }
}

extern "C" int pia_moe_router(const void *d_y, const void *d_gate_weight, int rows, int hidden, int n_experts, int top_k,
                              void *d_dense_out, void *stream) {
  PIA_REQUIRE(d_y && d_gate_weight && d_dense_out && rows > 0 && hidden > 0 && hidden % 8 == 0 && n_experts >= 1 &&
                  n_experts <= 64 && top_k >= 1 && top_k <= n_experts, "bad router arguments");
  PIA_CUDA_CHECK(launch_kernel(k_moe_router, dim3(rows), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16 *)d_y,
                              (const __nv_bfloat16 *)d_gate_weight, hidden, n_experts, top_k, (__nv_bfloat16 *)d_dense_out));
  count_launch();
  return PIA_OK;
}

// One warp per SM walks the ranges chunk by chunk (the bulk-prefetch issue rate of a single SM's TMA unit is only a
// few hundred GB/s, so the chunks are dealt round-robin over the whole grid); bytes_per_ns paces the grid against
// %globaltimer so that the demand loads of the kernels running beside it (attention's KV tiles) are not queued behind
// tens of MB of prefetch.  No shared memory, 32 threads: fits next to any resident CTA.
__global__ void __launch_bounds__(32) k_l2_prefetch(const char *base, long long n_ranges, long long stride,
                                                     long long range_bytes, int chunk, float bytes_per_ns) {
  const long long cpr = (range_bytes + chunk - 1) / chunk;
  const long long total = cpr * n_ranges;
  unsigned long long t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (long long c = (long long)threadIdx.x * gridDim.x + blockIdx.x; c < total; c += (long long)blockDim.x * gridDim.x) {
    const long long k = c / n_ranges, r = c % n_ranges;
    const long long off = k * chunk;
    const long long left = range_bytes - off;
    const unsigned sz = (unsigned)(left < chunk ? left : chunk);
    if (bytes_per_ns > 0.f) {
      const unsigned long long due = t0 + (unsigned long long)((float)(c * chunk) / bytes_per_ns);
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      while (now < due) {
        __nanosleep(64);
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      }
    }
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + r * stride + off), "r"(sz) : "memory");
  }
}

extern "C" int pia_l2_prefetch(const void *d_base, int64_t n_ranges, int64_t stride_bytes, int64_t range_bytes,
                               float gbytes_per_s, void *stream) {
  PIA_REQUIRE(d_base && n_ranges > 0 && range_bytes > 0 && range_bytes % 16 == 0 && ((uintptr_t)d_base & 15) == 0 &&
                  (n_ranges == 1 || (stride_bytes >= range_bytes && stride_bytes % 16 == 0)) && gbytes_per_s >= 0.f,
              "bad prefetch arguments");
  const int chunk = range_bytes < 16384 ? (int)range_bytes : 16384;
  // plain launch (no programmatic dependency): the kernel reads nothing its predecessors write
  static int n_sm = 0;
  if (!n_sm) {
    int dev = 0;
    PIA_CUDA_CHECK(cudaGetDevice(&dev));
    PIA_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
  }
  k_l2_prefetch<<<n_sm, 32, 0, (cudaStream_t)stream>>>((const char *)d_base, (long long)n_ranges, (long long)stride_bytes,
                                                     (long long)range_bytes, chunk, gbytes_per_s);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

extern "C" int pia_embed_gather(const void *d_table, const int32_t *d_ids, const int32_t *d_n, int rows, int hidden,
                                void *d_out, void *stream) {
  PIA_REQUIRE(d_table && d_ids && d_n && d_out && rows > 0 && hidden % 8 == 0, "bad embed arguments");
  PIA_CUDA_CHECK(launch_kernel(k_embed_gather, dim3(rows), dim3(256), 0, (cudaStream_t)stream,
                              (const __nv_bfloat16 *)d_table, (const int *)d_ids, (const int *)d_n, hidden,
                              (__nv_bfloat16 *)d_out));
  count_launch();
  return PIA_OK;
}
