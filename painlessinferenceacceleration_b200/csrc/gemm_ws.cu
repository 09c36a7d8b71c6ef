// Weight-streaming GEMM for the verify forward (sm_90a: TMA + wgmma).
//
//   Y[t, n] = sum_k X[t, k] * W[n, k]        X: [TOK <= 64 draft rows, K] bf16,  W: [N, K] bf16 (nn.Linear weight)
//
// i.e. the q/k/v/o/gate/up/down/lm_head projections of the reference's patched forward
// (models/llama/modeling_llama.py:254-256, :303, :185-186, :769) at the draft's row count.  With <= 64 rows the
// GEMM is a pure weight stream (arithmetic intensity = rows FLOP/B << ridge), so the kernel is built around HBM:
//   * swap-AB: 128 weight rows are the MMA M dimension (two warpgroups x wgmma M = 64), the 64 tokens the N
//     dimension; the fp32 accumulator D[128 x 64] lives in registers (32 per thread), so the big operand (W) is read
//     exactly once and only the small one (X, <= 1.4 MB, L2 resident) is re-read per tile;
//   * one CTA per (128-row weight tile, K split): warps 0-7 = two consumer warpgroups (wgmma.m64n64k16, both operands
//     from shared memory, then the epilogue), warp 8 = TMA producer over an mbarrier ring of {W tile 128x64 (16 KB),
//     X tile 64x64 (8 KB)} SWIZZLE_128B boxes.  ~100 KB of shared memory per CTA so that two CTAs share an SM and
//     one CTA's prologue/epilogue hides behind the other's stream;
//   * projections with few weight tiles (o_proj, down_proj: N = 4096 -> 32 tiles) split K across CTAs and write fp32
//     partial slices that the consumer (k_rmsnorm_partials) sums in a fixed order - deterministic, no atomics.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <new>

#include "common.cuh"

namespace pia {
namespace gemm {

constexpr int BMW = 128;   // weight rows per tile (two wgmma M = 64 halves)
constexpr int BK = 64;     // k elements per stage (one 128-byte swizzle row)
constexpr int TOK = 64;    // token rows (wgmma N)
constexpr int NTHREADS = 288;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int PRODUCER_WARP = 8;
constexpr int W_BYTES = BMW * BK * 2, X_BYTES = TOK * BK * 2, STAGE_BYTES = W_BYTES + X_BYTES;
constexpr int XCH_BYTES = TOK * 64 * 2;  // bf16 [64 tokens][64 rows] exchange tile of the SiLU*up epilogue
constexpr int smem_total(int nstage) { return nstage * STAGE_BYTES + 256 + XCH_BYTES + 1024; }
// the accumulator tile [128 rows][64 tokens] fp32 is staged through the (dead) pipeline stages after the main loop, one
// row per epilogue thread; it starts past the 32 KB that the cluster split-K reduction receives from its peers
constexpr int ACC_OFF = 32 * 1024, ACC_LD = TOK + 4;
static_assert(ACC_OFF + BMW * ACC_LD * 4 <= 4 * STAGE_BYTES, "accumulator staging must fit in the pipeline stages");

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_smem_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta_rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f4(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// K-major SWIZZLE_128B wgmma operand descriptor (sm_90 GMMA descriptor): 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t kmajor_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;           // LBO (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32; // SBO
  d |= (uint64_t)1 << 62;           // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// the accumulator registers are written asynchronously: this pins every read of them after the wait above
__device__ __forceinline__ void fence_acc(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 64] += A[64 x 16] * B[64 x 16]^T, bf16 in, fp32 accumulate, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}
// one stage (BK = 64 k) of this warpgroup's 64 weight rows against the 64 tokens
__device__ __forceinline__ void mma_stage(float (&acc)[32], uint32_t wa, uint32_t xa) {
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < BK / 16; ++j) wgmma_m64n64k16(acc, kmajor_desc(wa + j * 32), kmajor_desc(xa + j * 32));
  wgmma_commit();
  wgmma_wait_all();
  fence_acc(acc);
}
// accumulator fragment element -> (row of the warpgroup's 64, token): register 4*i + 2*h + e holds
// row 16 * (warp % 4) + lane / 4 + 8 * h, token 8 * i + 2 * (lane % 4) + e
__device__ __forceinline__ int frag_row(int warp, int lane, int h) { return 16 * (warp & 3) + (lane >> 2) + 8 * h; }
__device__ __forceinline__ int frag_tok(int lane, int i) { return 8 * i + 2 * (lane & 3); }

struct Params {
  int N, K, n_split, chunks_per_split, n_chunks, rows, tiled;
  int groups, w_group_rows, x_group_chunks;  // grouped GEMM (gridDim.z = groups): group g uses weight rows
                                             // [g*w_group_rows, +N) and activation columns [g*x_group_chunks*64, +K)
  long long out_group_stride;                // elements between the groups' [rows_cap, N] outputs
  int cluster;              // > 1: the K splits of a tile are one thread-block cluster and reduce through DSMEM (bf16 out)
  int silu;                 // 1: tile rows are 64 gate rows + 64 up rows of the same columns -> out = silu(g) * u
  int no_pdl;               // 1: plain kernel boundary - do not let the successor start early either
  __nv_bfloat16 *out_bf16;  // [rows_cap, N]  (or [rows_cap, N/2] with silu)   (n_split == 1)
  float *out_f32;           // [n_split, TOK, N] slices  (n_split > 1)
};

// NSTAGE = 4: ~100 KB of shared memory, two CTAs per SM (grids with more CTAs than SMs);
// NSTAGE = 8: ~200 KB, one CTA per SM with twice the bytes in flight (grids that do not fill the SMs twice) -
// HBM only saturates with several MB of loads in flight chip-wide.
template <int NSTAGE>
__global__ void __launch_bounds__(NTHREADS, NSTAGE <= 4 ? 2 : 1)
k_gemm_ws(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, Params p) {
  constexpr int SMEM_BAR = NSTAGE * STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t bar_full = base + SMEM_BAR, bar_empty = bar_full + 8 * NSTAGE;
  // grid = (tiles, splits), or (splits, tiles) when the splits of a tile form a cluster (clusters run along x)
  const int tile = p.cluster ? blockIdx.y : blockIdx.x, split = p.cluster ? blockIdx.x : blockIdx.y;
  const int n0 = tile * BMW;
  const int grp = blockIdx.z;  // 0 unless the plan is a grouped GEMM (one group = one MoE expert)
  const int xk0 = grp * p.x_group_chunks;
  const int c0 = split * p.chunks_per_split;
  int c1 = c0 + p.chunks_per_split;
  if (c1 > p.n_chunks) c1 = p.n_chunks;
  const int nch = c1 - c0;

  if (tid == 0) {
    // a stage is free again once each of the 8 consumer warps has seen its wgmma on it complete
    for (int s = 0; s < NSTAGE; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();  // warp 0 reconverges before the block barrier below
  if (!p.no_pdl) pdl_launch_dependents();
  __syncthreads();
  // Barriers are set up while the previous kernel drains, and - the weights being immutable - the first NSTAGE weight
  // tiles are already streaming from HBM before griddepcontrol.wait: only the activation tiles (and the output
  // stores) depend on the predecessor, so its run time hides this kernel's pipeline fill.

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      auto load_w = [&](int i, int s) {
        const uint32_t wd = base + s * STAGE_BYTES;
        if (p.tiled) tma_load_3d(wd, &map_w, bar_full + 8 * s, 0, 0, tile * p.n_chunks + c0 + i);
        else tma_load_2d(wd, &map_w, bar_full + 8 * s, (c0 + i) * BK, grp * p.w_group_rows + n0);
      };
      const int pre = nch < NSTAGE ? nch : NSTAGE;
      for (int i = 0; i < pre; ++i) {  // all stages start empty
        mbar_expect_tx(bar_full + 8 * i, STAGE_BYTES);
        load_w(i, i);
      }
      pdl_wait();
      for (int i = 0; i < pre; ++i) tma_load_2d(base + i * STAGE_BYTES + W_BYTES, &map_x, bar_full + 8 * i, (xk0 + c0 + i) * BK, 0);
      for (int i = pre; i < nch; ++i) {
        const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
        mbar_wait(bar_empty + 8 * s, ph ^ 1);
        mbar_expect_tx(bar_full + 8 * s, STAGE_BYTES);
        load_w(i, s);
        tma_load_2d(base + s * STAGE_BYTES + W_BYTES, &map_x, bar_full + 8 * s, (xk0 + c0 + i) * BK, 0);
      }
    }
    __syncwarp();
    if (p.cluster) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }

  // ---------------------------------------------------------------- consumers: warpgroup wg owns weight rows [64 wg, +64)
  pdl_wait();  // output stores (and the WAR hazard on the output buffer) are ordered after the predecessor
  const int wg = warp >> 2;
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int i = 0; i < nch; ++i) {
    const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
    mbar_wait(bar_full + 8 * s, ph);
    const uint32_t wa = base + s * STAGE_BYTES, xa = wa + W_BYTES;
    mma_stage(acc, wa + wg * 64 * 128, xa);
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
  }
  // stage the tile through shared memory so that the epilogue thread of weight row r holds its 64 tokens
  float *accs = reinterpret_cast<float *>(sm + ACC_OFF);
  asm volatile("bar.sync 2, 256;" ::: "memory");  // every wgmma of both warpgroups has read its last stage
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wg * 64 + frag_row(warp, lane, h);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<float2 *>(accs + r * ACC_LD + frag_tok(lane, i)) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
  }
  asm volatile("bar.sync 2, 256;" ::: "memory");
  if (wg == 1) {
    if (p.cluster) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }

  // epilogue (warps 0-3): thread = one weight row n, 64 token values in registers
  const int q = warp;
  const int n = n0 + q * 32 + lane;
  uint32_t v[64];
  {
    const float4 *src = reinterpret_cast<const float4 *>(accs + (q * 32 + lane) * ACC_LD);
#pragma unroll
    for (int t = 0; t < 16; ++t) {
      const float4 a = src[t];
      v[4 * t] = __float_as_uint(a.x); v[4 * t + 1] = __float_as_uint(a.y);
      v[4 * t + 2] = __float_as_uint(a.z); v[4 * t + 3] = __float_as_uint(a.w);
    }
  }
  if (p.cluster) {
    // split-K inside a cluster: after everyone has left its main loop (barrier A: the pipeline stages of every CTA
    // are dead) each thread pushes its fp32 row - 16 token quads, quad-major so that the lanes of a warp write
    // consecutive 16-byte words - into the CTA that owns that row slice, barrier B, and the owner adds the
    // cluster's partials in split order (deterministic) and writes bf16.  No fp32 round trip through HBM/L2.
    const int cs = p.cluster, RS = BMW / cs;      // rows per owner CTA: 64 (2 splits) or 32 (4 splits)
    cluster_sync_all();
    {
      const int row = q * 32 + lane;
      const int owner = row / RS, rl = row % RS;
      const uint32_t dst = map_to_cta(base + (uint32_t)((split * 16) * RS + rl) * 16, owner);
#pragma unroll
      for (int tq = 0; tq < 16; ++tq)
        st_cluster_f4(dst + (uint32_t)(tq * RS) * 16, __uint_as_float(v[4 * tq]), __uint_as_float(v[4 * tq + 1]),
                      __uint_as_float(v[4 * tq + 2]), __uint_as_float(v[4 * tq + 3]));
    }
    cluster_sync_all();
    {
      const int e = warp * 32 + lane;             // 0..127
      const int rl = e % RS, tg = e / RS;         // row of this CTA's slice, token group
      const int qpt = RS / 8;                     // token quads per thread: 16 / (128 / RS)
      const int n_out = n0 + split * RS + rl;     // this CTA's rank in the cluster == its split index
      const float4 *buf = reinterpret_cast<const float4 *>(sm);
      __nv_bfloat16 *ob = p.out_bf16 + grp * p.out_group_stride;
      if (n_out < p.N) {
        for (int tq = tg * qpt; tq < (tg + 1) * qpt; ++tq) {
          float4 a = buf[(0 * 16 + tq) * RS + rl];
          for (int src = 1; src < cs; ++src) {
            const float4 b = buf[(src * 16 + tq) * RS + rl];
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
          }
          const int t0 = 4 * tq;
          if (t0 < p.rows) ob[(long long)t0 * p.N + n_out] = __float2bfloat16_rn(a.x);
          if (t0 + 1 < p.rows) ob[(long long)(t0 + 1) * p.N + n_out] = __float2bfloat16_rn(a.y);
          if (t0 + 2 < p.rows) ob[(long long)(t0 + 2) * p.N + n_out] = __float2bfloat16_rn(a.z);
          if (t0 + 3 < p.rows) ob[(long long)(t0 + 3) * p.N + n_out] = __float2bfloat16_rn(a.w);
        }
      }
    }
  } else
  if (p.silu) {
    // act(gate) * up (modeling_llama.py:185-186) in the epilogue: rows 0-63 (warps q = 0, 1) hold gate rows, rows
    // 64-127 (q = 2, 3) the up rows of the same 64 output columns.  Each warp pair splits the 64 tokens: the gate warp
    // finishes tokens 0-31 (it receives the up values through shared memory), the up warp tokens 32-63 (it receives the
    // gate values), so all four warps share the exponentials.  Rounding points as in eager bf16 (and k_silu_mul):
    // GEMM out -> bf16, silu -> bf16, product -> bf16.
    __nv_bfloat16 *xu = reinterpret_cast<__nv_bfloat16 *>(sm + SMEM_BAR + 256);  // up   [32 tokens 0-31 ][64 rows]
    __nv_bfloat16 *xg = xu + 32 * 64;                                             // gate [32 tokens 32-63][64 rows]
    const int rr = (q & 1) * 32 + lane;
    if (q >= 2) {
#pragma unroll
      for (int t = 0; t < 32; ++t) xu[t * 64 + rr] = __float2bfloat16_rn(__uint_as_float(v[t]));
    } else {
#pragma unroll
      for (int t = 0; t < 32; ++t) xg[t * 64 + rr] = __float2bfloat16_rn(__uint_as_float(v[32 + t]));
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const int col = tile * 64 + rr;
    const int inter = p.N >> 1;
    if (col < inter) {
      const int tb = q < 2 ? 0 : 32;
#pragma unroll
      for (int t = 0; t < 32; ++t) {
        if (tb + t < p.rows) {
          const float g = q < 2 ? __bfloat162float(__float2bfloat16_rn(__uint_as_float(v[t]))) : __bfloat162float(xg[t * 64 + rr]);
          const float u = q < 2 ? __bfloat162float(xu[t * 64 + rr]) : __bfloat162float(__float2bfloat16_rn(__uint_as_float(v[32 + t])));
          const float sg = __bfloat162float(__float2bfloat16_rn(g / (1.f + expf(-g))));
          p.out_bf16[(long long)(tb + t) * inter + col] = __float2bfloat16_rn(sg * u);
        }
      }
    }
  } else
  if (n < p.N) {
    if (p.n_split == 1) {
#pragma unroll
      for (int t = 0; t < TOK; ++t)
        if (t < p.rows) p.out_bf16[grp * p.out_group_stride + (long long)t * p.N + n] = __float2bfloat16_rn(__uint_as_float(v[t]));
    } else {
      float *o = p.out_f32 + (long long)split * TOK * p.N;
#pragma unroll
      for (int t = 0; t < TOK; ++t)
        if (t < p.rows) o[(long long)t * p.N + n] = __uint_as_float(v[t]);
    }
  }
}


// ------------------------------------------------------------------------------------------------ stream-K
// Work = n_tiles x n_chunks (tile, k-chunk) units, cut into gridDim.x equal contiguous ranges: every SM streams
// the same number of bytes whatever N is (qkv: 96 tiles, o/down: 32 tiles on 132 SMs).  A tile whose chunks span
// several CTAs is finished by the CTA that holds its FIRST chunk (it reaches that tile last in its own range, so the
// other contributors - which meet the tile first in theirs - are normally done already): contributors store their
// fp32 partial to a workspace slot and bump the tile's flag, the owner adds the slots in slot order (deterministic)
// and writes bf16.  All CTAs are co-resident (grid <= #SMs, one CTA per SM), so the owner's wait cannot deadlock.
struct SkParams {
  int N, n_tiles, n_chunks, rows, max_contrib;
  long long units;
  __nv_bfloat16 *out;   // [rows_cap, N]
  float *ws;            // [n_tiles][max_contrib][128][64]
  int *flags;           // [n_tiles], zero between launches
};

// shared with the host, which sizes the fix-up workspace from the same partition
__host__ __device__ __forceinline__ long long sk_begin(long long b, long long U, int G) { return b * U / G; }
__host__ __device__ __forceinline__ int sk_cta_of(long long x, long long U, int G) {
  int b = (int)(x * G / U);
  while (b + 1 < G && sk_begin(b + 1, U, G) <= x) ++b;
  while (b > 0 && sk_begin(b, U, G) > x) --b;
  return b;
}

constexpr int SK_STAGES = 8;
constexpr int SK_SMEM_BAR = SK_STAGES * STAGE_BYTES;
constexpr int SK_SMEM_TOTAL = SK_SMEM_BAR + 256 + 1024;

__global__ void __launch_bounds__(NTHREADS, 1)
k_gemm_sk(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, SkParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t bar_full = base + SK_SMEM_BAR, bar_empty = bar_full + 8 * SK_STAGES;
  const int G = gridDim.x, b = blockIdx.x;
  const long long u0 = sk_begin(b, p.units, G), u1 = sk_begin(b + 1, p.units, G);

  if (tid == 0) {
    for (int s = 0; s < SK_STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();  // warp 0 reconverges before the block barrier below
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      int i = 0;
      for (long long u = u0; u < u1; ++u, ++i) {
        const int tile = (int)(u / p.n_chunks), ch = (int)(u % p.n_chunks);
        const int s = i % SK_STAGES, ph = (i / SK_STAGES) & 1;
        mbar_wait(bar_empty + 8 * s, ph ^ 1);
        mbar_expect_tx(bar_full + 8 * s, STAGE_BYTES);
        const uint32_t wd = base + s * STAGE_BYTES, xd = wd + W_BYTES;
        tma_load_3d(wd, &map_w, bar_full + 8 * s, 0, 0, tile * p.n_chunks + ch);
        tma_load_2d(xd, &map_x, bar_full + 8 * s, ch * BK, 0);
      }
    }
    return;
  }

  // consumers: one tile segment after the other; the epilogue works on the register fragments directly
  const int wg = warp >> 2;
  int i = 0;
  long long u = u0;
  float acc[32];
  while (u < u1) {
    const int tile = (int)(u / p.n_chunks);
    const long long ts = (long long)tile * p.n_chunks;
    long long ue = ts + p.n_chunks;
    if (ue > u1) ue = u1;
    const bool head = (u == ts), whole = head && (ue == ts + p.n_chunks);
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    for (; u < ue; ++u, ++i) {
      const int s = i % SK_STAGES, ph = (i / SK_STAGES) & 1;
      mbar_wait(bar_full + 8 * s, ph);
      const uint32_t wa = base + s * STAGE_BYTES, xa = wa + W_BYTES;
      mma_stage(acc, wa + wg * 64 * 128, xa);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
    }
    if (!head) {
      // contributor: slot = how many CTA ranges after the owner's this one is
      const int owner = sk_cta_of(ts, p.units, G);
      const int slot = b - owner - 1;
      float *ws = p.ws + ((long long)tile * p.max_contrib + slot) * BMW * TOK;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = wg * 64 + frag_row(warp, lane, h);
#pragma unroll
        for (int k = 0; k < 8; ++k)
          *reinterpret_cast<float2 *>(ws + r * TOK + frag_tok(lane, k)) = make_float2(acc[4 * k + 2 * h], acc[4 * k + 2 * h + 1]);
      }
      __threadfence();
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (tid == 0) atomicAdd(&p.flags[tile], 1);
    } else {
      if (!whole) {
        // owner: wait for the other contributors of this tile, then add their slots in order
        const int last = sk_cta_of(ts + p.n_chunks - 1, p.units, G);
        const int contributors = last - b;
        if (tid == 0) {
          while (atomicAdd(&p.flags[tile], 0) < contributors) __nanosleep(64);
          p.flags[tile] = 0;  // self-reset for the next launch
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        __threadfence();
        for (int c = 0; c < contributors; ++c) {
          const float *ws = p.ws + ((long long)tile * p.max_contrib + c) * BMW * TOK;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = wg * 64 + frag_row(warp, lane, h);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const float2 x = __ldcg(reinterpret_cast<const float2 *>(ws + r * TOK + frag_tok(lane, k)));
              acc[4 * k + 2 * h] += x.x;
              acc[4 * k + 2 * h + 1] += x.y;
            }
          }
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = tile * BMW + wg * 64 + frag_row(warp, lane, h);
        if (n < p.N) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int t = frag_tok(lane, k);
            if (t < p.rows) p.out[(long long)t * p.N + n] = __float2bfloat16_rn(acc[4 * k + 2 * h]);
            if (t + 1 < p.rows) p.out[(long long)(t + 1) * p.N + n] = __float2bfloat16_rn(acc[4 * k + 2 * h + 1]);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ fp8 (e4m3) weights
// W8A16: every weight row n is symmetric e4m3 with an fp32 scale s[n]; X stays bf16.  Same structure as k_gemm_ws
// (swap-AB, two consumer warpgroups x wgmma M = 64, TMA producer warp over the mbarrier ring, HBM-tiled weight), but a
// stage covers 128 k: one 16 KB weight block of 128 rows x 128 e4m3 bytes (one SWIZZLE_128B row per weight row) plus
// the two matching 64-k bf16 X boxes.  The consumers read their wgmma A fragment straight from the staged fp8 bytes,
// convert it to bf16 pairs in registers (exact: every finite e4m3 value is a bf16 value) and issue
// wgmma.m64n64k16 with A in registers and X from shared memory.  Epilogue: y = acc * s[n] (+ bias[n]) in fp32, one bf16
// rounding.  Row counts above 64: gridDim.z also runs over 64-row token blocks, each streaming the weight again.
constexpr int F8_BK = 128;                                // k per stage: 128 e4m3 bytes = one 128-byte swizzle row
constexpr int F8_W_BYTES = BMW * F8_BK;                   // 16 KB
constexpr int F8_STAGE_BYTES = F8_W_BYTES + 2 * X_BYTES;  // + two 64-k bf16 X boxes
constexpr int f8_smem_total(int nstage) { return nstage * F8_STAGE_BYTES + 256 + XCH_BYTES + 1024; }
static_assert(ACC_OFF + BMW * ACC_LD * 4 <= 3 * F8_STAGE_BYTES, "accumulator staging must fit in the pipeline stages");

// two e4m3 codes (low byte = lower k) -> bf16x2 (low half = lower k): e4m3 -> f16 is exact, f16 -> f32 -> bf16 too
__device__ __forceinline__ void e4m3x4_to_bf16x2(uint32_t w, uint32_t &lo, uint32_t &hi) {
  uint32_t h0, h1;
  asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\t"
      "cvt.rn.f16x2.e4m3x2 %0, l;\n\tcvt.rn.f16x2.e4m3x2 %1, h;\n\t}"
      : "=r"(h0), "=r"(h1) : "r"(w));
  const float2 f0 = __half22float2(*reinterpret_cast<const __half2 *>(&h0));
  const float2 f1 = __half22float2(*reinterpret_cast<const __half2 *>(&h1));
  const __nv_bfloat162 b0 = __floats2bfloat162_rn(f0.x, f0.y), b1 = __floats2bfloat162_rn(f1.x, f1.y);
  lo = *reinterpret_cast<const uint32_t *>(&b0);
  hi = *reinterpret_cast<const uint32_t *>(&b1);
}
// D[64 x 64] += A[64 x 16] * B[64 x 16]^T, A = bf16 pairs in registers, B K-major in shared memory
__device__ __forceinline__ void wgmma_m64n64k16_ra(float (&d)[32], const uint32_t *a, uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
      : "memory");
}

struct F8Params {
  int N, n_chunks, chunks_per_split, n_split, rows, ntb;  // n_chunks: K / 128; ntb: 64-row token blocks of this run
  int tiles;                   // N / 128
  int x_group_chunks;          // grouped: group g reads activation columns [g * x_group_chunks * 128, +K)
  long long out_group_stride;  // elements between the groups' [x_rows, N] outputs
  long long slice_stride;      // fp32 split-K slices: elements between two splits' [x_rows, N] slices
  int cluster, silu, no_pdl;
  int relu;                    // 1: y = max(acc * s[n] + bias[n], 0) before the bf16 rounding (bf16 outputs only)
  const float *scale;          // [groups * N], one per stored weight row
  const float *bias;           // [N] or null (split_k == 1 or cluster splits only)
  __nv_bfloat16 *out_bf16;
  float *out_f32;
};

// the bf16 epilogue's activation: OPT's fc1 ReLU (opt/modeling_opt.py:356) on the biased fp32 value, so that the one
// bf16 rounding of relu(x) equals relu of the rounded x (bf16 rounding is monotone and keeps 0)
__device__ __forceinline__ float f8_act(float v, int relu) { return relu ? fmaxf(v, 0.f) : v; }

// NSTAGE = 3: ~106 KB of shared memory, two CTAs per SM; NSTAGE = 6: ~202 KB, one CTA per SM (grids that do not
// fill the SMs twice) - 96 KB of weight bytes in flight per SM either way
template <int NSTAGE>
__global__ void __launch_bounds__(NTHREADS, NSTAGE <= 3 ? 2 : 1)
k_gemm_fp8(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, F8Params p) {
  constexpr int SMEM_BAR = NSTAGE * F8_STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t bar_full = base + SMEM_BAR, bar_empty = bar_full + 8 * NSTAGE;
  const int tile = p.cluster ? blockIdx.y : blockIdx.x, split = p.cluster ? blockIdx.x : blockIdx.y;
  const int n0 = tile * BMW;
  const int grp = blockIdx.z / p.ntb, t0 = (blockIdx.z % p.ntb) * TOK;  // expert, first token row of this CTA
  const int rows = p.rows - t0 < TOK ? p.rows - t0 : TOK;
  const int c0 = split * p.chunks_per_split;
  int c1 = c0 + p.chunks_per_split;
  if (c1 > p.n_chunks) c1 = p.n_chunks;
  const int nch = c1 - c0;

  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  if (!p.no_pdl) pdl_launch_dependents();
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      // the weight blocks are immutable: the first NSTAGE stream before griddepcontrol.wait, as in k_gemm_ws
      const int wblk = (grp * p.tiles + tile) * p.n_chunks + c0;
      const int xk = (grp * p.x_group_chunks + c0) * 2;  // in 64-k boxes
      auto load_x = [&](int i, int s) {
        const uint32_t xd = base + s * F8_STAGE_BYTES + F8_W_BYTES;
        tma_load_2d(xd, &map_x, bar_full + 8 * s, (xk + 2 * i) * BK, t0);
        tma_load_2d(xd + X_BYTES, &map_x, bar_full + 8 * s, (xk + 2 * i + 1) * BK, t0);
      };
      const int pre = nch < NSTAGE ? nch : NSTAGE;
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(bar_full + 8 * i, F8_STAGE_BYTES);
        tma_load_3d(base + i * F8_STAGE_BYTES, &map_w, bar_full + 8 * i, 0, 0, wblk + i);
      }
      pdl_wait();
      for (int i = 0; i < pre; ++i) load_x(i, i);
      for (int i = pre; i < nch; ++i) {
        const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
        mbar_wait(bar_empty + 8 * s, ph ^ 1);
        mbar_expect_tx(bar_full + 8 * s, F8_STAGE_BYTES);
        tma_load_3d(base + s * F8_STAGE_BYTES, &map_w, bar_full + 8 * s, 0, 0, wblk + i);
        load_x(i, s);
      }
    }
    __syncwarp();
    if (p.cluster) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }

  // ---------------------------------------------------------------- consumers: warpgroup wg owns weight rows [64 wg, +64)
  pdl_wait();
  const int wg = warp >> 2;
  // A fragment of m64k16 (register i of k-step j): a0 = (row r, k 2c..2c+1), a1 = (r + 8, same k), a2 = (r, k + 8),
  // a3 = (r + 8, k + 8) with r = 16 (warp % 4) + lane / 4, c = lane % 4.  The tiled weight stores each 16-byte k group
  // as [k0 k1 k8 k9 | k2 k3 k10 k11 | ...] (ops.tile_weight_fp8), so one 32-bit load yields a0's and a2's codes.  The
  // 16-byte group j of row r sits at chunk j ^ (r % 8) (SWIZZLE_128B); rows r and r + 8 share that pattern.
  const int r = wg * 64 + 16 * (warp & 3) + (lane >> 2);
  const uint32_t roff = (uint32_t)r * F8_BK + 4 * (lane & 3);
  const int sw = r & 7;
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int i = 0; i < nch; ++i) {
    const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
    mbar_wait(bar_full + 8 * s, ph);
    const uint8_t *ws = sm + s * F8_STAGE_BYTES;
    uint32_t a[32];
#pragma unroll
    for (int j = 0; j < F8_BK / 16; ++j) {
      const uint32_t off = roff + ((uint32_t)(j ^ sw) << 4);
      e4m3x4_to_bf16x2(*reinterpret_cast<const uint32_t *>(ws + off), a[4 * j], a[4 * j + 2]);
      e4m3x4_to_bf16x2(*reinterpret_cast<const uint32_t *>(ws + off + 8 * F8_BK), a[4 * j + 1], a[4 * j + 3]);
    }
    const uint32_t xa = base + s * F8_STAGE_BYTES + F8_W_BYTES;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < F8_BK / 16; ++j) wgmma_m64n64k16_ra(acc, a + 4 * j, kmajor_desc(xa + (j >> 2) * X_BYTES + (j & 3) * 32));
    wgmma_commit();
    wgmma_wait_all();
    fence_acc(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
  }
  float *accs = reinterpret_cast<float *>(sm + ACC_OFF);
  asm volatile("bar.sync 2, 256;" ::: "memory");
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int rr = wg * 64 + frag_row(warp, lane, h);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<float2 *>(accs + rr * ACC_LD + frag_tok(lane, i)) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
  }
  asm volatile("bar.sync 2, 256;" ::: "memory");
  if (wg == 1) {
    if (p.cluster) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }

  // epilogue (warps 0-3): thread = one weight row n, its 64 token values scaled by s[n] in fp32
  const int q = warp;
  const int n = n0 + q * 32 + lane;
  float v[64];
  {
    const float sc = p.scale[(long long)grp * p.N + n];
    const float4 *src = reinterpret_cast<const float4 *>(accs + (q * 32 + lane) * ACC_LD);
#pragma unroll
    for (int t = 0; t < 16; ++t) {
      const float4 a = src[t];
      v[4 * t] = a.x * sc; v[4 * t + 1] = a.y * sc; v[4 * t + 2] = a.z * sc; v[4 * t + 3] = a.w * sc;
    }
  }
  if (p.cluster) {
    // the scaled fp32 partials meet in the owner CTA of each row slice (as in k_gemm_ws), summed in split order; the
    // bias is added once, after the sum
    const int cs = p.cluster, RS = BMW / cs;
    cluster_sync_all();
    {
      const int row = q * 32 + lane;
      const int owner = row / RS, rl = row % RS;
      const uint32_t dst = map_to_cta(base + (uint32_t)((split * 16) * RS + rl) * 16, owner);
#pragma unroll
      for (int tq = 0; tq < 16; ++tq) st_cluster_f4(dst + (uint32_t)(tq * RS) * 16, v[4 * tq], v[4 * tq + 1], v[4 * tq + 2], v[4 * tq + 3]);
    }
    cluster_sync_all();
    {
      const int e = warp * 32 + lane;
      const int rl = e % RS, tg = e / RS;
      const int qpt = RS / 8;
      const int n_out = n0 + split * RS + rl;
      const float4 *buf = reinterpret_cast<const float4 *>(sm);
      __nv_bfloat16 *ob = p.out_bf16 + grp * p.out_group_stride + (long long)t0 * p.N;
      const float bs = p.bias ? p.bias[n_out] : 0.f;
      for (int tq = tg * qpt; tq < (tg + 1) * qpt; ++tq) {
        float4 a = buf[(0 * 16 + tq) * RS + rl];
        for (int src = 1; src < cs; ++src) {
          const float4 b = buf[(src * 16 + tq) * RS + rl];
          a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        const int tt = 4 * tq;
        if (tt < rows) ob[(long long)tt * p.N + n_out] = __float2bfloat16_rn(f8_act(a.x + bs, p.relu));
        if (tt + 1 < rows) ob[(long long)(tt + 1) * p.N + n_out] = __float2bfloat16_rn(f8_act(a.y + bs, p.relu));
        if (tt + 2 < rows) ob[(long long)(tt + 2) * p.N + n_out] = __float2bfloat16_rn(f8_act(a.z + bs, p.relu));
        if (tt + 3 < rows) ob[(long long)(tt + 3) * p.N + n_out] = __float2bfloat16_rn(f8_act(a.w + bs, p.relu));
      }
    }
  } else if (p.silu) {
    // SiLU(gate) * up exactly as k_gemm_ws's epilogue: rows 0-63 of the tile are gate rows, 64-127 the up rows of the
    // same 64 columns (scales permuted alike); GEMM out -> bf16, silu -> bf16, product -> bf16
    __nv_bfloat16 *xu = reinterpret_cast<__nv_bfloat16 *>(sm + SMEM_BAR + 256);
    __nv_bfloat16 *xg = xu + 32 * 64;
    const int rr = (q & 1) * 32 + lane;
    if (q >= 2) {
#pragma unroll
      for (int t = 0; t < 32; ++t) xu[t * 64 + rr] = __float2bfloat16_rn(v[t]);
    } else {
#pragma unroll
      for (int t = 0; t < 32; ++t) xg[t * 64 + rr] = __float2bfloat16_rn(v[32 + t]);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const int col = tile * 64 + rr;
    const int inter = p.N >> 1;
    __nv_bfloat16 *ob = p.out_bf16 + (long long)t0 * inter;
    const int tb = q < 2 ? 0 : 32;
#pragma unroll
    for (int t = 0; t < 32; ++t) {
      if (tb + t < rows) {
        const float g = q < 2 ? __bfloat162float(__float2bfloat16_rn(v[t])) : __bfloat162float(xg[t * 64 + rr]);
        const float u = q < 2 ? __bfloat162float(xu[t * 64 + rr]) : __bfloat162float(__float2bfloat16_rn(v[32 + t]));
        const float sg = __bfloat162float(__float2bfloat16_rn(g / (1.f + expf(-g))));
        ob[(long long)(tb + t) * inter + col] = __float2bfloat16_rn(sg * u);
      }
    }
  } else if (p.n_split == 1) {
    const float bs = p.bias ? p.bias[n] : 0.f;
    __nv_bfloat16 *ob = p.out_bf16 + grp * p.out_group_stride + (long long)t0 * p.N;
#pragma unroll
    for (int t = 0; t < TOK; ++t)
      if (t < rows) ob[(long long)t * p.N + n] = __float2bfloat16_rn(f8_act(v[t] + bs, p.relu));
  } else {
    float *o = p.out_f32 + split * p.slice_stride + (long long)t0 * p.N;
#pragma unroll
    for (int t = 0; t < TOK; ++t)
      if (t < rows) o[(long long)t * p.N + n] = v[t];
  }
}

// ------------------------------------------------------------------------------------------------ int4 weights
// W4A16 with group-wise scales and zero points (GPTQ / compressed-tensors pack-quantized checkpoints): the weight is
//   W[n, k] = bf16(dtype_s(s[g, n] * (u[n, k] - z[g, n]))),  g = k / group,
// u the unsigned 4-bit code, z its zero point (0..16), s the group's scale in the checkpoint's dtype (bf16 or fp16).
// Same structure as k_gemm_fp8 (swap-AB, two consumer warpgroups x wgmma M = 64 over 128 weight rows, TMA producer warp
// over an mbarrier ring, HBM-tiled weight, gridDim.z over 64-row token blocks), but a stage covers 256 k: one 16 KB
// block of 128 rows x 128 bytes of codes (ops.tile_weight_w4, one SWIZZLE_128B row per weight row), the four matching
// 64-k bf16 X boxes, and the scales and zero points of the stage's two 128-k halves (four bulk copies out of the
// [G, N] tables: 128 rows x {bf16|fp16} and 128 rows x uint8 per half).  The consumers dequantise their wgmma A fragment
// in registers: a nibble pair becomes (B + u) as a 16-bit pair (B = 128 in bf16, 1024 in fp16, both with ulp 1), minus
// (B + z) is exact, times s in the scale's own 16-bit arithmetic is the one rounding to dtype_s; fp16 then goes to bf16
// (a second rounding, as the checkpoint's dequantisation does).  W is bf16 before the MMA, so the epilogue has no scale:
// k_gemm_fp8's with the multiply removed (bias in fp32, SiLU*up, cluster split-K, fp32 slices).
constexpr int W4_BK = 256;                                 // k per stage: 128 bytes of packed codes per weight row
constexpr int W4_W_BYTES = BMW * W4_BK / 2;                // 16 KB
constexpr int W4_X_OFF = W4_W_BYTES;                       // four 64-k bf16 X boxes, 1024-byte aligned
constexpr int W4_META_OFF = W4_X_OFF + 4 * X_BYTES;        // scales [2 halves][128] 16-bit, zeros [2 halves][128] u8
constexpr int W4_STAGE_BYTES = W4_META_OFF + 1024;         // 49 KB: the 768 meta bytes padded to keep stages aligned
constexpr int w4_smem_total(int nstage) { return nstage * W4_STAGE_BYTES + 256 + XCH_BYTES + 1024; }
static_assert(ACC_OFF + BMW * ACC_LD * 4 <= 2 * W4_STAGE_BYTES, "accumulator staging must fit in the pipeline stages");

struct W4Params {
  int N, K, n_chunks, chunks_per_split, n_split, rows, ntb;  // n_chunks: ceil(K / 256); ntb: 64-row token blocks
  int tiles, group;            // N / 128, k per scale group (a multiple of 128)
  long long slice_stride;      // fp32 split-K slices: elements between two splits' [x_rows, N] slices
  int cluster, silu, no_pdl;
  const void *scale;           // [K / group, N] bf16 or fp16
  const uint8_t *zero;         // [K / group, N] zero points 0..16
  const float *bias;           // [N] or null
  __nv_bfloat16 *out_bf16;
  float *out_f32;
};

__device__ __forceinline__ void bulk_load(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// the nibbles at bits [0, 4) and [16, 20) of w -> a bf16x2 fragment register (low half = lower k).  zo = (B + z) in
// both halves, sc = s in both halves, in the scale's format.
template <bool F16>
__device__ __forceinline__ uint32_t w4_deq(uint32_t w, uint32_t zo, uint32_t sc) {
  uint32_t x = (w & 0x000F000Fu) | (F16 ? 0x64006400u : 0x43004300u), d;
  if (F16) {
    asm("{\n\t.reg .b32 t;\n\tsub.rn.f16x2 t, %1, %2;\n\tmul.rn.f16x2 %0, t, %3;\n\t}" : "=r"(d) : "r"(x), "r"(zo), "r"(sc));
    const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&d));
    const __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
    return *reinterpret_cast<const uint32_t *>(&b);
  }
  asm("{\n\t.reg .b32 t;\n\tsub.rn.bf16x2 t, %1, %2;\n\tmul.rn.bf16x2 %0, t, %3;\n\t}" : "=r"(d) : "r"(x), "r"(zo), "r"(sc));
  return d;
}

// NSTAGE = 2: ~107 KB of shared memory, two CTAs per SM; NSTAGE = 4: ~205 KB, one CTA per SM (grids that do not fill
// the SMs twice) - 64 KB of code bytes (128 K weights) in flight per SM either way
template <int NSTAGE, bool F16>
__global__ void __launch_bounds__(NTHREADS, NSTAGE <= 2 ? 2 : 1)
k_gemm_w4(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, W4Params p) {
  constexpr int SMEM_BAR = NSTAGE * W4_STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t bar_full = base + SMEM_BAR, bar_empty = bar_full + 8 * NSTAGE;
  const int tile = p.cluster ? blockIdx.y : blockIdx.x, split = p.cluster ? blockIdx.x : blockIdx.y;
  const int n0 = tile * BMW;
  const int t0 = blockIdx.z * TOK;  // first token row of this CTA
  const int rows = p.rows - t0 < TOK ? p.rows - t0 : TOK;
  const int c0 = split * p.chunks_per_split;
  int c1 = c0 + p.chunks_per_split;
  if (c1 > p.n_chunks) c1 = p.n_chunks;
  const int nch = c1 - c0;
  const int khalves = p.K / 128;    // a last chunk may hold one 128-k half only (K % 256 == 128)

  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  if (!p.no_pdl) pdl_launch_dependents();
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      // codes, scales and zero points are immutable: the first NSTAGE stages stream before griddepcontrol.wait
      const int wblk = tile * p.n_chunks + c0;
      constexpr int sb = 2;  // bytes per scale (bf16 or fp16)
      auto halves = [&](int i) { return 2 * (c0 + i) + 1 < khalves ? 2 : 1; };
      auto stage_bytes = [&](int i) { return (uint32_t)(W4_W_BYTES + halves(i) * (2 * X_BYTES + BMW * (sb + 1))); };
      auto load_w = [&](int i, int s) {
        const uint32_t st = base + s * W4_STAGE_BYTES, bar = bar_full + 8 * s;
        tma_load_3d(st, &map_w, bar, 0, 0, wblk + i);
        for (int h = 0; h < halves(i); ++h) {
          const long long g = (long long)((c0 + i) * W4_BK + h * 128) / p.group;
          bulk_load(st + W4_META_OFF + h * BMW * sb,
                    reinterpret_cast<const uint8_t *>(p.scale) + (g * p.N + n0) * sb, BMW * sb, bar);
          bulk_load(st + W4_META_OFF + 2 * BMW * sb + h * BMW, p.zero + g * p.N + n0, BMW, bar);
        }
      };
      auto load_x = [&](int i, int s) {
        const uint32_t xd = base + s * W4_STAGE_BYTES + W4_X_OFF;
        for (int b = 0; b < 2 * halves(i); ++b) tma_load_2d(xd + b * X_BYTES, &map_x, bar_full + 8 * s, ((c0 + i) * 4 + b) * BK, t0);
      };
      const int pre = nch < NSTAGE ? nch : NSTAGE;
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(bar_full + 8 * i, stage_bytes(i));
        load_w(i, i);
      }
      pdl_wait();
      for (int i = 0; i < pre; ++i) load_x(i, i);
      for (int i = pre; i < nch; ++i) {
        const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
        mbar_wait(bar_empty + 8 * s, ph ^ 1);
        mbar_expect_tx(bar_full + 8 * s, stage_bytes(i));
        load_w(i, s);
        load_x(i, s);
      }
    }
    __syncwarp();
    if (p.cluster) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }

  // ---------------------------------------------------------------- consumers: warpgroup wg owns weight rows [64 wg, +64)
  pdl_wait();
  const int wg = warp >> 2;
  // A fragment of m64k16 as in k_gemm_fp8: a0 = (row r, k 2c..2c+1), a1 = (r + 8, same k), a2 = (r, k + 8),
  // a3 = (r + 8, k + 8), r = 16 (warp % 4) + lane / 4, c = lane % 4.  Every 16-byte group (32 k) of a tiled row holds one
  // 32-bit word per c; nibble j of word c is k = 2c + {0, 8, 16, 24}[j % 4] + (j / 4) (ops.tile_weight_w4), so
  // word >> 8t (t = the k-step inside the group) masked with 0x000F000F is a0's pair, word >> (8t + 4) a2's.  The
  // 16-byte group j of row r sits at chunk j ^ (r % 8) (SWIZZLE_128B); rows r and r + 8 share that pattern.
  const int r = wg * 64 + 16 * (warp & 3) + (lane >> 2);
  const uint32_t roff = (uint32_t)r * 128 + 4 * (lane & 3);
  const int sw = r & 7;
  const uint32_t zbase = F16 ? 0x6400u : 0x4300u;
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int i = 0; i < nch; ++i) {
    const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
    mbar_wait(bar_full + 8 * s, ph);
    const uint8_t *ws = sm + s * W4_STAGE_BYTES;
    const uint16_t *ss = reinterpret_cast<const uint16_t *>(ws + W4_META_OFF);
    const uint8_t *zz = ws + W4_META_OFF + 4 * BMW;
    const uint32_t xa = base + s * W4_STAGE_BYTES + W4_X_OFF;
    const int nh = 2 * (c0 + i) + 1 < khalves ? 2 : 1;
    for (int h = 0; h < nh; ++h) {
      uint32_t sc[2], zo[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const uint32_t sv = ss[h * BMW + r + 8 * e], zv = zbase | zz[h * BMW + r + 8 * e];
        sc[e] = sv | (sv << 16);
        zo[e] = zv | (zv << 16);
      }
      uint32_t a[32];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const uint32_t off = roff + ((uint32_t)((4 * h + jj) ^ sw) << 4);
        const uint32_t w0 = *reinterpret_cast<const uint32_t *>(ws + off);
        const uint32_t w1 = *reinterpret_cast<const uint32_t *>(ws + off + 8 * 128);
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          a[8 * jj + 4 * t + 0] = w4_deq<F16>(w0 >> (8 * t), zo[0], sc[0]);
          a[8 * jj + 4 * t + 1] = w4_deq<F16>(w1 >> (8 * t), zo[1], sc[1]);
          a[8 * jj + 4 * t + 2] = w4_deq<F16>(w0 >> (8 * t + 4), zo[0], sc[0]);
          a[8 * jj + 4 * t + 3] = w4_deq<F16>(w1 >> (8 * t + 4), zo[1], sc[1]);
        }
      }
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 8; ++j) wgmma_m64n64k16_ra(acc, a + 4 * j, kmajor_desc(xa + (2 * h + (j >> 2)) * X_BYTES + (j & 3) * 32));
      wgmma_commit();
      wgmma_wait_all();
      fence_acc(acc);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
  }
  float *accs = reinterpret_cast<float *>(sm + ACC_OFF);
  asm volatile("bar.sync 2, 256;" ::: "memory");
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int rr = wg * 64 + frag_row(warp, lane, h);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<float2 *>(accs + rr * ACC_LD + frag_tok(lane, i)) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
  }
  asm volatile("bar.sync 2, 256;" ::: "memory");
  if (wg == 1) {
    if (p.cluster) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }

  // epilogue (warps 0-3): thread = one weight row n, its 64 token values
  const int q = warp;
  const int n = n0 + q * 32 + lane;
  float v[64];
  {
    const float4 *src = reinterpret_cast<const float4 *>(accs + (q * 32 + lane) * ACC_LD);
#pragma unroll
    for (int t = 0; t < 16; ++t) {
      const float4 a = src[t];
      v[4 * t] = a.x; v[4 * t + 1] = a.y; v[4 * t + 2] = a.z; v[4 * t + 3] = a.w;
    }
  }
  if (p.cluster) {
    const int cs = p.cluster, RS = BMW / cs;
    cluster_sync_all();
    {
      const int row = q * 32 + lane;
      const int owner = row / RS, rl = row % RS;
      const uint32_t dst = map_to_cta(base + (uint32_t)((split * 16) * RS + rl) * 16, owner);
#pragma unroll
      for (int tq = 0; tq < 16; ++tq) st_cluster_f4(dst + (uint32_t)(tq * RS) * 16, v[4 * tq], v[4 * tq + 1], v[4 * tq + 2], v[4 * tq + 3]);
    }
    cluster_sync_all();
    {
      const int e = warp * 32 + lane;
      const int rl = e % RS, tg = e / RS;
      const int qpt = RS / 8;
      const int n_out = n0 + split * RS + rl;
      const float4 *buf = reinterpret_cast<const float4 *>(sm);
      __nv_bfloat16 *ob = p.out_bf16 + (long long)t0 * p.N;
      for (int tq = tg * qpt; tq < (tg + 1) * qpt; ++tq) {
        float4 a = buf[(0 * 16 + tq) * RS + rl];
        for (int src = 1; src < cs; ++src) {
          const float4 b = buf[(src * 16 + tq) * RS + rl];
          a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        if (p.bias) { const float bs = p.bias[n_out]; a.x += bs; a.y += bs; a.z += bs; a.w += bs; }
        const int tt = 4 * tq;
        if (tt < rows) ob[(long long)tt * p.N + n_out] = __float2bfloat16_rn(a.x);
        if (tt + 1 < rows) ob[(long long)(tt + 1) * p.N + n_out] = __float2bfloat16_rn(a.y);
        if (tt + 2 < rows) ob[(long long)(tt + 2) * p.N + n_out] = __float2bfloat16_rn(a.z);
        if (tt + 3 < rows) ob[(long long)(tt + 3) * p.N + n_out] = __float2bfloat16_rn(a.w);
      }
    }
  } else if (p.silu) {
    __nv_bfloat16 *xu = reinterpret_cast<__nv_bfloat16 *>(sm + SMEM_BAR + 256);
    __nv_bfloat16 *xg = xu + 32 * 64;
    const int rr = (q & 1) * 32 + lane;
    if (q >= 2) {
#pragma unroll
      for (int t = 0; t < 32; ++t) xu[t * 64 + rr] = __float2bfloat16_rn(v[t]);
    } else {
#pragma unroll
      for (int t = 0; t < 32; ++t) xg[t * 64 + rr] = __float2bfloat16_rn(v[32 + t]);
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const int col = tile * 64 + rr;
    const int inter = p.N >> 1;
    __nv_bfloat16 *ob = p.out_bf16 + (long long)t0 * inter;
    const int tb = q < 2 ? 0 : 32;
#pragma unroll
    for (int t = 0; t < 32; ++t) {
      if (tb + t < rows) {
        const float g = q < 2 ? __bfloat162float(__float2bfloat16_rn(v[t])) : __bfloat162float(xg[t * 64 + rr]);
        const float u = q < 2 ? __bfloat162float(xu[t * 64 + rr]) : __bfloat162float(__float2bfloat16_rn(v[32 + t]));
        const float sg = __bfloat162float(__float2bfloat16_rn(g / (1.f + expf(-g))));
        ob[(long long)(tb + t) * inter + col] = __float2bfloat16_rn(sg * u);
      }
    }
  } else if (p.n_split == 1) {
    // no bias: the accumulator is rounded as it is (k_gemm_ws's epilogue; + 0.f would turn a -0 into +0)
    if (p.bias) {
      const float bs = p.bias[n];
#pragma unroll
      for (int t = 0; t < TOK; ++t) v[t] += bs;
    }
    __nv_bfloat16 *ob = p.out_bf16 + (long long)t0 * p.N;
#pragma unroll
    for (int t = 0; t < TOK; ++t)
      if (t < rows) ob[(long long)t * p.N + n] = __float2bfloat16_rn(v[t]);
  } else {
    float *o = p.out_f32 + split * p.slice_stride + (long long)t0 * p.N;
#pragma unroll
    for (int t = 0; t < TOK; ++t)
      if (t < rows) o[(long long)t * p.N + n] = v[t];
  }
}

}  // namespace gemm
}  // namespace pia

using namespace pia;
using namespace pia::gemm;

struct pia_gemm_plan {
  CUtensorMap map_w, map_x;
  Params p;
  int nstage;
  int no_pdl;  // 1: launched without the programmatic-dependent-launch attribute (a plain kernel boundary, like cuBLAS)
  // stream-K mode
  int stream_k, sk_grid;
  SkParams sk;
  // fp8 weight mode (pia_gemm_plan_create_fp8 / _grouped_fp8): k_gemm_fp8 with `f`, up to x_rows rows per run
  int fp8, groups, x_rows;
  F8Params f;
  // int4 weight mode (pia_gemm_plan_create_w4): k_gemm_w4 with `w`, up to x_rows rows per run
  int w4, w4_f16;
  W4Params w;
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult qres;
    void *ptr = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)ptr;
  }
  return fn;
}

// weights pre-tiled in HBM: [N/128 * K/64] contiguous 16 KB blocks of 128 rows x 64 k (one TMA box each), so a CTA
// streams one contiguous slab instead of 128 strided 128-byte pieces per stage
static int encode_tiled_w(CUtensorMap *m, const void *base, uint64_t n_blocks) {
  EncodeTiledFn fn = get_encode();
  PIA_REQUIRE(fn, "cuTensorMapEncodeTiled not available in this driver");
  cuuint64_t dims[3] = {(cuuint64_t)BK, (cuuint64_t)BMW, n_blocks};
  cuuint64_t strides[2] = {(cuuint64_t)BK * 2, (cuuint64_t)BK * BMW * 2};
  cuuint32_t box[3] = {BK, BMW, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return PIA_ERR_CUDA; }
  return PIA_OK;
}

static int encode_2d(CUtensorMap *m, const void *base, uint64_t inner, uint64_t outer, uint32_t box_inner,
                     uint32_t box_outer, CUtensorMapL2promotion promo) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult qres;
    void *ptr = nullptr;
    PIA_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres));
    PIA_REQUIRE(ptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available in this driver");
    fn = (EncodeTiledFn)ptr;
  }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {inner * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return PIA_ERR_CUDA; }
  return PIA_OK;
}

extern "C" int pia_gemm_plan_create(const void *d_w, int N, int K, const void *d_x, int x_rows, int split_k,
                                    int w_tiled, pia_gemm_plan_t **out) {
  PIA_REQUIRE(d_w && d_x && out, "null argument");
  PIA_REQUIRE(N > 0 && K > 0 && K % BK == 0, "K must be a multiple of %d", BK);
  PIA_REQUIRE(x_rows >= TOK, "the activation buffer must hold at least %d rows", TOK);
  PIA_REQUIRE((reinterpret_cast<uintptr_t>(d_w) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_x) & 15) == 0, "operands must be 16-byte aligned");
  pia_gemm_plan *g = new (std::nothrow) pia_gemm_plan();
  PIA_REQUIRE(g, "out of host memory");
  const int n_chunks = K / BK;
  const int want_stream_k = (split_k == -1);
  const int want_cluster = (split_k == -2 || split_k == -4 || split_k == -8) ? -split_k : 0;
  if (split_k < -1 && !want_cluster) { delete g; set_error("cluster split-K supports 2, 4 or 8 CTAs"); return PIA_ERR_INVALID; }
  if (want_cluster) split_k = want_cluster;
  if (split_k < 1) split_k = 1;
  if (split_k > n_chunks) split_k = n_chunks;
  g->p.N = N; g->p.K = K; g->p.n_chunks = n_chunks;
  g->p.chunks_per_split = (n_chunks + split_k - 1) / split_k;
  g->p.n_split = (n_chunks + g->p.chunks_per_split - 1) / g->p.chunks_per_split;
  g->p.rows = TOK; g->p.out_bf16 = nullptr; g->p.out_f32 = nullptr; g->p.silu = 0;
  g->p.groups = 1; g->p.w_group_rows = 0; g->p.x_group_chunks = 0; g->p.out_group_stride = 0;
  g->p.cluster = 0;
  if (want_cluster) {
    if (g->p.n_split != want_cluster) { delete g; set_error("K = %d is too short for %d cluster splits", K, want_cluster); return PIA_ERR_INVALID; }
    g->p.cluster = want_cluster;
  }
  g->p.tiled = w_tiled ? 1 : 0;
  if (w_tiled && N % BMW != 0) { delete g; set_error("a tiled weight needs N %% %d == 0", BMW); return PIA_ERR_INVALID; }
  int rc = w_tiled ? encode_tiled_w(&g->map_w, d_w, (uint64_t)(N / BMW) * n_chunks)
                   : encode_2d(&g->map_w, d_w, (uint64_t)K, (uint64_t)N, BK, BMW, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc == PIA_OK) rc = encode_2d(&g->map_x, d_x, (uint64_t)K, (uint64_t)x_rows, BK, TOK, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc == PIA_OK) {
    int n_sm = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    const int ctas = ((N + BMW - 1) / BMW) * g->p.n_split;
    g->nstage = ctas <= n_sm ? 8 : 4;
    cudaError_t e = cudaFuncSetAttribute(k_gemm_ws<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_total(4));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_gemm_ws<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_total(8));
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); rc = PIA_ERR_CUDA; }
  }
  g->stream_k = 0; g->no_pdl = 0;
  if (rc == PIA_OK && want_stream_k) {
    // stream-K over the HBM-tiled weight: grid = min(#SMs, units), fix-up workspace owned by the plan
    if (!w_tiled) { delete g; set_error("stream-K needs the tiled weight layout"); return PIA_ERR_INVALID; }
    int n_sm = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    SkParams &k = g->sk;
    k.N = N; k.n_tiles = N / BMW; k.n_chunks = n_chunks; k.rows = TOK;
    k.units = (long long)k.n_tiles * n_chunks;
    g->sk_grid = (int)(k.units < n_sm ? k.units : n_sm);
    // contributor slots of a tile = the CTAs after its owner that hold some of its chunks.  The ranges are
    // floor(U/G) or ceil(U/G) units long, so the count is read off the partition itself, tile by tile.
    k.max_contrib = 1;
    for (int t = 0; t < k.n_tiles; ++t) {
      const long long ts = (long long)t * n_chunks;
      const int c = sk_cta_of(ts + n_chunks - 1, k.units, g->sk_grid) - sk_cta_of(ts, k.units, g->sk_grid);
      if (c > k.max_contrib) k.max_contrib = c;
    }
    k.out = nullptr;
    cudaError_t e = cudaMalloc((void **)&k.ws, sizeof(float) * (size_t)k.n_tiles * k.max_contrib * BMW * TOK);
    if (e == cudaSuccess) e = cudaMalloc((void **)&k.flags, sizeof(int) * k.n_tiles);
    if (e == cudaSuccess) e = cudaMemset(k.flags, 0, sizeof(int) * k.n_tiles);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_gemm_sk, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM_TOTAL);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("stream-K plan: %s", cudaGetErrorString(e)); delete g; return PIA_ERR_CUDA; }
    g->stream_k = 1;
    g->p.n_split = 1;
  }
  if (rc != PIA_OK) { delete g; return rc; }
  *out = g;
  return PIA_OK;
}

extern "C" int pia_gemm_plan_destroy(pia_gemm_plan_t *g) {
  if (g) {
    if (g->stream_k) { cudaFree(g->sk.ws); cudaFree(g->sk.flags); }
    delete g;
  }
  return PIA_OK;
}
extern "C" int pia_gemm_plan_set_pdl(pia_gemm_plan_t *g, int on) {
  PIA_REQUIRE(g, "null plan");
  g->no_pdl = on ? 0 : 1;
  return PIA_OK;
}
extern "C" int pia_gemm_plan_splits(const pia_gemm_plan_t *g) {
  if (g && g->fp8) return g->f.cluster ? 1 : g->f.n_split;
  if (g && g->w4) return g->w.cluster ? 1 : g->w.n_split;
  return g ? (g->p.cluster ? 1 : g->p.n_split) : 0;
}
extern "C" int pia_gemm_plan_set_silu(pia_gemm_plan_t *g, int on) {
  if (g && g->fp8) {
    PIA_REQUIRE(g->f.n_split == 1 && !g->f.bias && g->groups == 1,
                "the SiLU*up epilogue needs split_k == 1, no bias and one group");
    PIA_REQUIRE(!on || !g->f.relu, "a plan has one epilogue activation: ReLU is already set");
    g->f.silu = on ? 1 : 0;
    return PIA_OK;
  }
  if (g && g->w4) {
    PIA_REQUIRE(g->w.n_split == 1 && !g->w.bias, "the SiLU*up epilogue needs split_k == 1 and no bias");
    g->w.silu = on ? 1 : 0;
    return PIA_OK;
  }
  PIA_REQUIRE(g && g->p.n_split == 1 && !g->stream_k && g->p.N % BMW == 0, "the SiLU*up epilogue needs split_k == 1 and N %% 128 == 0");
  g->p.silu = on ? 1 : 0;
  return PIA_OK;
}
extern "C" int pia_gemm_plan_set_relu(pia_gemm_plan_t *g, int on) {
  PIA_REQUIRE(g && g->fp8, "the ReLU epilogue exists on fp8 plans only");
  if (on) {
    PIA_REQUIRE(g->f.n_split == 1 || g->f.cluster, "the ReLU epilogue needs bf16 outputs: split_k == 1 or a cluster split");
    PIA_REQUIRE(!g->f.silu, "a plan has one epilogue activation: SiLU*up is already set");
  }
  g->f.relu = on ? 1 : 0;
  return PIA_OK;
}

// Grouped GEMM (MoE experts, mixtral/modeling_mixtral.py:692-759): out[g] = X[:, g*K:(g+1)*K] @ W[g]^T for `groups`
// stacked weights W [groups*N, K] (row-major) and activations X [x_rows, groups*K]; one launch, gridDim.z = groups.
extern "C" int pia_gemm_plan_create_grouped(const void *d_w, int groups, int N, int K, const void *d_x, int x_rows,
                                            pia_gemm_plan_t **out) {
  PIA_REQUIRE(d_w && d_x && out, "null argument");
  PIA_REQUIRE(groups >= 1 && groups <= 65535 && N > 0 && N % BMW == 0 && K > 0 && K % BK == 0,
              "grouped GEMM needs N %% %d == 0 and K %% %d == 0", BMW, BK);
  PIA_REQUIRE(x_rows >= TOK, "the activation buffer must hold at least %d rows", TOK);
  PIA_REQUIRE((reinterpret_cast<uintptr_t>(d_w) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_x) & 15) == 0, "operands must be 16-byte aligned");
  pia_gemm_plan *g = new (std::nothrow) pia_gemm_plan();
  PIA_REQUIRE(g, "out of host memory");
  const int n_chunks = K / BK;
  g->p.N = N; g->p.K = K; g->p.n_chunks = n_chunks; g->p.chunks_per_split = n_chunks; g->p.n_split = 1;
  g->p.rows = TOK; g->p.out_bf16 = nullptr; g->p.out_f32 = nullptr; g->p.silu = 0; g->p.tiled = 0; g->p.cluster = 0;
  g->p.groups = groups; g->p.w_group_rows = N; g->p.x_group_chunks = n_chunks; g->p.out_group_stride = (long long)TOK * N;
  g->stream_k = 0; g->no_pdl = 0;
  int rc = encode_2d(&g->map_w, d_w, (uint64_t)K, (uint64_t)groups * N, BK, BMW, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc == PIA_OK) rc = encode_2d(&g->map_x, d_x, (uint64_t)groups * K, (uint64_t)x_rows, BK, TOK, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc == PIA_OK) {
    int n_sm = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    g->nstage = (N / BMW) * groups <= n_sm ? 8 : 4;
    cudaError_t e = cudaFuncSetAttribute(k_gemm_ws<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_total(4));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_gemm_ws<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_total(8));
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); rc = PIA_ERR_CUDA; }
  }
  if (rc != PIA_OK) { delete g; return rc; }
  *out = g;
  return PIA_OK;
}

// fp8 weights, tiled by ops.tile_weight_fp8: [groups][N/128][K/128] contiguous 16 KB blocks of 128 rows x 128 e4m3
// bytes, one SWIZZLE_128B TMA box each
static int encode_tiled_w_fp8(CUtensorMap *m, const void *base, uint64_t n_blocks) {
  EncodeTiledFn fn = get_encode();
  PIA_REQUIRE(fn, "cuTensorMapEncodeTiled not available in this driver");
  cuuint64_t dims[3] = {(cuuint64_t)F8_BK, (cuuint64_t)BMW, n_blocks};
  cuuint64_t strides[2] = {(cuuint64_t)F8_BK, (cuuint64_t)F8_BK * BMW};
  cuuint32_t box[3] = {F8_BK, BMW, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void *>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return PIA_ERR_CUDA; }
  return PIA_OK;
}

static int f8_plan_create(const void *d_w, const void *d_scale, const void *d_bias, int groups, int N, int K,
                          const void *d_x, int x_rows, int split_k, pia_gemm_plan_t **out) {
  PIA_REQUIRE(d_w && d_scale && d_x && out, "null argument");
  PIA_REQUIRE(groups >= 1 && groups <= 4096 && N > 0 && N % BMW == 0 && K > 0 && K % F8_BK == 0,
              "the fp8 GEMM needs N %% %d == 0 and K %% %d == 0", BMW, F8_BK);
  PIA_REQUIRE(x_rows >= TOK, "the activation buffer must hold at least %d rows", TOK);
  PIA_REQUIRE((reinterpret_cast<uintptr_t>(d_w) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_x) & 15) == 0, "operands must be 16-byte aligned");
  const int n_chunks = K / F8_BK;
  const int want_cluster = (split_k == -2 || split_k == -4 || split_k == -8) ? -split_k : 0;
  PIA_REQUIRE(split_k >= 1 || want_cluster, "fp8 plans take split_k >= 1 or a cluster split of 2, 4 or 8 CTAs");
  PIA_REQUIRE(groups == 1 || split_k == 1, "a grouped fp8 plan has one K split");
  if (want_cluster) split_k = want_cluster;
  if (split_k > n_chunks) split_k = n_chunks;
  pia_gemm_plan *g = new (std::nothrow) pia_gemm_plan();
  PIA_REQUIRE(g, "out of host memory");
  F8Params &f = g->f;
  f.N = N; f.n_chunks = n_chunks; f.tiles = N / BMW;
  f.chunks_per_split = (n_chunks + split_k - 1) / split_k;
  f.n_split = (n_chunks + f.chunks_per_split - 1) / f.chunks_per_split;
  f.rows = TOK; f.ntb = 1;
  f.x_group_chunks = groups > 1 ? n_chunks : 0;
  f.out_group_stride = (long long)x_rows * N;
  f.slice_stride = (long long)x_rows * N;
  f.cluster = 0; f.silu = 0; f.no_pdl = 0; f.relu = 0;
  f.scale = (const float *)d_scale; f.bias = (const float *)d_bias;
  f.out_bf16 = nullptr; f.out_f32 = nullptr;
  if (want_cluster && f.n_split != want_cluster) { delete g; set_error("K = %d is too short for %d cluster splits", K, want_cluster); return PIA_ERR_INVALID; }
  f.cluster = want_cluster;
  if (d_bias && f.n_split > 1 && !f.cluster) { delete g; set_error("a bias needs split_k == 1 or a cluster split"); return PIA_ERR_INVALID; }
  g->fp8 = 1; g->groups = groups; g->x_rows = x_rows;
  int rc = encode_tiled_w_fp8(&g->map_w, d_w, (uint64_t)groups * f.tiles * n_chunks);
  if (rc == PIA_OK) rc = encode_2d(&g->map_x, d_x, (uint64_t)groups * K, (uint64_t)x_rows, BK, TOK, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc == PIA_OK) {
    int n_sm = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    g->nstage = f.tiles * f.n_split * groups <= n_sm ? 6 : 3;
    cudaError_t e = cudaFuncSetAttribute(k_gemm_fp8<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, f8_smem_total(3));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_gemm_fp8<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, f8_smem_total(6));
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); rc = PIA_ERR_CUDA; }
  }
  if (rc != PIA_OK) { delete g; return rc; }
  *out = g;
  return PIA_OK;
}

extern "C" int pia_gemm_plan_create_fp8(const void *d_w, const void *d_scale, const void *d_bias, int N, int K,
                                        const void *d_x, int x_rows, int split_k, pia_gemm_plan_t **out) {
  return f8_plan_create(d_w, d_scale, d_bias, 1, N, K, d_x, x_rows, split_k, out);
}

extern "C" int pia_gemm_plan_create_grouped_fp8(const void *d_w, const void *d_scale, int groups, int N, int K,
                                                const void *d_x, int x_rows, pia_gemm_plan_t **out) {
  return f8_plan_create(d_w, d_scale, nullptr, groups, N, K, d_x, x_rows, 1, out);
}

// int4 codes, tiled by ops.tile_weight_w4: [N/128][ceil(K/256)] contiguous 16 KB blocks of 128 rows x 128 bytes (256
// nibbles), one SWIZZLE_128B TMA box each
static int w4_plan_create(const void *d_codes, const void *d_scale, const void *d_zero, int scale_f16,
                          const void *d_bias, int N, int K, int group, const void *d_x, int x_rows, int split_k,
                          pia_gemm_plan_t **out) {
  PIA_REQUIRE(d_codes && d_scale && d_zero && d_x && out, "null argument");
  PIA_REQUIRE(N > 0 && N % BMW == 0 && K > 0 && K % 128 == 0, "the int4 GEMM needs N %% %d == 0 and K %% 128 == 0", BMW);
  PIA_REQUIRE(group > 0 && group % 128 == 0 && K % group == 0, "group size %d: a multiple of 128 that divides K = %d", group, K);
  PIA_REQUIRE(scale_f16 == 0 || scale_f16 == 1, "scale dtype: 0 = bf16, 1 = fp16");
  PIA_REQUIRE(x_rows >= TOK, "the activation buffer must hold at least %d rows", TOK);
  PIA_REQUIRE(((reinterpret_cast<uintptr_t>(d_codes) | reinterpret_cast<uintptr_t>(d_scale) |
                reinterpret_cast<uintptr_t>(d_zero) | reinterpret_cast<uintptr_t>(d_x)) & 15) == 0,
              "operands must be 16-byte aligned");
  const int n_chunks = (K + W4_BK - 1) / W4_BK;
  const int want_cluster = (split_k == -2 || split_k == -4 || split_k == -8) ? -split_k : 0;
  PIA_REQUIRE(split_k >= 1 || want_cluster, "int4 plans take split_k >= 1 or a cluster split of 2, 4 or 8 CTAs");
  if (want_cluster) split_k = want_cluster;
  if (split_k > n_chunks) split_k = n_chunks;
  W4Params w;
  w.N = N; w.K = K; w.n_chunks = n_chunks; w.tiles = N / BMW; w.group = group;
  w.chunks_per_split = (n_chunks + split_k - 1) / split_k;
  w.n_split = (n_chunks + w.chunks_per_split - 1) / w.chunks_per_split;
  w.rows = TOK; w.ntb = 1;
  w.slice_stride = (long long)x_rows * N;
  w.cluster = 0; w.silu = 0; w.no_pdl = 0;
  w.scale = d_scale; w.zero = (const uint8_t *)d_zero; w.bias = (const float *)d_bias;
  w.out_bf16 = nullptr; w.out_f32 = nullptr;
  if (want_cluster && w.n_split != want_cluster) { set_error("K = %d is too short for %d cluster splits", K, want_cluster); return PIA_ERR_INVALID; }
  w.cluster = want_cluster;
  if (d_bias && w.n_split > 1 && !w.cluster) { set_error("a bias needs split_k == 1 or a cluster split"); return PIA_ERR_INVALID; }
  pia_gemm_plan *g = new (std::nothrow) pia_gemm_plan();
  PIA_REQUIRE(g, "out of host memory");
  g->w = w; g->w4 = 1; g->w4_f16 = scale_f16; g->groups = 1; g->x_rows = x_rows;
  int rc = encode_tiled_w_fp8(&g->map_w, d_codes, (uint64_t)w.tiles * n_chunks);   // the same 128 x 128-byte boxes
  if (rc == PIA_OK) rc = encode_2d(&g->map_x, d_x, (uint64_t)K, (uint64_t)x_rows, BK, TOK, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (rc == PIA_OK) {
    int n_sm = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    g->nstage = w.tiles * w.n_split <= n_sm ? 4 : 2;
    cudaError_t e = cudaFuncSetAttribute(k_gemm_w4<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, w4_smem_total(2));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_gemm_w4<4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, w4_smem_total(4));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_gemm_w4<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, w4_smem_total(2));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_gemm_w4<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, w4_smem_total(4));
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); rc = PIA_ERR_CUDA; }
  }
  if (rc != PIA_OK) { delete g; return rc; }
  *out = g;
  return PIA_OK;
}

extern "C" int pia_gemm_plan_create_w4(const void *d_codes, const void *d_scale, const void *d_zero, int scale_dtype,
                                       const void *d_bias, int N, int K, int group_size, const void *d_x, int x_rows,
                                       int split_k, pia_gemm_plan_t **out) {
  return w4_plan_create(d_codes, d_scale, d_zero, scale_dtype, d_bias, N, K, group_size, d_x, x_rows, split_k, out);
}

struct PdlScope { int on; explicit PdlScope(int off) : on(off) { if (on) ++pia::g_pdl_off; } ~PdlScope() { if (on) --pia::g_pdl_off; } };

static int f8_run(pia_gemm_plan_t *g, int rows, void *d_out, void *stream) {
  PIA_REQUIRE(rows >= 1 && rows <= g->x_rows, "rows %d outside [1,%d]", rows, g->x_rows);
  PdlScope pdl_scope(g->no_pdl);
  F8Params f = g->f;
  f.rows = rows; f.ntb = (rows + TOK - 1) / TOK; f.no_pdl = g->no_pdl;
  if (f.n_split == 1 || f.cluster) f.out_bf16 = (__nv_bfloat16 *)d_out; else f.out_f32 = (float *)d_out;
  const unsigned z = (unsigned)(g->groups * f.ntb);
  const dim3 grid = f.cluster ? dim3(f.n_split, f.tiles, z) : dim3(f.tiles, f.n_split, z);
  const unsigned cs = f.cluster ? (unsigned)f.cluster : 1u;
  if (g->nstage == 6) PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_fp8<6>, grid, dim3(NTHREADS), f8_smem_total(6), (cudaStream_t)stream, cs, g->map_w, g->map_x, f));
  else PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_fp8<3>, grid, dim3(NTHREADS), f8_smem_total(3), (cudaStream_t)stream, cs, g->map_w, g->map_x, f));
  count_launch();
  return PIA_OK;
}

static int w4_run(pia_gemm_plan_t *g, int rows, void *d_out, void *stream) {
  PIA_REQUIRE(rows >= 1 && rows <= g->x_rows, "rows %d outside [1,%d]", rows, g->x_rows);
  PdlScope pdl_scope(g->no_pdl);
  W4Params w = g->w;
  w.rows = rows; w.ntb = (rows + TOK - 1) / TOK; w.no_pdl = g->no_pdl;
  if (w.n_split == 1 || w.cluster) w.out_bf16 = (__nv_bfloat16 *)d_out; else w.out_f32 = (float *)d_out;
  const dim3 grid = w.cluster ? dim3(w.n_split, w.tiles, w.ntb) : dim3(w.tiles, w.n_split, w.ntb);
  const unsigned cs = w.cluster ? (unsigned)w.cluster : 1u;
  const cudaStream_t st = (cudaStream_t)stream;
  if (g->nstage == 4) {
    if (g->w4_f16) PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_w4<4, true>, grid, dim3(NTHREADS), w4_smem_total(4), st, cs, g->map_w, g->map_x, w));
    else PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_w4<4, false>, grid, dim3(NTHREADS), w4_smem_total(4), st, cs, g->map_w, g->map_x, w));
  } else {
    if (g->w4_f16) PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_w4<2, true>, grid, dim3(NTHREADS), w4_smem_total(2), st, cs, g->map_w, g->map_x, w));
    else PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_w4<2, false>, grid, dim3(NTHREADS), w4_smem_total(2), st, cs, g->map_w, g->map_x, w));
  }
  count_launch();
  return PIA_OK;
}

extern "C" int pia_gemm_run(pia_gemm_plan_t *g, int rows, void *d_out, void *stream) {
  PIA_REQUIRE(g && d_out, "null argument");
  if (g->fp8) return f8_run(g, rows, d_out, stream);
  if (g->w4) return w4_run(g, rows, d_out, stream);
  PIA_REQUIRE(rows >= 1 && rows <= TOK, "rows %d outside [1,%d]", rows, TOK);
  PdlScope pdl_scope(g->no_pdl);
  if (g->stream_k) {
    SkParams k = g->sk;
    k.rows = rows;
    k.out = (__nv_bfloat16 *)d_out;
    PIA_CUDA_CHECK(launch_kernel(k_gemm_sk, dim3(g->sk_grid), dim3(NTHREADS), SK_SMEM_TOTAL, (cudaStream_t)stream, g->map_w, g->map_x, k));
    count_launch();
    return PIA_OK;
  }
  Params p = g->p;
  p.rows = rows; p.no_pdl = g->no_pdl;
  if (p.n_split == 1 || p.cluster) p.out_bf16 = (__nv_bfloat16 *)d_out; else p.out_f32 = (float *)d_out;
  if (p.cluster) {
    dim3 cgrid(p.n_split, (p.N + BMW - 1) / BMW);
    if (g->nstage == 8) PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_ws<8>, cgrid, dim3(NTHREADS), smem_total(8), (cudaStream_t)stream, (unsigned)p.cluster, g->map_w, g->map_x, p));
    else PIA_CUDA_CHECK(launch_kernel_cluster(k_gemm_ws<4>, cgrid, dim3(NTHREADS), smem_total(4), (cudaStream_t)stream, (unsigned)p.cluster, g->map_w, g->map_x, p));
    count_launch();
    return PIA_OK;
  }
  dim3 grid((p.N + BMW - 1) / BMW, p.n_split, p.groups);
  if (g->nstage == 8) PIA_CUDA_CHECK(launch_kernel(k_gemm_ws<8>, grid, dim3(NTHREADS), smem_total(8), (cudaStream_t)stream, g->map_w, g->map_x, p));
  else PIA_CUDA_CHECK(launch_kernel(k_gemm_ws<4>, grid, dim3(NTHREADS), smem_total(4), (cudaStream_t)stream, g->map_w, g->map_x, p));
  count_launch();
  return PIA_OK;
}
