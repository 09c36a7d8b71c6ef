// Tree-masked attention for the LOOKAHEAD verify forward (sm_90a: TMA + wgmma).
//
// Takes over the eager attention of the reference's patched models
//   models/llama/modeling_llama.py:243-308 (QK^T/sqrt(d) + mask, fp32 softmax, PV) with the lookahead mask of
//   :584-588 and common/pretrained_model.py:725-734 ([n, P+n] = visible prefix || tree mask).
// The mask is never materialised: prefix keys [pad_len, P) are visible to every row, the n draft keys follow the
// row's ancestor bit set (uint64 words, produced by the trie kernel) held in registers.
//
// One CTA = (KV split, head group).  A head group is up to two query heads of ONE KV head packed into a single 128-row
// tile: at 64 draft rows the G = Hq / Hkv query heads of a KV head fill ceil(G / 2) tiles of 2 heads, the last tile
// holding 1 head when G is odd (and the only one under MHA: rows 64..127 idle); at 128 draft rows 1 head per tile.
// Warp roles (288 threads):  warps 0-7 = two consumer warpgroups, each owning 64 rows (wgmma M = 64): they stage Q
//                            (and, fused, the draft tile), issue the MMAs and run the softmax in registers,
//                            warp 8 = TMA producer (K/V tiles of 128 keys, 2-stage ring, V on its own barriers).
// Per 128-key tile and warpgroup:  S = Q K^T (HD / 16 x wgmma m64n128k16, both operands from shared memory, fp32 in
//                    registers) -> hidden keys to -inf (one 32-bit visibility word per 32 keys), online softmax in
//                    fp32 -> P (bf16 pairs) stays in registers: the S accumulator layout is the A-fragment layout of
//                    -> O += P V (8 x wgmma m64n{HD}k16, A from registers, V consumed MN-major straight from the
//                    TMA tile).  The producer keeps the next tile's K/V in flight while a tile is computed.
// The kernel is a template on the head dim HD (64 or 128; the plan picks the instance): a 128-row operand tile is
// HD / 64 SWIZZLE_128B sub-tiles of 64 bf16 columns (one TMA box each), and the O accumulator holds HD / 2 fp32.
// The KV range is split across the CTAs of a thread-block cluster (one wave of clusters, split count decided on the
// device from the live length): a single-split CTA normalises and writes bf16 directly; otherwise every thread
// pushes its partial rows (acc, m, l) into the shared memory of the CTA that owns the row (DSMEM) and each CTA
// combines its row slice locally - no workspace in HBM, no separate combine launch.
// HBM-bound by design (arithmetic intensity = rows per KV byte: 64 FLOP/B for MHA, 256 for GQA-4;
// DESIGN.md gives the roofline).
#include <cuda.h>
#include <cuda_bf16.h>

#include <stdlib.h>

#include <new>

#include "common.cuh"

namespace pia {
namespace attn {

constexpr int BN = 128;      // keys per tile (wgmma N of QK^T, K extent of PV)
constexpr int NSTAGE = 2;
constexpr int NTHREADS = 288;   // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int PRODUCER_WARP = 8;
constexpr int SUB = 128 * 128;             // bytes of one [128 rows x 64 bf16] swizzle-128B sub-tile
constexpr int MAX_SPLIT = 8;            // KV splits per head group (merge keeps all partial rows in flight)
constexpr int ALIBI_SLOPE = 64;         // ALiBi instance, offsets from the barriers: 2 fp32 slopes (one per warpgroup),
constexpr int ALIBI_DEPTH = 128;        //   and the uint8 depth of each draft node
constexpr float LOG2E = 1.4426950408889634f;

// Shared-memory layout of the head-dim HD instance (HD = 128: two sub-tiles per operand tile, HD = 64: one)
template <int HD>
struct Smem {
  static constexpr int TILE_BYTES = HD / 64 * SUB;  // one 128 x HD bf16 operand tile
  static constexpr int Q = 0, K = TILE_BYTES, V = K + NSTAGE * TILE_BYTES;
  static constexpr int BAR = V + NSTAGE * TILE_BYTES;
  static constexpr int MRG_ACC = 0;                  // [HD / 4 chunks][128 + MAX_SPLIT] float4 partial rows pushed by the cluster (over dead Q/KV tiles)
  static constexpr int MRG_ML = 7 * TILE_BYTES / 2;  // [n_split * RS] (m, l) pairs (112 KB at HD = 128)
  // merge buffers that never alias a live tile (used when the CTA's rows fit: <= 64 rows): peers may push their
  // partial rows as soon as they are done, without first waiting for this CTA to leave its tile loop
  static constexpr int DED_ACC = BAR + 256, DED_ACC_BYTES = (64 + MAX_SPLIT) * HD * 4,  // ns * ceil(64 / ns) <= 64 + MAX_SPLIT - 1 rows
                       DED_ML = DED_ACC + DED_ACC_BYTES;
  static constexpr int TOTAL = DED_ML + 1024 + 1024;  // + alignment slack
  // the aliased merge area lies inside the Q / K / V tiles, which are dead once every CTA has left its tile loop
  static_assert(MRG_ACC + HD / 4 * (128 + MAX_SPLIT) * 16 <= MRG_ML, "aliased partial rows overlap the (m, l) pairs");
  static_assert(MRG_ML + (128 + MAX_SPLIT) * 8 <= BAR, "aliased merge area reaches the barriers");
  // the ALiBi depths (one byte per draft key) sit between the 3 x NSTAGE barriers and the dedicated merge buffers
  static_assert(3 * NSTAGE * 8 <= ALIBI_SLOPE && ALIBI_SLOPE + 8 <= ALIBI_DEPTH && BAR + ALIBI_DEPTH + 128 <= DED_ACC,
                "ALiBi slopes / depths overlap");
};

// ------------------------------------------------------------------------------------------------ PTX
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
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// registers a wgmma reads or writes asynchronously: pins every later access after the wait above
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void fence_regs(uint32_t (&a)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+r"(a[i])::"memory");
}
// D[64 x 128] += A[64 x 16] B[16 x 128]: A = Q (K-major, shared memory), B = K tile (K-major, shared memory)
__device__ __forceinline__ void wgmma_qk(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}
// D[64 x 128] += P[64 x 16] V[16 x 128]: A = P (bf16 pairs in registers), B = V tile (MN-major, shared memory)
__device__ __forceinline__ void wgmma_pv(float (&d)[64], const uint32_t *a, uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, 1, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
      : "memory");
}
// D[64 x 64] += P[64 x 16] V[16 x 64]: the head-dim-64 PV (one V sub-tile)
__device__ __forceinline__ void wgmma_pv(float (&d)[32], const uint32_t *a, uint64_t desc_b) {
  asm volatile(
      "{\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
      : "memory");
}
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_smem_addr, uint32_t cta_rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta_rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f2(uint32_t addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory matrix descriptor (sm_90 GMMA descriptor), SWIZZLE_128B
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}

union Pack8 { uint4 u; __nv_bfloat16 h[8]; };
__device__ __forceinline__ float bfr(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
// x * cos + rotate_half(x) * sin for 8 elements, every product / sum rounded to bf16 (k_rope_kv_append's arithmetic,
// modeling_llama.py:167-168); `lower` = these elements lie in the first half of the head (partner enters negated)
__device__ __forceinline__ uint4 rope8(uint4 xa, uint4 xb, uint4 cs, uint4 sn, bool lower) {
  Pack8 a, b, c, s, o;
  a.u = xa; b.u = xb; c.u = cs; s.u = sn;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float x = __bfloat162float(a.h[j]);
    const float r = lower ? -__bfloat162float(b.h[j]) : __bfloat162float(b.h[j]);
    o.h[j] = __float2bfloat16_rn(bfr(x * __bfloat162float(c.h[j])) + bfr(r * __bfloat162float(s.h[j])));
  }
  return o.u;
}

struct Params {
  const __nv_bfloat16 *q;  // [max_nodes, Hq, HD]
  const unsigned long long *mask;
  pia_slots_t sl;          // request slots: blockIdx.z = slot (rows, n, P, pad and KV planes of that slot)
  int slot_planes;         // KV planes between consecutive slots' caches (0: shared cache)
  int plane0;              // first plane of the cache slot 0 addresses
  int layer, n_q_heads, n_kv_heads, np, mask_words, heads_per_cta, max_seq, n_split, tiles_per_cta;
  int ctas_per_kv;         // head groups per KV head: ceil(G / heads_per_cta); heads_per_cta = 2 at 64 draft rows, 1 at 128
  float scale_log2;
  // fused mode (pia_tree_attn_fused_fwd): RoPE + KV append happen here.  Q and the draft nodes' K / V come straight from
  // the fused projection output, the draft keys are one extra tile built in shared memory, the cache only holds [0, P)
  int fused;
  const __nv_bfloat16 *qkv;      // [rows, (Hq + 2 Hkv) * HD]
  const __nv_bfloat16 *cos_t, *sin_t;  // [max_pos, HD / 2] bf16 (as k_rope_kv_append)
  int max_pos;
  __nv_bfloat16 *kc_layer, *vc_layer;  // this layer's [Hkv, max_seq, HD] planes of the cache slot 0 addresses
  __nv_bfloat16 *out;            // [max_nodes, Hq, HD]
  unsigned long long *dbg;       // optional per-CTA phase timestamps (pia_attn_plan_set_debug)
  const float *slopes;           // ALiBi instance (pia_tree_attn_alibi_fwd): [Hq] fp32 slopes
};

__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// head group (blockIdx.y) -> KV head hkv, its j-th tile of query heads, first query head hq0 and heads in the tile:
// the G query heads of a KV head fill ceil(G / heads_per_cta) tiles, the last one holding a single head when G is odd
struct HeadGroup { int hkv, j, hq0, heads; };
__device__ __forceinline__ HeadGroup head_group(const Params &p, int group) {
  const int G = p.n_q_heads / p.n_kv_heads;
  HeadGroup g;
  g.hkv = group / p.ctas_per_kv;
  g.j = group - g.hkv * p.ctas_per_kv;
  g.hq0 = g.hkv * G + g.j * p.heads_per_cta;
  g.heads = min(p.heads_per_cta, G - g.j * p.heads_per_cta);
  return g;
}

#define DBG(ev) do { if (p.dbg) p.dbg[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 16 + (ev)] = gtime(); } while (0)

// kAlibi (HD = 128 only, plain mode only): every score gets the linear position bias slope_h * (kpos - qpos) of ALiBi
// (baichuan_13b/modeling_baichuan.py:25-36, :146-157) at TREE positions, as the reference's BLOOM patch computes them
// (bloom/modeling_bloom.py:170): qpos = max(P - pad, 0) + depth(row) - 1, kpos = j - pad for a cached key j < P and
// max(P - pad, 0) + depth(k) - 1 for draft key k.  The row offset does not change the softmax, so this is the models'
// absolute slope_h * kpos; the verify logits of every node equal a causal forward over prefix + root-to-node path.
template <int HD, bool kAlibi>
__global__ void __launch_bounds__(NTHREADS, 1)
k_tree_attn(const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v, Params p) {
  constexpr int TILE_BYTES = Smem<HD>::TILE_BYTES, SMEM_Q = Smem<HD>::Q, SMEM_K = Smem<HD>::K, SMEM_V = Smem<HD>::V;
  constexpr int SMEM_BAR = Smem<HD>::BAR, MRG_ACC = Smem<HD>::MRG_ACC, MRG_ML = Smem<HD>::MRG_ML;
  constexpr int MRG_DED_ACC = Smem<HD>::DED_ACC, MRG_DED_ACC_BYTES = Smem<HD>::DED_ACC_BYTES, MRG_DED_ML = Smem<HD>::DED_ML;
  // staging splits a head row into two halves (the RoPE rotation pairs them) of CH 16-byte chunks; in the K-major
  // SWIZZLE_128B tile of 64-wide sub-tiles, half h starts h * HALF_SUB bytes and h * HALF_CH chunks into its rows
  constexpr int CH = HD / 16, HALF_SUB = HD == 128 ? SUB : 0, HALF_CH = HD == 128 ? 0 : CH;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t *sm = smem_raw + (base - smem_u32(smem_raw));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  const uint32_t bar0 = base + SMEM_BAR;
  // V tiles complete on their own barriers: QK^T starts as soon as K has landed
  const uint32_t bar_kv_full = bar0, bar_kv_empty = bar0 + 8 * NSTAGE, bar_v_full = bar0 + 16 * NSTAGE;

  pdl_launch_dependents();
  if (tid == 0) {  // the two TMA descriptors are fetched while the barriers are set up
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<unsigned long long>(&map_k)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<unsigned long long>(&map_v)) : "memory");
  }
  // Programmatic dependent launch: this CTA may be running while its predecessor (RoPE + KV append of the same layer)
  // still is.  What is read BEFORE griddepcontrol.wait is safe to read early: d_n / d_prefix_len / d_pad_len were
  // written before the first kernel of the layer chain (trie get and the previous step's accept are launched without
  // the PDL attribute, prefill meta is a stream-ordered copy), and cache rows below P were written by earlier steps.
  // Only Q, the rows [P, P + n) of this layer's K/V planes and the output buffer depend on the predecessor: the TMA
  // producer waits before its first tile that reaches row P, the consumer warps wait before they read Q.
  const int split = blockIdx.x, group = blockIdx.y;
  const int slot = blockIdx.z;
  const int n = p.sl.d_n[slot], P = p.sl.d_prefix_len[slot];
  const int pad_len = p.sl.d_pad_len ? p.sl.d_pad_len[slot] : 0;
  if (n <= 0) return;      // idle slot: every CTA of its clusters takes this exit
  const long long row0 = (long long)slot * p.sl.rows_per_slot;  // first activation / mask row of the slot
  const int L = P + n;
  const HeadGroup hg = head_group(p, group);
  const int hkv = hg.hkv, hq0 = hg.hq0, heads_here = hg.heads;
  // tiles: plain mode = the keys [0, L) of the cache; fused mode = the prefix tiles [0, P) of the cache + ONE draft tile
  // (the n draft keys, rotated and staged in shared memory by the consumer warps of the CTA that owns the last tile)
  const bool fused = !kAlibi && p.fused != 0;
  const int Tp = (P + BN - 1) / BN;
  const int tiles_total = fused ? Tp + 1 : (L + BN - 1) / BN;
  // Work split decided on the device from the live length: tiles_per_cta tiles per CTA (more only when the
  // plan's split limit is reached); a single split writes the final output directly (no partials, no merge).
  const int rows_used = heads_here * p.np;               // 64 (one head of 64 nodes) or 128
  const int n_wg = rows_used / 64;                       // consumer warpgroups with live rows
  const bool ded = (rows_used + MAX_SPLIT) * HD * 4 <= MRG_DED_ACC_BYTES;
  int ns = (tiles_total + p.tiles_per_cta - 1) / p.tiles_per_cta;
  if (ns > p.n_split) ns = p.n_split;
  if (ns < 1) ns = 1;
  if (split >= ns) {
    if (ns > 1) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }
  const int tps = (tiles_total + ns - 1) / ns;
  const int t0 = split * tps;
  int t1 = t0 + tps;
  if (t1 > tiles_total) t1 = tiles_total;
  const int ntile = t1 - t0;  // >= 1 for split < ns except possibly the last one
  // the CTA that owns the last tile takes the draft tile FIRST (slot 0 of the ring is free at kernel start; the order of
  // tiles does not matter to the online softmax) and its prefix tiles after it
  const bool has_draft = fused && ntile > 0 && t1 == tiles_total;
  auto tile_of = [&](int i) -> int { return has_draft ? (i == 0 ? Tp : t0 + i - 1) : t0 + i; };
  // cluster barrier A ("every CTA of the cluster is running and its merge buffers may be written"): with dedicated
  // merge buffers the arrive happens right here and the wait just before the push (it has long completed by then);
  // with aliased buffers (128-row tiles) A is a full barrier after the tile loop
  if (ns > 1 && ded) cluster_arrive();
  auto barrier_a = [&]() { if (ded) cluster_wait(); else cluster_sync_all(); };
  const int mrg_acc = ded ? MRG_DED_ACC : MRG_ACC, mrg_ml = ded ? MRG_DED_ML : MRG_ML;
  const int mrg_stride = ded ? 64 + MAX_SPLIT : 128 + MAX_SPLIT;  // slots per chunk column
  if (tid == 0) DBG(0);

  // ---- setup
  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      mbar_init(bar_kv_full + 8 * s, 1); mbar_init(bar_v_full + 8 * s, 1);
      mbar_init(bar_kv_empty + 8 * s, 4 * n_wg);  // one arrive per consumer warp with live rows
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  __syncthreads();
  if (tid == 0) DBG(1);

  if (warp == PRODUCER_WARP) {
    // ================================================================ TMA producer
    if (lane == 0 && ntile > 0) {
      const int plane = p.plane0 + slot * p.slot_planes + p.layer * p.n_kv_heads + hkv;
      // rows the predecessor may still be appending start at P - or, when the slots share one cache (the chain chunks
      // of a prefill pass: chunk c's prefix holds what the same RoPE launch appends for chunks < c), at the smallest P
      int p_safe = P;
      if (p.slot_planes == 0) for (int b2 = 0; b2 < p.sl.batch; ++b2) p_safe = min(p_safe, p.sl.d_prefix_len[b2]);
      bool waited = false;
      for (int i = 0; i < ntile; ++i) {
        const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
        if (has_draft && i == 0) {  // staged by the consumer warps; this arrive only keeps the phases aligned
          mbar_arrive(bar_kv_full);
          mbar_arrive(bar_v_full);
          continue;
        }
        const int key0 = tile_of(i) * BN;
        // fused mode: every TMA tile lies below P (a ragged last tile drags in rows >= P that are stale or being
        // appended by this very launch - finite bf16 either way, and masked), nothing to wait for
        if (!fused && !waited && key0 + BN > p_safe) { pdl_wait(); waited = true; }
        mbar_wait(bar_kv_empty + 8 * s, ph ^ 1);
        const uint32_t kd = base + SMEM_K + s * TILE_BYTES, vd = base + SMEM_V + s * TILE_BYTES;
        mbar_expect_tx(bar_kv_full + 8 * s, TILE_BYTES);  // one 64-wide box per sub-tile
#pragma unroll
        for (int b = 0; b < HD / 64; ++b) tma_load_3d(kd + b * SUB, &map_k, bar_kv_full + 8 * s, 64 * b, key0, plane);
        mbar_expect_tx(bar_v_full + 8 * s, TILE_BYTES);
#pragma unroll
        for (int b = 0; b < HD / 64; ++b) tma_load_3d(vd + b * SUB, &map_v, bar_v_full + 8 * s, 64 * b, key0, plane);
        if (i == 0) DBG(2);
      }
    }
    __syncwarp();
    if (ns > 1) { barrier_a(); cluster_sync_all(); }
  } else {
    pdl_wait();  // Q (or, fused, the projection output) below is the predecessor's output
    // ================================================================ staging: thread = (tile row srow, HD / 2-wide half)
    {
      const int srow = tid & 127, half = tid >> 7;
      const int hs = srow / p.np, node = srow % p.np;
      if (srow < rows_used) {
        if (!fused) {
          uint4 qv[CH];  // Q row -> shared memory (K-major SWIZZLE_128B); each half loads HD / 2 elements of d
          const bool have = hs < heads_here && node < n;
          const uint4 *src = reinterpret_cast<const uint4 *>(p.q + ((row0 + node) * p.n_q_heads + hq0 + hs) * HD) + half * CH;
#pragma unroll
          for (int ch = 0; ch < CH; ++ch) qv[ch] = have ? src[ch] : make_uint4(0, 0, 0, 0);
#pragma unroll
          for (int ch = 0; ch < CH; ++ch)
            *reinterpret_cast<uint4 *>(sm + SMEM_Q + half * HALF_SUB + srow * 128 + (((half * HALF_CH + ch) ^ (srow & 7)) << 4)) = qv[ch];
        } else {
          unsigned long long mr0 = 0ull, mr1 = 0ull;
          if (node < n) {
            mr0 = p.mask[(row0 + node) * p.mask_words];
            if (p.mask_words > 1) mr1 = p.mask[(row0 + node) * p.mask_words + 1];
          }
          // RoPE at the node's position = rowsum(mask) - 1 (modeling_llama.py:587): visible prefix + tree depth
          int pos = (P > pad_len ? P - pad_len : 0) + __popcll(mr0) + __popcll(mr1) - 1;
          pos = pos < 0 ? 0 : (pos >= p.max_pos ? p.max_pos - 1 : pos);
          const uint4 *cs = reinterpret_cast<const uint4 *>(p.cos_t + (long long)pos * (HD / 2));
          const uint4 *sn = reinterpret_cast<const uint4 *>(p.sin_t + (long long)pos * (HD / 2));
          const long long row_elems = (long long)(p.n_q_heads + 2 * p.n_kv_heads) * HD;
          const __nv_bfloat16 *xr = p.qkv + (row0 + node) * row_elems;
          const bool have = hs < heads_here && node < n;
          // All global loads of a batch are issued (read-only path: the compiler may not move plain loads across the
          // shared memory stores in between, and eight dependent load rounds would serialise the prologue) before the
          // first value is used; four 16-byte chunks per batch bound the registers.
          {  // Q: rotate this thread's half (the other half of the head is the rotation partner)
            const uint4 *qa = reinterpret_cast<const uint4 *>(xr + (long long)(hq0 + hs) * HD) + half * CH;
            const uint4 *qb = reinterpret_cast<const uint4 *>(xr + (long long)(hq0 + hs) * HD) + (half ^ 1) * CH;
#pragma unroll
            for (int b4 = 0; b4 < CH / 4; ++b4) {
              uint4 ra[4], rb[4], rc[4], rs[4];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int ch = b4 * 4 + j;
                if (have) { ra[j] = __ldg(qa + ch); rb[j] = __ldg(qb + ch); rc[j] = __ldg(cs + ch); rs[j] = __ldg(sn + ch); }
              }
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int ch = b4 * 4 + j;
                const uint4 o = have ? rope8(ra[j], rb[j], rc[j], rs[j], half == 0) : make_uint4(0, 0, 0, 0);
                *reinterpret_cast<uint4 *>(sm + SMEM_Q + half * HALF_SUB + srow * 128 + (((half * HALF_CH + ch) ^ (srow & 7)) << 4)) = o;
              }
            }
          }
          if (has_draft) {
            // the draft tile (ring slot 0): key row r = draft node r, K rotated at r's position, V as projected; rows
            // that hold no node are zero.  The threads of the tile's first head (hs == 0: srow == node) own the key
            // rows; one CTA per KV head also appends the rows to the cache for the steps to come (pretrained_model.py:
            // the reference's torch.cat of past and new K/V, modeling_llama.py:265-268)
            const bool key_row = hs == 0 && node < n;
            const bool writer = hg.j == 0;  // the first head group of the KV head (hq0 % G == 0)
            const uint4 *ka = reinterpret_cast<const uint4 *>(xr + (long long)(p.n_q_heads + hkv) * HD) + half * CH;
            const uint4 *kb = reinterpret_cast<const uint4 *>(xr + (long long)(p.n_q_heads + hkv) * HD) + (half ^ 1) * CH;
            const uint4 *va = reinterpret_cast<const uint4 *>(xr + (long long)(p.n_q_heads + p.n_kv_heads + hkv) * HD) + half * CH;
            const long long crow = (long long)slot * p.sl.kv_slot_stride + ((long long)hkv * p.max_seq + P + node) * HD + half * (HD / 2);
            uint4 *kdst = reinterpret_cast<uint4 *>(p.kc_layer + crow), *vdst = reinterpret_cast<uint4 *>(p.vc_layer + crow);
#pragma unroll
            for (int b4 = 0; b4 < CH / 4; ++b4) {
              uint4 ra[4], rb[4], rc[4], rs[4], rv[4];
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int ch = b4 * 4 + j;
                if (key_row) {
                  ra[j] = __ldg(ka + ch); rb[j] = __ldg(kb + ch); rc[j] = __ldg(cs + ch); rs[j] = __ldg(sn + ch);
                  rv[j] = __ldg(va + ch);
                }
              }
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const int ch = b4 * 4 + j;
                const uint32_t off = half * HALF_SUB + srow * 128 + (((half * HALF_CH + ch) ^ (srow & 7)) << 4);
                uint4 ko = make_uint4(0, 0, 0, 0), vo = make_uint4(0, 0, 0, 0);
                if (key_row) { ko = rope8(ra[j], rb[j], rc[j], rs[j], half == 0); vo = rv[j]; }
                *reinterpret_cast<uint4 *>(sm + SMEM_K + off) = ko;
                *reinterpret_cast<uint4 *>(sm + SMEM_V + off) = vo;
                if (key_row && writer) { kdst[ch] = ko; vdst[ch] = vo; }
              }
            }
          }
        }
      } else if (has_draft) {
        // rows 64..127 of a 64-row tile: the draft tile's key rows there are never live, they are zeroed
#pragma unroll
        for (int ch = 0; ch < CH; ++ch) {
          const uint32_t off = half * HALF_SUB + srow * 128 + (((half * HALF_CH + ch) ^ (srow & 7)) << 4);
          *reinterpret_cast<uint4 *>(sm + SMEM_K + off) = make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4 *>(sm + SMEM_V + off) = make_uint4(0, 0, 0, 0);
        }
      }
      if constexpr (kAlibi) {
        // in the spare bytes after the barriers: the depth popc(mask[k]) of every draft node (the bias of the draft
        // keys, and of the query rows) and each warpgroup's slope in the log2 domain.  The tile loop reads them back
        // from shared memory: held in registers through the loop they would spill.
        if (tid < p.np) {
          int d = 0;
          if (tid < n) {
            d = __popcll(p.mask[(row0 + tid) * p.mask_words]);
            if (p.mask_words > 1) d += __popcll(p.mask[(row0 + tid) * p.mask_words + 1]);
          }
          sm[SMEM_BAR + ALIBI_DEPTH + tid] = (uint8_t)d;
        }
        if (tid < 2) {
          const int hs_wg = tid * 64 / p.np;  // the query head of warpgroup tid (64 rows each)
          reinterpret_cast<float *>(sm + SMEM_BAR + ALIBI_SLOPE)[tid] =
              hs_wg < heads_here ? p.slopes[hq0 + hs_wg] * LOG2E : 0.f;
        }
      }
      fence_async_smem();  // generic-proxy stores -> visible to the wgmma (async proxy) reads
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (tid == 0) DBG(5);

    const int wg = warp >> 2;
    if (wg < n_wg) {
      // ================================================================ QK^T, softmax, PV of this warpgroup's 64 rows
      // accumulator fragments: register 4 * nb + 2 * h + e holds row rw[h] = 64 wg + 16 (warp % 4) + lane / 4 + 8 h,
      // column 8 nb + 2 (lane % 4) + e (a key of S, a head-dim element of O)
      int rw[2], hs[2], node[2];
      bool live[2];
      unsigned long long mrow[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        rw[h] = wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * h;
        hs[h] = rw[h] / p.np; node[h] = rw[h] % p.np;
        live[h] = node[h] < n;
        mrow[h][0] = mrow[h][1] = 0ull;
        if (!kAlibi && live[h]) {  // the ALiBi instance reads the rows again per masked tile (registers)
          mrow[h][0] = p.mask[(row0 + node[h]) * p.mask_words];
          if (p.mask_words > 1) mrow[h][1] = p.mask[(row0 + node[h]) * p.mask_words + 1];
        }
      }
      const uint32_t qa = base + SMEM_Q + wg * 64 * 128;
      float o[HD / 2];
#pragma unroll
      for (int j = 0; j < HD / 2; ++j) o[j] = 0.f;
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // l_run: this thread's 32 columns of the row
      for (int i = 0; i < ntile; ++i) {
        const int tl = tile_of(i);
        const bool is_draft = fused && tl == Tp;
        const int s = i % NSTAGE, ph = (i / NSTAGE) & 1;
        const uint32_t ka = base + SMEM_K + s * TILE_BYTES, va = base + SMEM_V + s * TILE_BYTES;
        mbar_wait(bar_kv_full + 8 * s, ph);
        float sv[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) sv[j] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < HD / 16; ++j) {  // K-major operands: 32 B per k-block inside the 128 B swizzle row
          const uint32_t off = (j >> 2) * SUB + (j & 3) * 32;
          wgmma_qk(sv, make_desc(qa + off, 16, 1024), make_desc(ka + off, 16, 1024));
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_regs(sv);
        if (tid == 0 && i == 0) DBG(6);
        // 32-bit visibility word of keys [kb, kb+32): prefix keys [pad_len, P) are visible to every row, the n draft
        // keys follow the row's ancestor bits (bits beyond the live nodes are never set in the trie's mask rows)
        const bool all_visible = !is_draft && (tl * BN >= pad_len) && (tl * BN + BN <= P);
        if (!all_visible) {  // tree / padded / ragged tile: hidden keys -> -inf once, then the dense code
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            unsigned long long m0 = mrow[h][0], m1 = mrow[h][1];
            if (kAlibi && live[h]) {
              m0 = p.mask[(row0 + node[h]) * p.mask_words];
              if (p.mask_words > 1) m1 = p.mask[(row0 + node[h]) * p.mask_words + 1];
            }
            auto vis32 = [&](int kb) -> uint32_t {
              if (is_draft) {  // key kb - Tp * BN is draft node j0: visible iff it is an ancestor (or the node itself)
                const int j0 = kb - Tp * BN;
                if (j0 < 64) {
                  unsigned long long x = m0 >> j0;
                  if (j0 > 32) x |= m1 << (64 - j0);
                  return (uint32_t)x;
                }
                return (uint32_t)(m1 >> (j0 - 64));
              }
              uint32_t m = 0;
              const int lo = kb < pad_len ? pad_len : kb;
              const int hi = kb + 32 < P ? kb + 32 : P;
              if (hi > lo) m = (hi - lo >= 32 ? 0xffffffffu : ((1u << (hi - lo)) - 1u)) << (lo - kb);
              const int j0 = kb - P;
              if (!fused && j0 + 32 > 0 && j0 < n) {
                uint32_t d;
                if (j0 < 0) d = (uint32_t)(m0 << (-j0));
                else if (j0 < 64) {
                  unsigned long long x = m0 >> j0;
                  if (j0 > 32) x |= m1 << (64 - j0);
                  d = (uint32_t)x;
                } else d = (uint32_t)(m1 >> (j0 - 64));
                m |= d;
              }
              return m;
            };
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const uint32_t vm = vis32(tl * BN + 32 * c) >> (2 * (lane & 3));
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const int nb = 4 * c + k;
                if (!((vm >> (8 * k)) & 1u)) sv[4 * nb + 2 * h] = -INFINITY;
                if (!((vm >> (8 * k + 1)) & 1u)) sv[4 * nb + 2 * h + 1] = -INFINITY;
              }
            }
          }
        }
        if constexpr (kAlibi) {
          // scores -> log2 domain with the bias: s * scale_log2 + sl2 * (kpos - qpos); hidden keys stay -inf.
          // sl2 = the warpgroup's slope * log2(e); a row at depth dq sees cached key j at kpos - qpos = j - cq and
          // draft key k at depth(k) - dq
          const uint8_t *depth = sm + SMEM_BAR + ALIBI_DEPTH;
          const float sl2 = reinterpret_cast<const float *>(sm + SMEM_BAR + ALIBI_SLOPE)[wg];
          int dq[2], cq[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            dq[h] = depth[(wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * h) & (p.np - 1)];  // the row's node
            cq[h] = pad_len + (P > pad_len ? P - pad_len : 0) - 1 + dq[h];
          }
          if (all_visible) {  // cached keys only: the bias is linear in the column, one FMA per score on top
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float rb = sl2 * (float)(tl * BN + 2 * (lane & 3) - cq[h]);
#pragma unroll
              for (int nb = 0; nb < 16; ++nb) {
                sv[4 * nb + 2 * h] = fmaf(sv[4 * nb + 2 * h], p.scale_log2, fmaf(sl2, (float)(8 * nb), rb));
                sv[4 * nb + 2 * h + 1] = fmaf(sv[4 * nb + 2 * h + 1], p.scale_log2, fmaf(sl2, (float)(8 * nb + 1), rb));
              }
            }
          } else {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
              for (int c = 0; c < 32; ++c) {
                const int j = tl * BN + 8 * (c >> 1) + 2 * (lane & 3) + (c & 1);
                const int d = j < P ? j - cq[h] : (int)depth[(j - P) & 127] - dq[h];  // beyond the draft: hidden
                const int r = 4 * (c >> 1) + 2 * h + (c & 1);
                sv[r] = fmaf(sv[r], p.scale_log2, sl2 * (float)d);
              }
            }
          }
        }
        // row max: this thread's 32 columns, then the four lanes that share the row
        float m_new[2], m_use[2], alpha[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
          for (int nb = 0; nb < 16; ++nb) {
            mx0 = fmaxf(mx0, sv[4 * nb + 2 * h]);
            mx1 = fmaxf(mx1, sv[4 * nb + 2 * h + 1]);
          }
          float mx = fmaxf(mx0, mx1);
          mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(FULL, mx, 2));
          m_new[h] = fmaxf(m_run[h], kAlibi ? mx : mx * p.scale_log2);  // ALiBi: already in the log2 domain
          m_use[h] = (m_new[h] == -INFINITY) ? 0.f : m_new[h];
          alpha[h] = (m_run[h] == -INFINITY) ? 0.f : ex2(m_run[h] - m_use[h]);
        }
        // p = exp2(s*scale - m) -> bf16 pairs: register pair (2 m, 2 m + 1) of S is A-fragment register m of PV
        // (k-block m / 4), so P never leaves the registers; the row sum uses the bf16-rounded probabilities, i.e.
        // exactly what the PV MMA consumes
        uint32_t pa[32];
        float ls[2] = {0.f, 0.f};
#pragma unroll
        for (int m = 0; m < 32; ++m) {  // ex2(-inf) = 0 for the hidden keys (m_use is finite)
          const int h = m & 1;
          const float p0 = ex2(kAlibi ? sv[2 * m] - m_use[h] : sv[2 * m] * p.scale_log2 - m_use[h]);
          const float p1 = ex2(kAlibi ? sv[2 * m + 1] - m_use[h] : sv[2 * m + 1] * p.scale_log2 - m_use[h]);
          const __nv_bfloat162 b = __floats2bfloat162_rn(p0, p1);
          ls[h] += __bfloat162float(b.x) + __bfloat162float(b.y);
          pa[m] = *reinterpret_cast<const uint32_t *>(&b);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          l_run[h] = l_run[h] * alpha[h] + ls[h];
          m_run[h] = m_new[h];
        }
#pragma unroll
        for (int nb = 0; nb < HD / 8; ++nb) {
          o[4 * nb] *= alpha[0]; o[4 * nb + 1] *= alpha[0];
          o[4 * nb + 2] *= alpha[1]; o[4 * nb + 3] *= alpha[1];
        }
        if (tid == 0 && i == 0) DBG(7);
        mbar_wait(bar_v_full + 8 * s, ph);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < BN / 16; ++j) {
          // B = V, MN-major: 16 keys = 2 groups of 8 rows (SBO 1024 B), 64-wide d sub-tiles 16 KB apart (LBO);
          // wgmma N = HD (the overload taking this o[])
          wgmma_pv(o, pa + 4 * j, make_desc(va + j * 2048, SUB, 1024));
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_regs(o);
        fence_regs(pa);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_kv_empty + 8 * s);  // this warp is done with the stage's K and V
      }
      if (tid == 0) DBG(8);
      // derived again from blockIdx.y rather than held through the tile loop (holding it there adds register spills)
      const HeadGroup hl = head_group(p, group);
      // total row sum = the four lanes of the row (same running max, so the partial sums just add)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        l_run[h] += __shfl_xor_sync(FULL, l_run[h], 1);
        l_run[h] += __shfl_xor_sync(FULL, l_run[h], 2);
      }
      if (tid == 0) DBG(9);
      if (ns == 1) {
        // single split: normalise and write the final bf16 rows
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (live[h]) {
            const float inv = l_run[h] > 0.f ? 1.f / l_run[h] : 0.f;
            uint32_t *dst = reinterpret_cast<uint32_t *>(p.out + ((row0 + node[h]) * p.n_q_heads + hl.hq0 + hs[h]) * HD);
#pragma unroll
            for (int nb = 0; nb < HD / 8; ++nb) {
              __nv_bfloat162 b = __floats2bfloat162_rn(o[4 * nb + 2 * h] * inv, o[4 * nb + 2 * h + 1] * inv);
              dst[4 * nb + (lane & 3)] = *reinterpret_cast<uint32_t *>(&b);
            }
          }
        }
      } else {
        // several splits: the ns CTAs of this head group form one thread-block cluster.  After everyone has left its
        // tile loop (barrier A: the Q/KV tiles of every CTA are dead) each thread pushes its rows' pieces - acc, and
        // the row's (m, l) - straight into the shared memory of the CTA that owns that row's slice (DSMEM), barrier B,
        // and every CTA combines its slice locally: no workspace round trip through L2, no serial last-arriver merge.
        barrier_a();
        if (tid == 0) DBG(14);
        const int RS = (hl.heads * p.np + ns - 1) / ns;  // rows per owner CTA
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (live[h]) {
            const int owner = rw[h] / RS, rl = rw[h] % RS;
            // partial rows are stored chunk-major ([HD / 4 float4 chunks][slot]): head-dim element d = 8 nb + 2 (lane % 4)
            // lies in chunk d / 4 = 2 nb + (lane % 4) / 2, at float offset 2 (lane % 2)
            const uint32_t dst = map_to_cta(base + mrg_acc + (uint32_t)((((lane & 3) >> 1) * mrg_stride + split * RS + rl) * 16 + (lane & 1) * 8), owner);
#pragma unroll
            for (int nb = 0; nb < HD / 8; ++nb)
              st_cluster_f2(dst + (uint32_t)(2 * nb * mrg_stride) * 16, o[4 * nb + 2 * h], o[4 * nb + 2 * h + 1]);
            if ((lane & 3) == 0) st_cluster_f2(map_to_cta(base + mrg_ml + (uint32_t)(split * RS + rl) * 8, owner), m_run[h], l_run[h]);
          }
        }
        __syncwarp();  // the live-row branch above diverges; the cluster barrier is warp-aligned
        if (tid == 0) DBG(15);
        cluster_sync_all();
      }
      if (tid == 0) DBG(10);
    } else {
      if (ns > 1) { barrier_a(); cluster_sync_all(); }  // idle warpgroup (rows 64..127 of a one-head tile)
    }
  }
  if (ns > 1) {
    // combine this CTA's row slice: out[r][:] = sum_i acc_i 2^(m_i - M) / sum_i l_i 2^(m_i - M), all operands local
    const HeadGroup hl = head_group(p, group);  // derived again (see above)
    const int rows_late = hl.heads * p.np;
    const int RS = (rows_late + ns - 1) / ns;
    const float4 *macc = reinterpret_cast<const float4 *>(sm + mrg_acc);
    const float2 *mml = reinterpret_cast<const float2 *>(sm + mrg_ml);
    const int items = RS * (HD / 4);
    // RS and np are powers of two in every configuration but ragged ones: shifts instead of four integer divisions per
    // item, and all ns partials of an item are loaded before the first is used (a loop over a runtime ns would be a
    // chain of dependent shared-memory round trips)
    const bool pow2 = (RS & (RS - 1)) == 0 && (p.np & (p.np - 1)) == 0;
    const int rs_sh = 31 - __clz(RS), np_sh = 31 - __clz(p.np);
    for (int it = tid; it < items; it += NTHREADS) {
      const int rl = pow2 ? (it & (RS - 1)) : it % RS, c4 = pow2 ? (it >> rs_sh) : it / RS;
      const int r = split * RS + rl;
      if (r >= rows_late) continue;
      const int rh = pow2 ? (r >> np_sh) : r / p.np, rn = pow2 ? (r & (p.np - 1)) : r % p.np;
      if (rn >= n) continue;
      float2 ml[MAX_SPLIT];
      float4 a4[MAX_SPLIT];
#pragma unroll
      for (int i = 0; i < MAX_SPLIT; ++i) {
        if (i < ns) { ml[i] = mml[i * RS + rl]; a4[i] = macc[c4 * mrg_stride + i * RS + rl]; }
        else { ml[i] = make_float2(-INFINITY, 0.f); a4[i] = make_float4(0.f, 0.f, 0.f, 0.f); }
      }
      float M = -INFINITY;
#pragma unroll
      for (int i = 0; i < MAX_SPLIT; ++i) M = fmaxf(M, ml[i].x);
      float den = 0.f;
      float4 o4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int i = 0; i < MAX_SPLIT; ++i) {
        const float w = ml[i].x == -INFINITY ? 0.f : ex2(ml[i].x - M);
        den += ml[i].y * w;
        o4.x += a4[i].x * w; o4.y += a4[i].y * w; o4.z += a4[i].z * w; o4.w += a4[i].w * w;
      }
      const float inv = den > 0.f ? 1.f / den : 0.f;
      __nv_bfloat162 b0 = __floats2bfloat162_rn(o4.x * inv, o4.y * inv), b1 = __floats2bfloat162_rn(o4.z * inv, o4.w * inv);
      reinterpret_cast<uint2 *>(p.out + ((row0 + rn) * p.n_q_heads + hl.hq0 + rh) * HD)[c4] =
          make_uint2(*reinterpret_cast<uint32_t *>(&b0), *reinterpret_cast<uint32_t *>(&b1));
    }
  }
  if (tid == 0) DBG(12);
}

}  // namespace attn
}  // namespace pia

// =====================================================================================================
using namespace pia;
using namespace pia::attn;

struct pia_attn_plan {
  pia_attn_config_t cfg;
  CUtensorMap map_k, map_v;
  int heads_per_cta, ctas_per_kv, n_groups, n_split, mask_words, tiles_per_cta;
  unsigned long long *dbg;
  __nv_bfloat16 *k_base, *v_base;  // the caches the TMA maps describe (fused mode appends the draft rows itself)
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int encode_kv_map(CUtensorMap *m, void *base, const pia_attn_config_t &c) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    cudaDriverEntryPointQueryResult qres;
    void *ptr = nullptr;
    PIA_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres));
    PIA_REQUIRE(ptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available in this driver");
    fn = (EncodeTiledFn)ptr;
  }
  // cache viewed as [planes = n_layers * n_kv_heads][max_seq][head_dim] bf16, box = 64 d x 128 keys x 1 plane
  cuuint64_t dims[3] = {(cuuint64_t)c.head_dim, (cuuint64_t)c.max_seq,
                        (cuuint64_t)(c.n_slots > 0 ? c.n_slots : 1) * c.n_layers * c.n_kv_heads};
  cuuint64_t strides[2] = {(cuuint64_t)c.head_dim * 2, (cuuint64_t)c.max_seq * c.head_dim * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)BN, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return PIA_ERR_CUDA; }
  return PIA_OK;
}

extern "C" int pia_attn_plan_create(const pia_attn_config_t *cfg, void *d_k_cache, void *d_v_cache,
                                    pia_attn_plan_t **out) {
  PIA_REQUIRE(cfg && d_k_cache && d_v_cache && out, "null argument");
  if (cfg->head_dim != 64 && cfg->head_dim != 128) {
    set_error("head_dim %d: k_tree_attn is built for 64 and 128", cfg->head_dim);
    return PIA_ERR_UNSUPPORTED;
  }
  PIA_REQUIRE(cfg->max_nodes == 64 || cfg->max_nodes == 128, "max_nodes must be 64 or 128");
  PIA_REQUIRE(cfg->n_q_heads > 0 && cfg->n_kv_heads > 0 && cfg->n_q_heads % cfg->n_kv_heads == 0, "bad head counts");
  PIA_REQUIRE(cfg->max_seq > 0 && cfg->n_layers > 0, "bad cache shape");
  PIA_REQUIRE((reinterpret_cast<uintptr_t>(d_k_cache) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_v_cache) & 15) == 0, "cache must be 16-byte aligned");
  pia_attn_plan *p = new (std::nothrow) pia_attn_plan();
  PIA_REQUIRE(p, "out of host memory");
  p->cfg = *cfg;
  const int G = cfg->n_q_heads / cfg->n_kv_heads;
  // two query heads of one KV head per 128-row tile at 64 draft rows (any G: an odd G leaves one head in its KV head's
  // last tile), one head at 128 draft rows
  p->heads_per_cta = cfg->max_nodes == 64 ? 2 : 1;
  p->ctas_per_kv = (G + p->heads_per_cta - 1) / p->heads_per_cta;
  p->n_groups = cfg->n_kv_heads * p->ctas_per_kv;
  p->mask_words = cfg->max_nodes / 64;
  int n_sm = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  const int max_tiles = (cfg->max_seq + BN - 1) / BN;
  // one wave: the split CTAs of a head group are one thread-block cluster, so idle splits still occupy an SM each
  int ns = cfg->kv_split_max > 0 ? cfg->kv_split_max : n_sm / p->n_groups;
  if (ns > max_tiles) ns = max_tiles;
  if (ns < 1) ns = 1;
  if (ns > MAX_SPLIT) ns = MAX_SPLIT;
  p->n_split = ns;
  p->tiles_per_cta = 1;
  if (const char *e = getenv("PIA_ATTN_TILES_PER_CTA")) { int v = atoi(e); if (v >= 1 && v <= 64) p->tiles_per_cta = v; }
  int rc = encode_kv_map(&p->map_k, d_k_cache, *cfg);
  if (rc == PIA_OK) rc = encode_kv_map(&p->map_v, d_v_cache, *cfg);
  if (rc == PIA_OK) {
    cudaError_t e = cfg->head_dim == 64
                        ? cudaFuncSetAttribute(k_tree_attn<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Smem<64>::TOTAL)
                        : cudaFuncSetAttribute(k_tree_attn<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Smem<128>::TOTAL);
    if (e == cudaSuccess && cfg->head_dim == 128)
      e = cudaFuncSetAttribute(k_tree_attn<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Smem<128>::TOTAL);
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(e)); rc = PIA_ERR_CUDA; }
  }
  p->dbg = nullptr;
  p->k_base = (__nv_bfloat16 *)d_k_cache; p->v_base = (__nv_bfloat16 *)d_v_cache;
  if (rc != PIA_OK) { delete p; return rc; }
  *out = p;
  return PIA_OK;
}

extern "C" int pia_attn_plan_set_debug(pia_attn_plan_t *p, void *d_timestamps) {
  PIA_REQUIRE(p, "null plan");
  p->dbg = (unsigned long long *)d_timestamps;
  return PIA_OK;
}
extern "C" int pia_attn_plan_grid(const pia_attn_plan_t *p, int *n_split, int *n_groups) {
  PIA_REQUIRE(p && n_split && n_groups, "null argument");
  *n_split = p->n_split; *n_groups = p->n_groups;
  return PIA_OK;
}

extern "C" int pia_attn_plan_destroy(pia_attn_plan_t *p) {
  if (p) delete p;
  return PIA_OK;
}

static int attn_launch(pia_attn_plan_t *p, int layer, const void *d_q, const void *d_qkv, const void *d_cos,
                       const void *d_sin, int max_pos, const uint64_t *d_mask, const pia_slots_t *slots, float scale_mul,
                       void *d_out, void *stream, const float *d_slopes = nullptr) {
  const bool fused = d_qkv != nullptr;
  PIA_REQUIRE(p && (d_q || d_qkv) && d_mask && slots && slots->d_n && slots->d_prefix_len && d_out, "null argument");
  if (d_slopes && p->cfg.head_dim != 128) {
    set_error("head_dim %d: the ALiBi tree attention is built for head_dim 128 only", p->cfg.head_dim);
    return PIA_ERR_UNSUPPORTED;
  }
  PIA_REQUIRE(layer >= 0 && layer < p->cfg.n_layers, "layer %d outside [0,%d)", layer, p->cfg.n_layers);
  PIA_REQUIRE(slots->batch >= 1 && slots->batch <= 65535 && slots->rows_per_slot >= 1 &&
                  slots->rows_per_slot <= p->cfg.max_nodes, "bad slot table");
  const long long cache_elems = (long long)p->cfg.n_layers * p->cfg.n_kv_heads * p->cfg.max_seq * p->cfg.head_dim;
  const int plan_slots = p->cfg.n_slots > 0 ? p->cfg.n_slots : 1;
  PIA_REQUIRE(slots->kv_first_slot >= 0 && slots->kv_first_slot < plan_slots, "kv_first_slot outside the plan's caches");
  PIA_REQUIRE(slots->kv_slot_stride == 0 || (slots->kv_slot_stride == cache_elems &&
                                              slots->kv_first_slot + slots->batch <= plan_slots),
              "kv_slot_stride must be 0 or one whole cache, and the plan must span `batch` caches");
  // fused mode appends the draft rows of every slot from inside the launch: slots that share one cache (the chain
  // chunks of a prefill pass) would read rows their neighbours are still writing - they take the two-kernel path
  PIA_REQUIRE(!fused || slots->batch == 1 || slots->kv_slot_stride != 0,
              "the fused RoPE / KV-append attention needs one cache per slot");
  PIA_REQUIRE(!fused || (d_cos && d_sin && max_pos > 0), "fused mode needs the RoPE tables");
  Params a;
  a.q = (const __nv_bfloat16 *)d_q;
  a.mask = (const unsigned long long *)d_mask;
  a.sl = *slots;
  a.slot_planes = slots->kv_slot_stride ? p->cfg.n_layers * p->cfg.n_kv_heads : 0;
  a.plane0 = slots->kv_first_slot * p->cfg.n_layers * p->cfg.n_kv_heads;
  a.layer = layer; a.n_q_heads = p->cfg.n_q_heads; a.n_kv_heads = p->cfg.n_kv_heads; a.np = p->cfg.max_nodes;
  a.mask_words = p->mask_words; a.max_seq = p->cfg.max_seq;
  a.heads_per_cta = p->heads_per_cta; a.ctas_per_kv = p->ctas_per_kv;
  // KV splits per (slot, head group): one wave of CTAs over ALL slots - a batch of requests brings its own parallelism,
  // so each cluster shrinks (8 slots x 32 head groups already cover the SMs without any split)
  int ns = p->n_split / slots->batch;
  if (ns < 1) ns = 1;
  a.n_split = ns; a.tiles_per_cta = p->tiles_per_cta;
  a.out = (__nv_bfloat16 *)d_out; a.dbg = p->dbg;
  a.fused = fused ? 1 : 0;
  a.qkv = (const __nv_bfloat16 *)d_qkv; a.cos_t = (const __nv_bfloat16 *)d_cos; a.sin_t = (const __nv_bfloat16 *)d_sin;
  a.max_pos = max_pos;
  const long long layer_off = ((long long)slots->kv_first_slot * p->cfg.n_layers + layer) * p->cfg.n_kv_heads *
                              (long long)p->cfg.max_seq * p->cfg.head_dim;
  a.kc_layer = p->k_base + layer_off; a.vc_layer = p->v_base + layer_off;
  a.scale_log2 = scale_mul * 1.4426950408889634f / sqrtf((float)p->cfg.head_dim);
  a.slopes = d_slopes;
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid(ns, p->n_groups, slots->batch);
  if (d_slopes)
    PIA_CUDA_CHECK(launch_kernel_cluster(k_tree_attn<128, true>, grid, dim3(NTHREADS), Smem<128>::TOTAL, s,
                                         (unsigned)ns, p->map_k, p->map_v, a));
  else if (p->cfg.head_dim == 64)
    PIA_CUDA_CHECK(launch_kernel_cluster(k_tree_attn<64, false>, grid, dim3(NTHREADS), Smem<64>::TOTAL, s, (unsigned)ns,
                                         p->map_k, p->map_v, a));
  else
    PIA_CUDA_CHECK(launch_kernel_cluster(k_tree_attn<128, false>, grid, dim3(NTHREADS), Smem<128>::TOTAL, s, (unsigned)ns,
                                         p->map_k, p->map_v, a));
  count_launch();
  return PIA_OK;
}

extern "C" int pia_tree_attn_fwd(pia_attn_plan_t *p, int layer, const void *d_q, const uint64_t *d_mask,
                                 const pia_slots_t *slots, float scale_mul, void *d_out, void *stream) {
  PIA_REQUIRE(d_q, "null q");
  return attn_launch(p, layer, d_q, nullptr, nullptr, nullptr, 0, d_mask, slots, scale_mul, d_out, stream);
}

extern "C" int pia_tree_attn_fused_fwd(pia_attn_plan_t *p, int layer, const void *d_qkv, const void *d_cos,
                                       const void *d_sin, int max_pos, const uint64_t *d_mask, const pia_slots_t *slots,
                                       float scale_mul, void *d_out, void *stream) {
  PIA_REQUIRE(d_qkv, "null qkv");
  return attn_launch(p, layer, nullptr, d_qkv, d_cos, d_sin, max_pos, d_mask, slots, scale_mul, d_out, stream);
}

extern "C" int pia_tree_attn_alibi_fwd(pia_attn_plan_t *p, int layer, const void *d_q, const uint64_t *d_mask,
                                       const pia_slots_t *slots, float scale_mul, const float *d_slopes, void *d_out,
                                       void *stream) {
  PIA_REQUIRE(d_q && d_slopes, "null q / slopes");
  return attn_launch(p, layer, d_q, nullptr, nullptr, nullptr, 0, d_mask, slots, scale_mul, d_out, stream, d_slopes);
}
