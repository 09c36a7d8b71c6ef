// Longest-prefix accept, sequence update and KV compaction of the LOOKAHEAD loop (sm_90a).
//
// Takes over common/pretrained_model.py:764-892 (_lookahead_update_model_kwargs_for_generation) and :894-945
// (_update_cache*).  The reference walks the draft on the host with one GPU arg-max plus one .tolist() sync per
// accepted token; here
//   k_row_argmax : every draft node's (penalised) arg-max in parallel - the penalised set of node k is
//                  context U {tokens on the path root..k}, a pure function of the node (SURVEY A.2-12), so the
//                  sequential logits_processor calls of :834 collapse into one pass over the [n, V] logits;
//   k_accept_walk: one warp follows the unique surviving branch (:827-860), appends the accepted tokens to the
//                  device-resident sequence and advances seq_len / prefix_len, raises `finished` (:1225-1231);
//   k_kv_compact : moves the accepted nodes' K/V rows next to the prefix in place (:863-875, 894-907).
// The host sees one small D2H copy per step (count + tokens).
#include <cuda_bf16.h>

#include "common.cuh"

namespace pia {
namespace accept {

__device__ __forceinline__ float bf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// Gumbel noise for multinomial accept (pretrained_model.py:835-837: probs = softmax(scores); multinomial(probs, 1)):
// arg-max_v (score_v + G_v) with independent standard Gumbel G_v is a draw from softmax(scores).  G_v is a pure function
// of (seed, step counter, activation row, token), so every draft node of a step draws independently and a replayed
// CUDA graph draws fresh numbers every step (the walk advances the counter).
__device__ __forceinline__ float gumbel(unsigned seed, unsigned counter, unsigned row, unsigned tok) {
  unsigned x = seed ^ (counter * 0x9E3779B1u) ^ (row * 0x85EBCA6Bu) ^ (tok * 0xC2B2AE35u);
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  const float u = ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0, 1)
  return -__logf(-__logf(u));
}

constexpr int NT = 1024;

// (v, i) comes first in torch.argmax order: a NaN above every number, then the larger value, then the lower index
__device__ __forceinline__ bool beats(float v, int i, float best, int best_i) {
  const bool vn = v != v, bn = best != best;
  if (vn != bn) return vn;
  return v > best || ((vn || v == best) && i < best_i);
}

// grid = batch * rows_per_slot activation rows (rows >= n of their slot idle).  dynamic smem: vocab bits (only when
// penalty != 1)
__global__ void __launch_bounds__(NT) k_row_argmax(const __nv_bfloat16 *logits, int vocab, const int *ids,
                                                   const unsigned long long *mask, int mask_words, const int *d_n,
                                                   int rows_per_slot, const int *seq, int seq_stride,
                                                   const int *d_seq_len, float penalty, float inv_penalty,
                                                   const unsigned *rng, int *row_tok) {
  extern __shared__ unsigned bits[];
  __shared__ float s_val[NT / 32];
  __shared__ int s_idx[NT / 32];
  const int row = blockIdx.x, tid = threadIdx.x;
  const int slot = row / rows_per_slot, node = row % rows_per_slot;
  const int n = d_n[slot];
  if (node >= n) return;
  const long long r0 = (long long)slot * rows_per_slot;  // first draft row of the slot
  const bool pen = penalty != 1.0f;
  if (pen) {
    const int words = (vocab + 31) >> 5;
    for (int w = tid; w < words; w += NT) bits[w] = 0u;
    __syncthreads();
    const int len = d_seq_len[slot];
    const int *sq = seq + (long long)slot * seq_stride;
    // RepetitionPenaltyLogitsProcessor sees input_ids (left pads included) + the tokens accepted so far this step
    for (int i = tid; i < len; i += NT) { const int t = sq[i]; if (t >= 0 && t < vocab) atomicOr(&bits[t >> 5], 1u << (t & 31)); }
    if (tid < n && tid >= 1) {
      if ((mask[(r0 + node) * mask_words + (tid >> 6)] >> (tid & 63)) & 1ull) {
        const int t = ids[r0 + tid];
        if (t >= 0 && t < vocab) atomicOr(&bits[t >> 5], 1u << (t & 31));
      }
    }
    __syncthreads();
  }
  const __nv_bfloat16 *lr = logits + (long long)row * vocab;
  const bool sample = rng != nullptr;
  const unsigned seed = sample ? rng[0] : 0u, counter = sample ? rng[1] : 0u;
  float best = -INFINITY;
  int best_i = 0x7fffffff;
  for (int v0 = tid * 8; v0 < vocab; v0 += NT * 8) {
    __nv_bfloat16 h[8];
    if (v0 + 8 <= vocab && ((((long long)row * vocab + v0) & 7) == 0)) {
      *reinterpret_cast<uint4 *>(h) = *reinterpret_cast<const uint4 *>(lr + v0);
    } else {
      for (int j = 0; j < 8; ++j) h[j] = v0 + j < vocab ? lr[v0 + j] : __float2bfloat16_rn(-INFINITY);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int t = v0 + j;
      if (t >= vocab) break;
      float x = __bfloat162float(h[j]);
      // RepetitionPenaltyLogitsProcessor: score * p below zero, else score / p - which PyTorch's CUDA true division
      // by a Python scalar computes as score * fl32(1 / p), the reciprocal taken in double (div_true_kernel_cuda)
      if (pen && ((bits[t >> 5] >> (t & 31)) & 1u)) x = x < 0.f ? bf(x * penalty) : bf(x * inv_penalty);
      if (sample) x += gumbel(seed, counter, (unsigned)row, (unsigned)t);
      // torch.argmax order: !(x <= best) also takes a NaN, and once best is a NaN nothing replaces it; ascending t
      // inside a thread keeps the first maximum
      if (!(x <= best) && best == best) { best = x; best_i = t; }
    }
  }
  // first-index arg-max (torch.argmax returns the first maximal index)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(FULL, best, o);
    const int oi = __shfl_xor_sync(FULL, best_i, o);
    if (beats(ov, oi, best, best_i)) { best = ov; best_i = oi; }
  }
  if ((tid & 31) == 0) { s_val[tid >> 5] = best; s_idx[tid >> 5] = best_i; }
  __syncthreads();
  if (tid < 32) {
    best = s_val[tid]; best_i = s_idx[tid];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(FULL, best, o);
      const int oi = __shfl_xor_sync(FULL, best_i, o);
      if (beats(ov, oi, best, best_i)) { best = ov; best_i = oi; }
    }
    if (tid == 0) row_tok[row] = best_i == 0x7fffffff ? 0 : best_i;
  }
}

// one CTA of 128 threads per slot (thread j <-> draft node j of the slot)
__global__ void __launch_bounds__(128) k_accept_walk(pia_accept_config_t cfg, const int *row_tok, const int *ids,
                                                     const unsigned long long *mask, int mask_words, const int *d_n,
                                                     int rows_per_slot, int *seq, int seq_stride, int *d_seq_len,
                                                     const int *d_max_length, unsigned *rng, int *acc_tokens,
                                                     int *acc_count, int *acc_nodes, int *d_prefix, int *d_finished) {
  __shared__ int s_parent[128], s_ids[128], s_next;
  const int j = threadIdx.x, slot = blockIdx.x;
  const int n = d_n[slot];
  if (rng != nullptr && slot == 0 && j == 0) rng[1] = rng[1] + 1u;  // k_row_argmax of this step has drawn its noise
  // idle slot, or a request that already finished (a step launched ahead of the host's stop check is a no-op)
  if (n <= 0 || d_finished[slot] != 0) { if (j == 0) acc_count[slot] = 0; return; }
  const long long r0 = (long long)slot * rows_per_slot;
  row_tok += r0; ids += r0; mask += r0 * mask_words;
  seq += (long long)slot * seq_stride;
  acc_tokens += (long long)slot * cfg.max_nodes; acc_nodes += (long long)slot * cfg.max_nodes;
  const int max_length = d_max_length ? *d_max_length : cfg.max_length;
  // parent(j) = nearest ancestor = highest set bit below j in row j (DFS pre-order)
  int parent = -1;
  if (j < n && j >= 1) {
    for (int w = mask_words - 1; w >= 0 && parent < 0; --w) {
      unsigned long long m = mask[(long long)j * mask_words + w];
      if (w == (j >> 6)) m &= (1ull << (j & 63)) - 1ull;
      else if (w > (j >> 6)) m = 0ull;
      if (m) parent = w * 64 + 63 - __clzll((long long)m);
    }
  }
  s_parent[j] = parent;
  s_ids[j] = j < n ? ids[j] : -1;
  __syncthreads();
  int cur = 0, count = 0;
  const int len0 = d_seq_len[slot];
  // batched loop: the walk never writes past max_length (pretrained_model_batch.py:862); the per-request loop clamps
  // the draft depth when it queries the trie instead (pretrained_model.py:680)
  const int cap = cfg.bound_walk ? max_length - len0 : 0x7fffffff;
  bool fin = false;
  while (true) {
    const int t = row_tok[cur];
    if (j == 0) {
      acc_tokens[count] = t; acc_nodes[count] = cur;
      if (len0 + count < seq_stride) seq[len0 + count] = t;
      s_next = -1;
    }
    for (int e = 0; e < cfg.n_eos; ++e) fin |= (t == cfg.eos[e]);
    ++count;
    __syncthreads();
    if (j >= 1 && j < n && s_parent[j] == cur && s_ids[j] == t) s_next = j;  // children carry distinct tokens
    __syncthreads();
    const int nx = s_next;
    __syncthreads();
    if (nx < 0 || count >= n || count >= cap) break;
    cur = nx;
  }
  if (j == 0) {
    const int len1 = len0 + count;
    acc_count[slot] = count;
    d_seq_len[slot] = len1;
    d_prefix[slot] = d_prefix[slot] + count;
    if (len1 >= max_length) fin = true;  // MaxLengthCriteria (:1225) / cursor + 1 >= max_length (batch :1274)
    if (fin) d_finished[slot] = 1;
  }
}

// grid = (n_layers * n_kv_heads, 2, batch); thread = one 16-byte chunk of a row; ascending k is hazard free
// because the k-th accepted node has draft index >= k (pre-order), so a destination never lies above its source
__global__ void __launch_bounds__(64) k_kv_compact(__nv_bfloat16 *kc, __nv_bfloat16 *vc, int max_seq, int hd,
                                                   long long kv_slot_stride, const int *acc_nodes, int nodes_stride,
                                                   const int *acc_count, const int *d_prefix) {
  const int slot = blockIdx.z;
  const int count = acc_count[slot];
  if (count <= 1) return;
  acc_nodes += (long long)slot * nodes_stride;
  const int p_old = d_prefix[slot] - count;
  __nv_bfloat16 *basep = (blockIdx.y == 0 ? kc : vc) + slot * kv_slot_stride + (long long)blockIdx.x * max_seq * hd;
  for (int c = threadIdx.x; c * 8 < hd; c += blockDim.x) {
    for (int k = 1; k < count; ++k) {
      const int node = acc_nodes[k];
      if (node == k) continue;
      const uint4 v = *reinterpret_cast<const uint4 *>(basep + (long long)(p_old + node) * hd + c * 8);
      *reinterpret_cast<uint4 *>(basep + (long long)(p_old + k) * hd + c * 8) = v;
    }
  }
}

}  // namespace accept
}  // namespace pia

using namespace pia;
using namespace pia::accept;

extern "C" int64_t pia_accept_workspace_bytes(const pia_accept_config_t *cfg) {
  return cfg ? (int64_t)cfg->max_nodes * (int64_t)sizeof(int) : 0;
}

extern "C" int pia_accept(const pia_accept_config_t *cfg, const void *d_logits, const int32_t *d_ids,
                          const uint64_t *d_mask, int mask_words, int batch, int rows_per_slot, const int32_t *d_n,
                          int32_t *d_seq, int32_t *d_seq_len, int seq_stride, const int32_t *d_max_length,
                          uint32_t *d_rng, int32_t *d_accept_tokens, int32_t *d_accept_count, int32_t *d_accept_nodes,
                          int32_t *d_prefix_len, int32_t *d_finished, void *d_workspace, void *stream) {
  PIA_REQUIRE(cfg && d_logits && d_ids && d_mask && d_n && d_seq && d_seq_len && d_accept_tokens && d_accept_count &&
                  d_accept_nodes && d_prefix_len && d_finished && d_workspace, "null argument");
  PIA_REQUIRE(cfg->max_nodes >= 1 && cfg->max_nodes <= 128 && mask_words >= 1 && mask_words <= 2, "bad draft size");
  PIA_REQUIRE(batch >= 1 && rows_per_slot >= 1 && batch * rows_per_slot <= cfg->max_nodes,
              "batch * rows_per_slot must fit the %d draft rows", cfg->max_nodes);
  PIA_REQUIRE(cfg->vocab > 0 && cfg->n_eos >= 0 && cfg->n_eos <= 8, "bad accept config");
  PIA_REQUIRE(cfg->repetition_penalty > 0.f && cfg->inv_repetition_penalty > 0.f,
              "repetition_penalty and its reciprocal must be > 0");
  cudaStream_t s = (cudaStream_t)stream;
  int *row_tok = (int *)d_workspace;
  const bool pen = cfg->repetition_penalty != 1.0f;
  const size_t smem = pen ? (size_t)((cfg->vocab + 31) / 32) * 4 : 0;
  if (smem > 48 * 1024) {
    static bool attr_set = false;
    if (!attr_set) { PIA_CUDA_CHECK(cudaFuncSetAttribute(k_row_argmax, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr_set = true; }
    PIA_REQUIRE(smem <= 200 * 1024, "vocab too large for the penalty bitmap");
  }
  k_row_argmax<<<batch * rows_per_slot, accept::NT, smem, s>>>((const __nv_bfloat16 *)d_logits, cfg->vocab, d_ids,
                                                              (const unsigned long long *)d_mask, mask_words, d_n,
                                                              rows_per_slot, d_seq, seq_stride, d_seq_len,
                                                              cfg->repetition_penalty, cfg->inv_repetition_penalty,
                                                              d_rng, row_tok);
  PIA_LAUNCH_CHECK();
  k_accept_walk<<<batch, 128, 0, s>>>(*cfg, row_tok, d_ids, (const unsigned long long *)d_mask, mask_words, d_n,
                                      rows_per_slot, d_seq, seq_stride, d_seq_len, d_max_length, d_rng, d_accept_tokens,
                                      d_accept_count, d_accept_nodes, d_prefix_len, d_finished);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

extern "C" int pia_kv_compact(void *d_k_cache, void *d_v_cache, int n_layers, int n_kv_heads, int max_seq, int head_dim,
                              int batch, int64_t kv_slot_stride, const int32_t *d_accept_nodes, int nodes_stride,
                              const int32_t *d_accept_count, const int32_t *d_prefix_len, void *stream) {
  PIA_REQUIRE(d_k_cache && d_v_cache && d_accept_nodes && d_accept_count && d_prefix_len, "null argument");
  PIA_REQUIRE(head_dim % 8 == 0 && batch >= 1 && batch <= 65535, "bad kv_compact arguments");
  k_kv_compact<<<dim3(n_layers * n_kv_heads, 2, batch), 64, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16 *)d_k_cache, (__nv_bfloat16 *)d_v_cache, max_seq, head_dim, (long long)kv_slot_stride,
      d_accept_nodes, nodes_stride, d_accept_count, d_prefix_len);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}
