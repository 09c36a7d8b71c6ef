// FLOOD's hash-table lookahead draft behind its `Spec` interface (sm_90a) -- SURVEY.md 8f-4.
//
// Takes over the Triton kernels of /root/reference/flood/flood/ops/draft.py that flood/utils/speculative.py's
// `Lookahead(Spec)` (:23-124) calls:
//   update_draft_table_kernel   :92-165   (update_state)      -> k_flood_update
//   retrieve_draft_table_kernel :278-349  (proposal_draft)    -> k_flood_retrieve
//   verify_draft_kernel         :406-488  (verify_draft)      -> k_flood_verify
//   update_draft_cache_kernel   :547-559  (update_cache)      -> k_flood_cache_move
// The tables are FLOOD's: freq_table float32 [table_size], draft_table int32 [table_size, branch_length]; a 2-token
// context hashes to bucket (p0 * vocab + p1) % (table_size - branch_count) and owns the branch_count slots from there.
// Integer / byte work, HBM- and latency-bound: one warp per request (lanes = slots or branches), ballots instead of the
// Triton kernels' serial slot loops.
//
// update: the reference launches one program per 32 positions and lets them race on overlapping bucket windows; the
// result it produces when the programs run in order (which is what the Triton interpreter - the parity oracle - does)
// is the sequential application of the positions, and that is what this kernel computes: one warp walks the positions in
// order, the slot loops of a position are lane-parallel.
#include "common.cuh"

namespace pia {
namespace flood {

__device__ __forceinline__ int lane() { return threadIdx.x & 31; }

// one warp; sequential over positions (see header), lanes = slots j of the bucket window (branch_count <= 32)
__global__ void __launch_bounds__(32) k_flood_update(const int *tokens, int token_count, float *freq_table,
                                                     int *draft_table, long long size, int BL, int BC, long long vocab) {
  const int j = lane();
  for (int p = 0; p + 4 <= token_count; ++p) {
    const long long uid = (long long)tokens[p] * vocab + tokens[p + 1];
    const long long bucket = uid % (size - BC);
    // branch = tokens[p+2 .. p+2+BL) (0 beyond the list), branch_uid = its int32 sum (:118-123)
    int branch_uid = 0;
    for (int d = 0; d < BL; ++d) branch_uid += (p + 2 + d < token_count) ? tokens[p + 2 + d] : 0;
    // pass 1 (:127-148): the first slot that matches or is empty takes the branch
    int draft_uid = 0;
    float freq = 0.f;
    if (j < BC) {
      const int *row = draft_table + (bucket + j) * BL;
      for (int d = 0; d < BL; ++d) draft_uid += row[d];
      freq = freq_table[bucket + j];
    }
    const bool cand = j < BC && (branch_uid == draft_uid || freq == 0.f);
    const unsigned m = __ballot_sync(FULL, cand);
    const bool hit = m != 0u;
    if (hit && j == __ffs(m) - 1) {
      const bool match = branch_uid == draft_uid, empty = freq == 0.f;
      freq = match ? freq + 1.0f : 1.0f;
      if (empty) {
        int *row = draft_table + (bucket + j) * BL;
        for (int d = 0; d < BL; ++d) row[d] = (p + 2 + d < token_count) ? tokens[p + 2 + d] : 0;
      }
    }
    // pass 2 (:152-165): every slot decays; without a hit the slots that fall below 1 are replaced by the branch
    if (j < BC) {
      const float half = freq / 2.0f;
      const bool replace = half < 1.0f && !hit;
      freq_table[bucket + j] = replace ? 1.0f : half;
      if (replace) {
        int *row = draft_table + (bucket + j) * BL;
        for (int d = 0; d < BL; ++d) row[d] = (p + 2 + d < token_count) ? tokens[p + 2 + d] : 0;
      }
    }
    __syncwarp();
    __threadfence_block();
  }
}

// one warp per request; lanes = the BRANCH_LENGTH slots the reference examines (`indices = arange(BRANCH_LENGTH)`, :290)
__global__ void __launch_bounds__(32) k_flood_retrieve(const int *queries, const float *freq_table, const int *draft_table,
                                                       long long size, long long vocab, int BL, int BC, int RC,
                                                       int *out_tokens) {
  const int b = blockIdx.x, j = lane();
  const int p0 = queries[2 * b], p1 = queries[2 * b + 1];
  const long long bucket = ((long long)p0 * vocab + p1) % (size - BC);
  int *out = out_tokens + (long long)b * (RC * BL + 1);
  const float freq = j < BL ? freq_table[bucket + j] : -1.f;
  bool done = false;
  for (int i = 0; i <= 8 && !done; ++i) {
    // thresholds 64, 32, ..., 0.5 need >= RC hits (:300-325); the fallback (i == 8) takes whatever passes 0.5 (:327-345)
    const float thr = i < 8 ? exp2f(8.0f - (float)i - 2.0f) : 0.5f;
    const bool valid = j < BL && freq >= thr;
    const unsigned m = __ballot_sync(FULL, valid);
    const int rank = __popc(m & ((1u << j) - 1u));            // cumsum - 1
    const bool selected = valid && rank < RC;
    const int hits = min(__popc(m), RC);
    if (hits >= RC || i == 8) {
      if (selected) {
        const int *row = draft_table + (bucket + j) * BL;
        for (int d = 0; d < BL; ++d) out[1 + rank * BL + d] = row[d];
      }
      done = true;
    }
  }
  if (j == 0) out[0] = p1;
}

// one warp per request; lanes = branches (retrieve_count <= 32).  input / next ids are the flattened [bs, BC * BL] draft
// layout of retrieve_draft_table: [root, branch 0 (BL tokens), branch 1, ...] cut to BC * BL tokens (:491-530)
__global__ void __launch_bounds__(32) k_flood_verify(const int *input_ids, const int *next_ids, const int *cache_offsets,
                                                     int BC, int BL, int *output_ids, int *cache_src, int *cache_dst) {
  const int b = blockIdx.x, i = lane();
  const int *in = input_ids + (long long)b * BC * BL, *nx = next_ids + (long long)b * BC * BL;
  // tile[i][c]: c == 0 -> flat[0]; 1 <= c < BL -> flat[i*BL + c]; c == BL -> flat[(i+1)*BL] (or -1 for the last branch)
  auto tile = [&](const int *flat, int br, int c) -> int {
    if (c == 0) return flat[0];
    if (c < BL) return flat[br * BL + c];
    return br + 1 < BC ? flat[(br + 1) * BL] : -1;
  };
  int accept = 0;
  if (i < BC) {
    for (int jj = 0; jj < BL; ++jj) {
      if (tile(in, i, jj + 1) == tile(nx, i, jj)) ++accept; else break;
    }
  }
  // the first branch that reaches the maximum wins (`accept > max_accept_count`, :432); all-zero -> branch 0
  int best = accept, best_i = i < BC ? i : 0x7fffffff;
  for (int o = 16; o > 0; o >>= 1) {
    const int oa = __shfl_xor_sync(FULL, best, o), oi = __shfl_xor_sync(FULL, best_i, o);
    if (oa > best || (oa == best && oi < best_i)) { best = oa; best_i = oi; }
  }
  if (best == 0) best_i = 0;
  if (i == 0) {
    int *out = output_ids + (long long)b * (BL + 1);
    const int off = cache_offsets[b];
    for (int jj = 0; jj < BL; ++jj) {
      const int input_id = tile(in, best_i, jj + 1), next_id = tile(nx, best_i, jj);
      if (jj == 0) out[0] = next_id;
      if (input_id != next_id) break;
      out[jj + 1] = tile(nx, best_i, jj + 1);
      cache_src[b * BL + jj] = off + BL * best_i + 1 + jj;
      cache_dst[b * BL + jj] = off + 1 + jj;
    }
  }
}

// grid = moves; a move copies one cache row (16-byte vectors) unless src < 0 or src == dst (:547-559)
__global__ void __launch_bounds__(128) k_flood_cache_move(unsigned char *cache, long long row_bytes, const int *src,
                                                          const int *dst) {
  const int s = src[blockIdx.x];
  if (s < 0) return;
  const int d = dst[blockIdx.x];
  if (d == s) return;
  const unsigned char *from = cache + (long long)s * row_bytes;
  unsigned char *to = cache + (long long)d * row_bytes;
  if ((row_bytes & 15) == 0 && ((reinterpret_cast<uintptr_t>(cache) & 15) == 0)) {
    for (long long v = threadIdx.x; v * 16 < row_bytes; v += blockDim.x)
      reinterpret_cast<uint4 *>(to)[v] = reinterpret_cast<const uint4 *>(from)[v];
  } else {
    for (long long v = threadIdx.x; v < row_bytes; v += blockDim.x) to[v] = from[v];
  }
}

}  // namespace flood
}  // namespace pia

using namespace pia;
using namespace pia::flood;

static bool pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }

extern "C" int pia_flood_update_draft_table(const int32_t *d_tokens, int token_count, float *d_freq_table,
                                            int32_t *d_draft_table, int64_t table_size, int branch_length,
                                            int branch_count, int vocab, void *stream) {
  PIA_REQUIRE(d_freq_table && d_draft_table, "null table");
  PIA_REQUIRE(pow2(branch_length) && pow2(branch_count) && branch_count <= 32 && branch_length <= 32 &&
                  table_size > branch_count && vocab > 0, "bad table geometry");
  if (token_count <= 3) return PIA_OK;  // min segment: 2 prefix + 2 draft tokens (draft.py:181-182)
  PIA_REQUIRE(d_tokens, "null tokens");
  k_flood_update<<<1, 32, 0, (cudaStream_t)stream>>>(d_tokens, token_count, d_freq_table, d_draft_table,
                                                    (long long)table_size, branch_length, branch_count, (long long)vocab);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

extern "C" int pia_flood_retrieve_draft_table(const int32_t *d_queries, int batch, const float *d_freq_table,
                                              const int32_t *d_draft_table, int64_t table_size, int vocab,
                                              int branch_length, int branch_count, int retrieve_count,
                                              int32_t *d_out_tokens, void *stream) {
  PIA_REQUIRE(d_queries && d_freq_table && d_draft_table && d_out_tokens && batch >= 1, "null argument");
  PIA_REQUIRE(pow2(branch_length) && pow2(branch_count) && branch_count <= 32 && branch_length <= 32 &&
                  retrieve_count >= 1 && retrieve_count <= branch_count && table_size > branch_count && vocab > 0,
              "bad table geometry");
  k_flood_retrieve<<<batch, 32, 0, (cudaStream_t)stream>>>(d_queries, d_freq_table, d_draft_table, (long long)table_size,
                                                          (long long)vocab, branch_length, branch_count, retrieve_count,
                                                          d_out_tokens);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

extern "C" int pia_flood_verify_draft(const int32_t *d_input_ids, const int32_t *d_next_ids,
                                      const int32_t *d_cache_offsets, int batch, int branch_count, int branch_length,
                                      int32_t *d_output_ids, int32_t *d_cache_src, int32_t *d_cache_dst, void *stream) {
  PIA_REQUIRE(d_input_ids && d_next_ids && d_cache_offsets && d_output_ids && d_cache_src && d_cache_dst && batch >= 1,
              "null argument");
  PIA_REQUIRE(branch_count >= 1 && branch_count <= 32 && branch_length >= 1, "bad draft geometry");
  k_flood_verify<<<batch, 32, 0, (cudaStream_t)stream>>>(d_input_ids, d_next_ids, d_cache_offsets, branch_count,
                                                        branch_length, d_output_ids, d_cache_src, d_cache_dst);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

extern "C" int pia_flood_update_draft_cache(void *d_cache, int64_t row_bytes, const int32_t *d_src, const int32_t *d_dst,
                                            int count, void *stream) {
  PIA_REQUIRE(d_cache && d_src && d_dst && row_bytes > 0 && count >= 0, "bad cache move");
  if (count == 0) return PIA_OK;
  k_flood_cache_move<<<count, 128, 0, (cudaStream_t)stream>>>((unsigned char *)d_cache, (long long)row_bytes, d_src, d_dst);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}
