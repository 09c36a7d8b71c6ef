// GPU-resident trie draft cache for PIA LOOKAHEAD (sm_90a).
//
// Takes over common/lookahead_cache.py of the reference (Tree :24-333, LookaheadCache :336-587): the
// reference keeps one Python dict-of-dicts per first token; here the whole forest lives in HBM as
//   * 32-byte node records (one DRAM sector each): {token, n_child, child, cap, fo(f64), fi(f32), aux}
//   * 8-byte (token,node) child entries in insertion order for nodes with >= 2 children
//     (a single child is stored inline, so n-gram chains cost one sector per node)
//   * per-first-token root table, per-tree counters and the two "touched trees" lists.
// Child ORDER is part of the contract: the reference sorts children by fm with Python's stable sort, so
// ties fall back to dict insertion order (lookahead_cache.py:254-258); child lists therefore only ever
// append, and squeeze compacts them in place.
//
// Frequencies: fo = freqs[-1] is an IEEE double exactly as in Python (squeeze halves it, :306-307);
// fi = freqs[idx] only ever counts +1.0 and is reset to 0, so fp32 holds it exactly.  fm is evaluated
// as (1-w)*fi + w*fo with two rounded multiplies and one rounded add (__dmul_rn/__dadd_rn, no FMA).
//
// Kernels: k_put_prepare / k_put_insert / k_put_finish (put, stream_put :349-406),
//          k_get (hier_get / one_get -> Tree.get :65-144, 224-293, 171-222): warp match, level-synchronous frequency
//                walk (pruned by the parent >= child count bound; full, as an 8-CTA cluster per row, when that bound is
//                not known to hold), k-th largest from exact shared-memory histograms, DFS emit with ranked frames,
//          k_reset_input (:320-333, 566-570), k_squeeze (:295-318, 572-576), k_fresh (:563-564).
// Host:    pia_trie_compact (storage reclamation between requests), export / import (save_mem / load_mem).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <vector>

#include "common.cuh"

namespace pia {
namespace trie {

struct __align__(32) Node {
  int token;
  int n_child;
  int child;  // cap == 0: node id of the only child (n_child <= 1); cap > 0: offset of the child block
  int cap;    // capacity of the child block in the edge pool (0 = inline)
  double fo;
  float fi;   // input slot 0
  int aux;
};
static_assert(sizeof(Node) == 32, "node record must be one 32-byte sector");

struct Hdr {
  unsigned long long node_top, edge_top;
  unsigned long long nodes_visited, edges_visited;
  int n_trees, n_upd, n_updin, n_upd_stale;
  int err;
  int n_eos;
  int eos[8];
  int max_node, max_out;
  int put_len, put_npos;
  int get_ticket, get_done;  // dynamic row scheduling of batched k_get (self-resetting)
};


struct Dev {
  Node *nodes;
  int2 *edges;
  float *fi_extra;  // [(n_slots-1), node_cap]
  Hdr *hdr;
  int *root_of, *tree_n_node, *tree_n_out, *tree_flags;
  int *upd_list, *updin_list;
  unsigned *stop_bits;
  int *out_buf, *out_len;
  int out_cap;
  long long node_cap, edge_cap;
  int vocab, n_slots;
  int *frontier;
  int fr_cap, max_resident;
};

constexpr int ERR_NODE_POOL = 1, ERR_EDGE_POOL = 2, ERR_FRONTIER = 4, ERR_OUTBUF = 8, ERR_HIST = 16, ERR_TOKEN = 32;
constexpr int FLAG_UPD = 1, FLAG_UPDIN = 2;
constexpr int NT = 256;  // threads per CTA of every trie kernel

// -DPIA_TRIE_PHASES: the leader's thread 0 prints the nanoseconds between the phases of one tree_get (diagnostic builds
// only: scripts/time_trie_get.py)
#ifdef PIA_TRIE_PHASES
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define PHASE(i) do { if (threadIdx.x == 0 && rank == 0) ph[i] = gtime(); } while (0)
#else
#define PHASE(i) do { } while (0)
#endif

__device__ __forceinline__ float load_fi(const Dev &D, const Node &nd, int id, int idx) {
  return idx == 0 ? nd.fi : D.fi_extra[(long long)(idx - 1) * D.node_cap + id];
}
__device__ __forceinline__ bool is_stop(const Dev &D, int tok) { return (D.stop_bits[tok >> 5] >> (tok & 31)) & 1u; }
__device__ __forceinline__ unsigned long long dbits(double x) { return (unsigned long long)__double_as_longlong(x); }
// fm = (1-w)*fi + w*fo, IEEE double, no contraction (lookahead_cache.py:151, :254)
__device__ __forceinline__ double mix_freq(double one_minus_w, double w, double fi, double fo) {
  return __dadd_rn(__dmul_rn(one_minus_w, fi), __dmul_rn(w, fo));
}

// ---------------------------------------------------------------------------------------------------
// warp-cooperative child lookup: dict.get(token) on a node's children
// ---------------------------------------------------------------------------------------------------
__device__ int find_child(const Dev &D, const Node &p, int token) {
  if (p.n_child == 0) return -1;
  if (p.cap == 0) {
    int c = p.child;
    return D.nodes[c].token == token ? c : -1;
  }
  const int lane = lane_id();
  // UF x 32 child entries are in flight before the first ballot: with one load per lane and iteration the scan of a
  // hot node's child block (tens of thousands of entries under a frequent token) was one L2 round trip per 32 entries
  constexpr int UF = 8;
  for (int base = 0; base < p.n_child; base += 32 * UF) {
    int2 e[UF];
#pragma unroll
    for (int u = 0; u < UF; ++u) {
      const int i = base + u * 32 + lane;
      e[u] = i < p.n_child ? D.edges[p.child + i] : make_int2(-1, -1);
    }
#pragma unroll
    for (int u = 0; u < UF; ++u) {
      const unsigned m = __ballot_sync(FULL, base + u * 32 + lane < p.n_child && e[u].x == token);
      if (m) return __shfl_sync(FULL, e[u].y, __ffs(m) - 1);
    }
  }
  return -1;
}

// ---------------------------------------------------------------------------------------------------
// put / stream_put
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int live_slot(const Dev &D, int slot, const int *d_slot) {
  if (d_slot != nullptr) { slot = *d_slot; if (slot < 0 || slot >= D.n_slots) slot = 0; }
  return slot;
}

__global__ void __launch_bounds__(NT) k_put_prepare(Dev D, const int *tokens, int n, const int *d_n, int B,
                                                    int is_stream, int final, int slot, const int *d_slot) {
  __shared__ int s_cut;
  const int tid = threadIdx.x;
  slot = live_slot(D, slot, d_slot);
  int n_in = n;
  if (d_n != nullptr) { int v = *d_n; n_in = v < n ? v : n; }
  if (n_in < 0) n_in = 0;
  if (tid == 0) s_cut = n_in;
  __syncthreads();
  // eos truncation: cut at the first occurrence of any eos id (lookahead_cache.py:350-352, 378-380)
  const int n_eos = D.hdr->n_eos;
  for (int i = tid; i < n_in; i += NT) {
    int t = tokens[i];
    bool hit = false;
    for (int e = 0; e < n_eos; ++e) hit |= (t == D.hdr->eos[e]);
    if (t < 0 || t >= D.vocab) { atomicOr(&D.hdr->err, ERR_TOKEN); hit = true; }
    if (hit) atomicMin(&s_cut, i);
  }
  __syncthreads();
  const int n_eff = s_cut;
  if (is_stream) {
    int *buf = D.out_buf + (long long)slot * D.out_cap;
    int have = D.out_len[slot];
    int room = D.out_cap - have;
    int take = n_eff;
    if (take > room) { take = room > 0 ? room : 0; if (tid == 0) atomicOr(&D.hdr->err, ERR_OUTBUF); }
    for (int i = tid; i < take; i += NT) buf[have + i] = tokens[i];
    __syncthreads();
    if (tid == 0) {
      int ts = have + take;
      int min_bl = final ? 1 : B;
      D.out_len[slot] = ts;
      D.hdr->put_len = ts;
      D.hdr->put_npos = ts > min_bl ? ts - min_bl : 0;
    }
  } else if (tid == 0) {
    D.hdr->put_len = n_eff;
    D.hdr->put_npos = n_eff >= 2 ? n_eff - 1 : 0;
  }
}

// one warp: Tree.put of `path[0..len)` into the tree keyed by `key` (lookahead_cache.py:33-63)
__device__ void warp_insert(const Dev &D, int key, const int *path, int len, bool out_mode, int idx) {
  const int lane = lane_id();
  int root = D.root_of[key];
  if (root < 0) {
    if (lane == 0) {
      unsigned long long id = atomicAdd(&D.hdr->node_top, 1ull);
      if (id >= (unsigned long long)D.node_cap) { atomicOr(&D.hdr->err, ERR_NODE_POOL); root = -1; }
      else {
        root = (int)id;
        Node r; r.token = key; r.n_child = 0; r.child = -1; r.cap = 0; r.fo = 0.0; r.fi = 0.f; r.aux = 0;
        D.nodes[root] = r;
        D.root_of[key] = root;
        D.tree_n_node[key] = 0; D.tree_n_out[key] = 0;
        atomicAdd(&D.hdr->n_trees, 1);
      }
    }
    root = __shfl_sync(FULL, root, 0);
    if (root < 0) return;
  }
  __syncwarp();
  int cur = root;
  for (int j = 0; j < len; ++j) {
    Node pn = D.nodes[cur];
    const int tok = path[j];
    int c = find_child(D, pn, tok);
    if (c >= 0) {  // existing node: freqs[idx] += 1 (:53)
      if (lane == 0) {
        if (out_mode) D.nodes[c].fo += 1.0;
        else if (idx == 0) D.nodes[c].fi += 1.0f;
        else D.fi_extra[(long long)(idx - 1) * D.node_cap + c] += 1.0f;
      }
      __syncwarp();
      cur = c;
      continue;
    }
    // missing suffix: _pack a chain of r new nodes (:57-63) and hang it under `cur` as its LAST child
    const int r = len - j;
    long long base = -1;
    if (lane == 0) {
      unsigned long long b = atomicAdd(&D.hdr->node_top, (unsigned long long)r);
      if (b + r > (unsigned long long)D.node_cap) atomicOr(&D.hdr->err, ERR_NODE_POOL);
      else base = (long long)b;
    }
    base = __shfl_sync(FULL, base, 0);
    if (base < 0) return;
    for (int k = lane; k < r; k += 32) {
      Node nn;
      nn.token = path[j + k];
      nn.n_child = (k < r - 1) ? 1 : 0;
      nn.child = (k < r - 1) ? (int)(base + k + 1) : -1;
      nn.cap = 0;
      nn.fo = out_mode ? 1.0 : 0.0;
      nn.fi = (!out_mode && idx == 0) ? 1.0f : 0.0f;
      nn.aux = 0;
      D.nodes[base + k] = nn;
      for (int s = 1; s < D.n_slots; ++s)
        D.fi_extra[(long long)(s - 1) * D.node_cap + base + k] = (!out_mode && idx == s) ? 1.0f : 0.0f;
    }
    // link
    if (pn.n_child == 0 && pn.cap == 0) {
      if (lane == 0) { D.nodes[cur].child = (int)base; D.nodes[cur].n_child = 1; }
    } else if (pn.cap == 0) {  // inline -> block of 4
      long long off = -1;
      if (lane == 0) {
        unsigned long long o = atomicAdd(&D.hdr->edge_top, 4ull);
        if (o + 4 > (unsigned long long)D.edge_cap) atomicOr(&D.hdr->err, ERR_EDGE_POOL);
        else {
          off = (long long)o;
          D.edges[off] = make_int2(D.nodes[pn.child].token, pn.child);
          D.edges[off + 1] = make_int2(tok, (int)base);
          D.nodes[cur].child = (int)off; D.nodes[cur].cap = 4; D.nodes[cur].n_child = 2;
        }
      }
      off = __shfl_sync(FULL, off, 0);
      if (off < 0) return;
    } else if (pn.n_child < pn.cap) {
      if (lane == 0) { D.edges[pn.child + pn.n_child] = make_int2(tok, (int)base); D.nodes[cur].n_child = pn.n_child + 1; }
    } else {  // grow: copy into a block of twice the capacity (the old block is abandoned)
      long long off = -1;
      const int ncap = pn.cap * 2;
      if (lane == 0) {
        unsigned long long o = atomicAdd(&D.hdr->edge_top, (unsigned long long)ncap);
        if (o + ncap > (unsigned long long)D.edge_cap) atomicOr(&D.hdr->err, ERR_EDGE_POOL);
        else off = (long long)o;
      }
      off = __shfl_sync(FULL, off, 0);
      if (off < 0) return;
      for (int k = lane; k < pn.n_child; k += 32) D.edges[off + k] = D.edges[pn.child + k];
      if (lane == 0) {
        D.edges[off + pn.n_child] = make_int2(tok, (int)base);
        D.nodes[cur].child = (int)off; D.nodes[cur].cap = ncap; D.nodes[cur].n_child = pn.n_child + 1;
      }
    }
    if (lane == 0) {  // counters (:48-50)
      D.tree_n_node[key] += r;
      if (out_mode) D.tree_n_out[key] += r;
    }
    __syncwarp();
    return;
  }
}

__device__ void add_update(const Dev &D, int key, int flag, int *list, int *count) {
  int old = atomicOr(&D.tree_flags[key], flag);
  if (!(old & flag)) { int p = atomicAdd(count, 1); list[p] = key; }
}

// One warp per position p.  Positions that share their key token touch the same tree and must be applied
// in list order (child insertion order is observable), so the first occurrence of a key is the "leader"
// and replays every later occurrence itself; distinct keys own disjoint trees and run concurrently.
__global__ void __launch_bounds__(NT) k_put_insert(Dev D, const int *tokens, int B, int mode, int idx, int is_stream,
                                                   int slot, const int *d_slot) {
  const int lane = lane_id();
  slot = live_slot(D, slot, d_slot);
  const int p = blockIdx.x * (NT / 32) + warp_id();
  const int npos = D.hdr->put_npos, len = D.hdr->put_len;
  if (p >= npos) return;
  const int *src = is_stream ? D.out_buf + (long long)slot * D.out_cap : tokens;
  const int key = src[p];
  if (key < 0 || key >= D.vocab) return;
  if (is_stream && is_stop(D, key)) return;  // stop words never become tree keys (:388-389)
  for (int q0 = 0; q0 < p; q0 += 32) {
    int q = q0 + lane;
    if (__any_sync(FULL, q < p && src[q] == key)) return;  // not the leader
  }
  const bool existed = D.root_of[key] >= 0;
  const bool out_mode = (mode == PIA_MODE_OUTPUT);
  int count = 0;
  for (int q0 = p; q0 < npos; q0 += 32) {
    int q = q0 + lane;
    unsigned m = __ballot_sync(FULL, q < npos && src[q] == key);
    while (m) {
      int b = __ffs(m) - 1;
      m &= m - 1;
      int qq = q0 + b;
      int plen = len - (qq + 1);
      if (plen > B) plen = B;
      warp_insert(D, key, src + qq + 1, plen, out_mode, idx);
      ++count;
    }
  }
  if (lane == 0) {
    // put(): only a tree that already existed when a position reached it joins _update_trees (:361-367);
    // stream_put(): always (:400)
    if (is_stream || existed || count >= 2) add_update(D, key, FLAG_UPD, D.upd_list, &D.hdr->n_upd);
    if (mode == PIA_MODE_INPUT) add_update(D, key, FLAG_UPDIN, D.updin_list, &D.hdr->n_updin);
  }
}

// Tree.put on one tree (:33-37)
__global__ void k_tree_put(Dev D, int key, const int *tokens, int n, int mode, int idx) {
  if (n > 0) warp_insert(D, key, tokens, n, mode == PIA_MODE_OUTPUT, idx);
}

__global__ void k_put_finish(Dev D, int B, int final, int slot, const int *d_slot) {
  slot = live_slot(D, slot, d_slot);
  // stream_put tail: keep the last B tokens as carry (:401-402) or clear on final (:404)
  __shared__ int tmp[128];
  const int tid = threadIdx.x;
  int *buf = D.out_buf + (long long)slot * D.out_cap;
  const int ts = D.hdr->put_len, npos = D.hdr->put_npos;
  if (final) { if (tid == 0) D.out_len[slot] = 0; return; }
  if (npos > 0) {  // ts > B
    if (tid < B) tmp[tid] = buf[ts - B + tid];
    __syncthreads();
    if (tid < B) buf[tid] = tmp[tid];
    if (tid == 0) D.out_len[slot] = B;
  }
}

// ---------------------------------------------------------------------------------------------------
// Breadth-first walk below `start`; visit(id, node) -> descend?   One CTA, or the CL CTAs of a thread-block cluster
// working on the same frontier (a hot subtree is a latency problem: ~3 dependent memory round trips per node, so the
// cure is more loads in flight than one SM's 256 threads can hold).
//   * the level counters live in the LEADER CTA's shared memory (`sh`, a generic pointer that is a distributed-
//     shared-memory address for the other ranks); every warp reserves its slice of the next level with one atomic;
//   * CL == 1: the first SFR entries of every level stay in shared memory (`sfr`), only larger levels touch the
//     per-CTA region in HBM - cold queries (a few hundred nodes) never write global memory;
//   * CL > 1: the frontier is the leader's region in global memory, written/read through L2 (st.cg / ld.cg), one
//     cluster barrier (release/acquire) per level.
// ---------------------------------------------------------------------------------------------------
struct BfsShared { int next_cnt[3]; int err; };  // three rotating level counters: one barrier per BFS level
constexpr int BFS_U = 4;                         // frontier entries per thread and round
static_assert(NT * BFS_U == 1024, "bfs_below searches its expansion table in 10 steps");
// wsum is 16-byte aligned: the compiler reads it with 128-bit loads, and unaligned those reach back into src[]
// (harmless, but compute-sanitizer racecheck reports the overlap with the thread that writes src's last entry)
struct ExpandTab { int start[NT * BFS_U + 1]; int src[NT * BFS_U]; alignas(16) int wsum[2][NT / 32]; int rbase; };  // see bfs_below
constexpr int SFR = 1024;                        // shared-memory frontier entries per buffer (CL == 1)

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned cluster_rank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ unsigned cluster_size() { unsigned r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
// generic address of `p` (a generic pointer into this CTA's shared memory) in CTA `rank` of the cluster
template <class T>
__device__ __forceinline__ T *map_to_rank(T *p, unsigned rank) {
  unsigned long long r;
  asm volatile("mapa.u64 %0, %1, %2;" : "=l"(r) : "l"((unsigned long long)p), "r"(rank));
  return reinterpret_cast<T *>(r);
}

// node records and child entries are read-only while a query kernel runs: the non-coherent path lets the compiler keep
// several of them in flight across the frontier stores in between
template <bool RO>
__device__ __forceinline__ Node load_node(const Node *p) {
  if (!RO) return *p;  // walks that modify the records they visit (reset_input_freqs) use coherent loads
  union { Node n; uint4 v[2]; } u;
  u.v[0] = __ldg(reinterpret_cast<const uint4 *>(p));
  u.v[1] = __ldg(reinterpret_cast<const uint4 *>(p) + 1);
  return u.n;
}

struct Frontier {
  int *g;  // global region (fr_cap entries)
  int *s;  // shared-memory head (SFR entries) or nullptr
  __device__ __forceinline__ int get(int e) const { return (s != nullptr && e < SFR) ? s[e] : __ldcg(g + e); }
  __device__ __forceinline__ void put(int e, int v) const { if (s != nullptr && e < SFR) s[e] = v; else __stcg(g + e, v); }
};

// level_end() runs in every thread (uniform) between two levels, after the level barrier: the query walk uses it to
// tighten its pruning thresholds (CL == 1 only).
template <bool RO, class Visit, class LevelEnd>
__device__ __forceinline__ void bfs_below(const Dev &D, int start, int *fr0, int *fr1, int *sfr, ExpandTab *xt,
                                          BfsShared *sh, int CL, int rank, Visit &&visit, LevelEnd &&level_end,
                                          unsigned long long &nv,
                                          unsigned long long &ne) {
  const int tid = threadIdx.x, lane = lane_id();
  auto sync_all = [&]() { if (CL > 1) cluster_sync_all(); else __syncthreads(); };
  const Node s = load_node<RO>(D.nodes + start);
  if (rank == 0 && tid == 0) { sh->next_cnt[0] = 0; sh->next_cnt[1] = 0; sh->next_cnt[2] = 0; }
  Frontier cur = {fr0, sfr}, nxt = {fr1, sfr ? sfr + SFR : nullptr};
  int round = 0;
  int cnt = s.n_child;
  if (s.cap == 0) {
    if (rank == 0 && tid == 0 && cnt == 1) cur.put(0, s.child);
  } else {
    if (cnt > D.fr_cap) { if (rank == 0 && tid == 0) atomicOr(&sh->err, ERR_FRONTIER); cnt = 0; }
    for (int i0 = rank * NT + tid; i0 < cnt; i0 += 4 * CL * NT) {  // four child entries in flight per thread
      int c[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { const int i = i0 + j * CL * NT; c[j] = i < cnt ? __ldg(&D.edges[s.child + i].y) : 0; }
#pragma unroll
      for (int j = 0; j < 4; ++j) { const int i = i0 + j * CL * NT; if (i < cnt) cur.put(i, c[j]); }
    }
    if (rank == 0 && tid == 0) ne += cnt;
  }
  sync_all();
#ifdef PIA_TRIE_PHASES
  __shared__ unsigned long long lv_t[16], lv_e[16];
  __shared__ int lv_c[16], lv_n;
  if (tid == 0) { lv_e[0] = gtime(); lv_n = 1; }
#endif
  for (int level = 0; cnt > 0; ++level) {
    int *push_cnt = &sh->next_cnt[(level + 1) % 3];
    if (rank == 0 && tid == 0) sh->next_cnt[(level + 2) % 3] = 0;  // the counter of the level after next: idle during this level
    // U frontier entries per thread and iteration: the U node records (dependent on the U frontier loads) are all in
    // flight before the first is inspected - one record per thread at a time left a hot subtree latency-bound
    constexpr int U = BFS_U;
    int level_base = 0;
    for (int base = rank * NT * U; base < cnt; base += CL * NT * U) {
      int id[U], push[U];
      Node nd[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int e = base + u * NT + tid;
        id[u] = e < cnt ? cur.get(e) : -1;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (id[u] >= 0) nd[u] = load_node<RO>(D.nodes + id[u]);
        else { nd[u].child = -1; nd[u].cap = 0; nd[u].n_child = 0; }
      }
      // visit() is called by every lane (valid or not): it may use warp collectives
      int mine = 0;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool valid = id[u] >= 0;
        if (valid) ++nv;
        const bool descend = visit(id[u], nd[u], valid);
        push[u] = (valid && descend && nd[u].n_child > 0) ? nd[u].n_child : 0;
        mine += push[u];
      }
      // Load-balanced expansion.  The CTA reserves one slice [rbase, rbase + total) of the next level per round (block
      // scan + one atomic) and fills it with all threads, flat index by flat index: each (thread, u) entry publishes
      // where its children start in the slice and where they come from (the inline child, or its block of child
      // entries), a flat index finds its entry by binary search.  A hot node with hundreds of children no longer
      // serialises the level behind one lane or one warp, four child entries are in flight per thread, stores are
      // contiguous.
      int incl = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
      int *wsum = xt->wsum[round & 1];  // double buffered: the sparse path below has no second barrier
      ++round;
      if (lane == 31) wsum[warp_id()] = incl;
      __syncthreads();
      int woff = 0, total = 0;
#pragma unroll
      for (int w2 = 0; w2 < NT / 32; ++w2) { const int v = wsum[w2]; if (w2 < warp_id()) woff += v; total += v; }
      if (total == 0) continue;  // uniform
      const bool dense = total > 64;
      int rbase;
      if (CL == 1) {  // a lone CTA keeps the level's running count in a register: no atomic, no broadcast
        rbase = level_base;
        level_base += total;
      } else {
        if (tid == 0) xt->rbase = atomicAdd(push_cnt, total);
      }
      if (dense) {
        int off = woff + incl - mine;
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const bool one = push[u] == 1 && nd[u].cap == 0;
          xt->start[tid * U + u] = off;
          xt->src[tid * U + u] = one ? -(nd[u].child + 1) : nd[u].child;
          off += push[u];
        }
        if (tid == NT - 1) xt->start[NT * U] = total;
      }
      if (dense || CL > 1) __syncthreads();
      if (CL > 1) rbase = xt->rbase;
#pragma unroll
      for (int u = 0; u < U; ++u) if (!(push[u] == 1 && nd[u].cap == 0)) ne += push[u];
      if (rbase + total > D.fr_cap) {
        if (tid == 0) atomicOr(&sh->err, ERR_FRONTIER);
      } else if (!dense) {
        // a handful of children in the whole round (chains, cold subtrees): every thread appends its own
        int pos = rbase + woff + incl - mine;
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (push[u] == 1 && nd[u].cap == 0) nxt.put(pos, nd[u].child);
          else {
            for (int k0 = 0; k0 < push[u]; k0 += 4) {
              int c[4];
#pragma unroll
              for (int j = 0; j < 4; ++j)
                c[j] = k0 + j < push[u] ? (RO ? __ldg(&D.edges[nd[u].child + k0 + j].y) : D.edges[nd[u].child + k0 + j].y) : 0;
#pragma unroll
              for (int j = 0; j < 4; ++j) if (k0 + j < push[u]) nxt.put(pos + k0 + j, c[j]);
            }
          }
          pos += push[u];
        }
      } else {
        for (int f0 = 0; f0 < total; f0 += NT * 4) {
          int val[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int f = f0 + j * NT + tid;
            val[j] = 0;
            if (f < total) {
              int lo = 0, hi = NT * U;  // the entry e with start[e] <= f < start[e + 1] (empty entries never qualify)
#pragma unroll
              for (int step = 0; step < 10; ++step) { const int mid = (lo + hi) >> 1; if (xt->start[mid] <= f) lo = mid; else hi = mid; }
              const int src = xt->src[lo];
              const int k = f - xt->start[lo];
              val[j] = src < 0 ? -(src + 1) : (RO ? __ldg(&D.edges[src + k].y) : D.edges[src + k].y);
            }
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) { const int f = f0 + j * NT + tid; if (f < total) nxt.put(rbase + f, val[j]); }
        }
      }
      if ((dense || CL > 1) && base + CL * NT * U < cnt) __syncthreads();  // table / rbase are rewritten by the next round
    }
    sync_all();
    cnt = CL == 1 ? level_base : *push_cnt;
    if (cnt > D.fr_cap) cnt = 0;  // overflowed level: err already set
    const Frontier t = cur; cur = nxt; nxt = t;
#ifdef PIA_TRIE_PHASES
    if (tid == 0 && rank == 0 && level < 15) { lv_t[level + 1] = gtime(); lv_c[level + 1] = cnt; lv_n = level + 2; }
#endif
    if (cnt > 0) level_end(cnt);
#ifdef PIA_TRIE_PHASES
    if (tid == 0 && rank == 0 && level < 15) lv_e[level + 1] = gtime();
#endif
  }
  sync_all();
#ifdef PIA_TRIE_PHASES
  if (tid == 0 && rank == 0)
    for (int i = 1; i < lv_n; ++i)
      printf("  bfs level %d: walk %llu ns, level_end %llu ns, next cnt %d\n", i - 1, lv_t[i] - lv_e[i - 1], lv_e[i] - lv_t[i], lv_c[i]);
#endif
}

// ---------------------------------------------------------------------------------------------------
// get
// ---------------------------------------------------------------------------------------------------
constexpr int HCAP = 512;                        // distinct frequency values per histogram
constexpr unsigned long long HEMPTY = ~0ull;
static_assert(HCAP % NT == 0, "kth_value compacts with whole warps");

struct Hist { unsigned long long key[HCAP]; unsigned cnt[HCAP]; };

__device__ __forceinline__ void hist_add(Hist *h, unsigned long long bits, unsigned count, int *ovf) {
  unsigned s = (unsigned)((bits * 0x9E3779B97F4A7C15ull) >> 54) & (HCAP - 1);
  for (int probe = 0; probe < HCAP; ++probe) {
    unsigned long long old = atomicCAS(&h->key[s], HEMPTY, bits);
    if (old == HEMPTY || old == bits) { atomicAdd(&h->cnt[s], count); return; }
    s = (s + 1) & (HCAP - 1);
  }
  *ovf = 1;
}
// one update per distinct value of a warp (all lanes call; `active` lanes contribute)
__device__ __forceinline__ void warp_hist_add(Hist *h, unsigned long long bits, bool active, int *ovf) {
  const unsigned m = __match_any_sync(FULL, active ? bits : HEMPTY);
  if (active && lane_id() == __ffs(m) - 1) hist_add(h, bits, __popc(m), ovf);
}

struct GetParams {
  const int *queries, *qlen, *d_idx, *d_max_seq;
  int batch, q_stride, max_query, idx, dl, bl, min_in, min_out, mode, kind, flags, max_seq;
  int *out_ids; unsigned long long *out_mask; int *out_n, *out_sizes, *out_nsizes, *status;
  int prune;  // 1: the frequency walk may skip subtrees that cannot reach the thresholds (see tree_get)
};

template <int MAXS, int MAXD>
struct GetSmem {
  Hist hin, hout;
  // merge pool for frame construction
  unsigned long long pkey[MAXS + NT];
  int pord[MAXS + NT], pnode[MAXS + NT], ptok[MAXS + NT], pflag[MAXS + NT];
  unsigned long long qkey[MAXS];
  int qord[MAXS], qnode[MAXS], qtok[MAXS], qflag[MAXS];
  // DFS frames
  int fnode[MAXD][MAXS], ftok[MAXD][MAXS];
  unsigned char fflag[MAXD][MAXS];
  int fcnt[MAXD], fcur[MAXD], fpid[MAXD];
  // outputs
  unsigned long long mask[MAXS][(MAXS + 63) / 64];
  int ids[MAXS];
  int q[16];
  int sfr[2 * SFR];  // shared-memory head of the two BFS frontiers
  ExpandTab xt;
  BfsShared bfs;
  int hist_ovf;
  long long n_live, n_in, n_out;
  unsigned long long thr_bits; int thr_found;
  unsigned long long hk[HCAP]; unsigned hc[HCAP]; int hn;  // the occupied histogram slots, compacted (kth_value)
  unsigned long long t_in, t_out;                          // running pruning thresholds (bits of non-negative doubles)
  int pool_n, pool_ovf, match_node, n, sizes0, sizes1, depth, state, ticket;
  int pub_rc, pub_n;  // leader -> followers of a cluster: result of the last tree_get
  int best_node, best_tok; unsigned long long best_key; int best_ord;
};

constexpr int CF_FI = 1, CF_FO = 2, CF_KIDS = 4;

// sorted(values, reverse=True)[rank-1] from a histogram -> S->thr_bits; false if rank is out of range.  CTA-uniform,
// synchronises.  The occupied slots (a few dozen distinct n-gram counts) are compacted first, then ranked pairwise.
// `lo`: a known lower bound of the answer (0 = none) - slots below it are left out of the pairwise ranking.
template <class SM>
__device__ bool kth_value(SM *S, const Hist *h, long long rank, unsigned long long lo) {
  const int tid = threadIdx.x;
  __syncthreads();
  if (tid == 0) { S->hn = 0; S->thr_found = 0; }
  __syncthreads();
  for (int s = tid; s < HCAP; s += NT) {  // HCAP is a multiple of NT: whole warps
    const unsigned long long k = h->key[s];
    const bool keep = k != HEMPTY && k >= lo;
    const unsigned m = __ballot_sync(FULL, keep);
    int base = 0;
    if (lane_id() == 0 && m) base = atomicAdd(&S->hn, __popc(m));
    base = __shfl_sync(FULL, base, 0);
    if (keep) { const int j = base + __popc(m & ((1u << lane_id()) - 1)); S->hk[j] = k; S->hc[j] = h->cnt[s]; }
  }
  __syncthreads();
  const int n = S->hn;
  for (int e = tid; e < n; e += NT) {
    const unsigned long long k = S->hk[e];
    long long greater = 0;
    for (int j = 0; j < n; ++j) if (S->hk[j] > k) greater += S->hc[j];
    if (greater < rank && rank <= greater + (long long)S->hc[e]) { S->thr_bits = k; S->thr_found = 1; }
  }
  __syncthreads();
  return S->thr_found != 0;
}


// Builds the sorted candidate list of `parent`'s children for one DFS frame: children that pass the
// threshold filter (lookahead_cache.py:264-272), ordered by fm descending, ties by insertion order (:254-258),
// truncated to K (no more than K can still be emitted).
template <int MAXS, int MAXD, int U>
__device__ __noinline__ int build_frame_u(const Dev &D, GetSmem<MAXS, MAXD> *S, const Node p, int K, int idx, int mode, double omw,
                           double w, double min_in, double min_out, double min_mix, int *onode, int *otok,
                           unsigned char *oflag, unsigned long long &nv, unsigned long long &ne) {
  const int tid = threadIdx.x;
  const int C = p.n_child;
#ifdef PIA_TRIE_PHASES
  const unsigned long long tf0 = gtime();
#endif
  int m = 0;  // current size of the running top list (uniform)
  // U child chunks are fetched together: a frame below a hot node ranks thousands of children, and every chunk costs
  // two dependent memory round trips (child entry -> record); only the fields the ranking needs are kept
  struct Slim { int token, n_child; double fo; float fi; };
  for (int base = 0; base < C; base += NT * U) {
    int cid[U];
    Slim cn[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = base + u * NT + tid;
      cid[u] = -1;
      if (i < C) { if (p.cap == 0) cid[u] = p.child; else { cid[u] = __ldg(&D.edges[p.child + i].y); ++ne; } }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (cid[u] >= 0) {
        const Node full = load_node<true>(D.nodes + cid[u]);
        cn[u].token = full.token; cn[u].n_child = full.n_child; cn[u].fo = full.fo;
        cn[u].fi = idx == 0 ? full.fi : __ldg(&D.fi_extra[(long long)(idx - 1) * D.node_cap + cid[u]]);
        ++nv;
      }
    // One pool round over the chunks [u_lo, u_hi): survivors of the threshold filter join the running top list, the
    // first K in (key desc, insertion index asc) order stay.  All U chunks go through one round (a hot node's frame
    // is mostly children below the thresholds); if their survivors do not fit the pool the chunks are redone one by
    // one (a chunk cannot overflow).  Selecting the top K of a union in pieces gives the same list.
    auto round = [&](int u_lo, int u_hi) -> bool {
      if (tid == 0) { S->pool_n = m; S->pool_ovf = 0; }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (u < u_lo || u >= u_hi || cid[u] < 0) continue;
        const int i = base + u * NT + tid;
        const Slim &c = cn[u];
        const double fi = (double)c.fi, fo = c.fo;
        const double fm = mix_freq(omw, w, fi, fo);
        bool skip;
        if (mode == PIA_MODE_MIX) skip = (fi < min_in && fo < min_out && fm < min_mix);
        else if (mode == PIA_MODE_INPUT) skip = fi < min_in;
        else skip = fo < min_out;
        // once K candidates are held, a later child (larger insertion index) only displaces one of them with a
        // strictly larger key: ties go to the earlier child (:254-258)
        if (!skip && m >= K && K > 0 && dbits(fm) <= S->pkey[K - 1]) skip = true;
        if (!skip && K <= 0) skip = true;
        if (!skip) {
          const int slot = atomicAdd(&S->pool_n, 1);
          if (slot < MAXS + NT) {
            S->pkey[slot] = dbits(fm);
            S->pord[slot] = i;
            S->pnode[slot] = cid[u];
            S->ptok[slot] = c.token;
            S->pflag[slot] = (fi > 0.0 ? CF_FI : 0) | (fo > 0.0 ? CF_FO : 0) | (c.n_child > 0 ? CF_KIDS : 0);
          } else {
            S->pool_ovf = 1;
          }
        }
      }
      __syncthreads();
      if (S->pool_ovf) { __syncthreads(); return false; }  // uniform; the held list [0, m) is untouched
      const int total = S->pool_n;
      if (total == m) return true;  // nothing new (uniform): the running list stands
      // rank every pool element; the first K in (key desc, ord asc) order survive
      for (int e = tid; e < total; e += NT) {
        const unsigned long long k = S->pkey[e];
        const int o = S->pord[e];
        int rank = 0;
        for (int j = 0; j < total; ++j) {
          const unsigned long long kj = S->pkey[j];
          rank += (kj > k) || (kj == k && S->pord[j] < o);
        }
        if (rank < K) {
          S->qkey[rank] = k; S->qord[rank] = o; S->qnode[rank] = S->pnode[e]; S->qtok[rank] = S->ptok[e];
          S->qflag[rank] = S->pflag[e];
        }
      }
      __syncthreads();
      m = total < K ? total : K;
      for (int e = tid; e < m; e += NT) {
        S->pkey[e] = S->qkey[e]; S->pord[e] = S->qord[e]; S->pnode[e] = S->qnode[e]; S->ptok[e] = S->qtok[e];
        S->pflag[e] = S->qflag[e];
      }
      __syncthreads();
      return true;
    };
    if (!round(0, U)) {
      for (int u = 0; u < U && base + u * NT < C; ++u) round(u, u + 1);
    }
  }
  for (int e = tid; e < m; e += NT) { onode[e] = S->pnode[e]; otok[e] = S->ptok[e]; oflag[e] = (unsigned char)S->pflag[e]; }
  __syncthreads();
#ifdef PIA_TRIE_PHASES
#ifdef PIA_TRIE_PHASES_FRAMES
  if (tid == 0) printf("  frame: C %d K %d kept %d  %llu ns\n", C, K, m, gtime() - tf0);
#endif
#endif
  return m;
}

// narrow nodes (the common case) take the 2-chunk instance: its registers stay registers; wide nodes the 8-chunk one
template <int MAXS, int MAXD>
__device__ __forceinline__ int build_frame(const Dev &D, GetSmem<MAXS, MAXD> *S, int parent, int K, int idx, int mode, double omw,
                           double w, double min_in, double min_out, double min_mix, int *onode, int *otok,
                           unsigned char *oflag, unsigned long long &nv, unsigned long long &ne) {
  const Node p = load_node<true>(D.nodes + parent);
  if (p.n_child <= 2 * NT)
    return build_frame_u<MAXS, MAXD, 2>(D, S, p, K, idx, mode, omw, w, min_in, min_out, min_mix, onode, otok, oflag, nv, ne);
  return build_frame_u<MAXS, MAXD, 8>(D, S, p, K, idx, mode, omw, w, min_in, min_out, min_mix, onode, otok, oflag, nv, ne);
}

// Tree.get (lookahead_cache.py:65-144) for the tree rooted at `root`, query suffix q[0..nq).
// Result is left in S->ids / S->mask / S->n / S->sizes*.  returns PIA_OK / PIA_ERR_INDEX / PIA_ERR_CAPACITY.
template <int MAXS, int MAXD>
__device__ __forceinline__ int tree_get(const Dev &D, GetSmem<MAXS, MAXD> *S, int root, int tree_token, const int *q, int nq,
                        int max_size, int max_length, int min_in_sz, int min_out_sz, int mode, int idx, int *fr0,
                        int *fr1, int CL, int rank, int prune, unsigned long long &nv, unsigned long long &ne) {
  const int tid = threadIdx.x;
  constexpr int W = (MAXS + 63) / 64;
  // CL > 1: the CTAs of a cluster share the frequency walk below the match (everything up to the merge is executed by
  // every rank with identical control flow); thresholds and _ravel are the leader's
  GetSmem<MAXS, MAXD> *L = CL > 1 ? map_to_rank(S, 0) : S;
#ifdef PIA_TRIE_PHASES
  unsigned long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#endif
  PHASE(0);
  // ---- _match (:224-246), one warp
  if (tid < 32) {
    int cur = root;
    for (int j = 0; j < nq && cur >= 0; ++j) {
      const Node pn = D.nodes[cur];
      const int c = find_child(D, pn, q[j]);
      if (c < 0) { cur = -1; break; }
      const Node cn = D.nodes[c];
      const float fi = load_fi(D, cn, c, idx);
      bool live;
      if (mode == PIA_MODE_INPUT) live = fi > 0.f;
      else if (mode == PIA_MODE_OUTPUT) live = cn.fo > 0.0;
      else live = fi > 0.f || cn.fo > 0.0;
      cur = live ? c : -1;
    }
    if (cur >= 0 && D.nodes[cur].n_child == 0) cur = -1;  // len(nodes) == 0 (:70)
    if (tid == 0) {
      S->match_node = cur;
      S->sizes0 = 0; S->sizes1 = 0;
      S->hist_ovf = 0; S->n_live = 0; S->n_in = 0; S->n_out = 0; S->thr_found = 0; S->t_in = 0; S->t_out = 0;
    }
  }
  for (int s = tid; s < HCAP; s += NT) { S->hin.key[s] = HEMPTY; S->hin.cnt[s] = 0; S->hout.key[s] = HEMPTY; S->hout.cnt[s] = 0; }
  __syncthreads();
  PHASE(1);
  const int start = S->match_node;
  if (start < 0) {  // miss: ([last query token or tree token], ones(1,1), [0,0])  (:70-72)
    if (tid == 0) {
      S->ids[0] = nq > 0 ? q[nq - 1] : tree_token;
      for (int w = 0; w < W; ++w) S->mask[0][w] = 0;
      S->mask[0][0] = 1ull;
      S->n = 1;
    }
    __syncthreads();
    return PIA_OK;
  }
  // ---- _dfs_get_freqs (:146-154): every live node below the match, any order
  const bool need_in = (mode == PIA_MODE_INPUT) || (mode == PIA_MODE_MIX && min_in_sz > 0);
  const bool need_out = (mode == PIA_MODE_OUTPUT) || (mode == PIA_MODE_MIX && min_out_sz > 0);
  // Pruned walk.  The reference lists the frequencies of EVERY live node below the match and takes the k-th largest
  // fi / fo as thresholds when there are more than max_size of them (:74-125).  Counts only ever grow along root
  // paths (_put :40-56 adds `freq` to every node of the path, _squeeze :302-310 halves top-down and drops whole
  // subtrees, _reset_input_freq :326-333 zeroes top-down), so a node's fi and fo bound those of its descendants.  Once
  // more than max_size live nodes have been seen (the `size > max_size` decision is then made) a subtree below a
  // node with fo <= the running k-th largest fo (and fi likewise) cannot change the k-th largest value: it is not
  // entered.  The running thresholds are recomputed after every level from the nodes seen so far (a subset, hence a
  // lower bound of the final value).  A hot match (137 k nodes below a frequent bigram) visits the first level and a
  // few hundred nodes instead of all of them; the thresholds, hence the draft, are bit-identical.  Not applicable
  // (full walk) when an index is python-negative (k == 0 -> rank N) or beyond max_size, when the forest was imported
  // with a violated bound (pia_trie_import checks), or in cluster mode.
  const bool may_prune = prune && CL == 1 && (!need_in || (min_in_sz >= 1 && min_in_sz <= max_size)) &&
                         (!need_out || (min_out_sz >= 1 && min_out_sz <= max_size));
  unsigned long long t_in = 0, t_out = 0;  // running thresholds of the pruned walk: lower bounds of the final ones
  {
    long long my_live = 0, my_in = 0, my_out = 0;
    bool pruning = false;
    // called convergently by all lanes of a warp; equal values of a warp reach the shared histogram as one update
    // (n-gram counts are overwhelmingly 1.0: one contended address otherwise).  While pruning, values at or below the
    // running threshold are not recorded at all: they cannot change the k-th largest value.
    auto visit = [&](int id, const Node &nd, bool valid) -> bool {
      float fi = 0.f;
      double fo = 0.0;
      if (valid) { fi = load_fi(D, nd, id, idx); fo = nd.fo; }
      const bool live = valid && (fo > 0.0 || fi > 0.f);
      const unsigned long long bi = dbits((double)fi), bo = dbits(fo);
      if (!pruning) { my_live += live; my_in += live && fi > 0.f; my_out += live && fo > 0.0; }
      if (need_in) warp_hist_add(&S->hin, bi, live && (!pruning || bi > t_in), &S->hist_ovf);
      if (need_out) warp_hist_add(&S->hout, bo, live && (!pruning || bo > t_out), &S->hist_ovf);
      if (!live) return false;
      if (pruning) return (need_in && bi > t_in) || (need_out && bo > t_out);
      return true;
    };
    long long pushed = 0;  // nodes handed to the walk so far (uniform): an upper bound of the live nodes seen
    auto level_end = [&](int next_cnt) {
      pushed += next_cnt;
      // nothing to decide while fewer than max_size nodes were reached at all; once pruning is on, the thresholds are
      // only tightened ahead of a large level (a stale threshold is a valid, lower, bound)
      if (!may_prune || pushed <= max_size || (pruning && next_cnt < 2 * NT)) return;
      for (int o = 16; o > 0; o >>= 1) {
        my_live += __shfl_down_sync(FULL, my_live, o); my_in += __shfl_down_sync(FULL, my_in, o);
        my_out += __shfl_down_sync(FULL, my_out, o);
      }
      if (lane_id() == 0 && my_live) { atomicAdd((unsigned long long *)&S->n_live, (unsigned long long)my_live);
                                       atomicAdd((unsigned long long *)&S->n_in, (unsigned long long)my_in);
                                       atomicAdd((unsigned long long *)&S->n_out, (unsigned long long)my_out); }
      my_live = 0; my_in = 0; my_out = 0;
      __syncthreads();
      const long long seen = mode == PIA_MODE_INPUT ? S->n_in : (mode == PIA_MODE_OUTPUT ? S->n_out : S->n_live);
      if (seen <= max_size || S->hist_ovf) return;  // uniform
      if (need_in && kth_value(S, &S->hin, min_in_sz, t_in)) t_in = S->thr_bits;
      if (need_out && kth_value(S, &S->hout, min_out_sz, t_out)) t_out = S->thr_bits;
      pruning = true;
    };
    if (CL > 1) cluster_sync_all();  // the leader's counters / histograms are initialised before any remote access
    PHASE(2);
    bfs_below<true>(D, start, fr0, fr1, CL > 1 ? nullptr : S->sfr, &S->xt, &L->bfs, CL, rank, visit, level_end, nv, ne);
    PHASE(3);
    if (my_live) { atomicAdd((unsigned long long *)&L->n_live, (unsigned long long)my_live);
                   atomicAdd((unsigned long long *)&L->n_in, (unsigned long long)my_in);
                   atomicAdd((unsigned long long *)&L->n_out, (unsigned long long)my_out); }
    __syncthreads();
    if (CL > 1) {  // followers fold their histograms into the leader's (distributed-shared-memory atomics)
      if (rank != 0) {
        for (int e = tid; e < HCAP; e += NT) {
          if (need_in && S->hin.key[e] != HEMPTY) hist_add(&L->hin, S->hin.key[e], S->hin.cnt[e], &L->hist_ovf);
          if (need_out && S->hout.key[e] != HEMPTY) hist_add(&L->hout, S->hout.key[e], S->hout.cnt[e], &L->hist_ovf);
        }
        if (tid == 0 && S->hist_ovf) L->hist_ovf = 1;
      }
      cluster_sync_all();
      if (rank != 0) return PIA_OK;
    }
  }
  PHASE(4);
  if (S->bfs.err) return PIA_ERR_CAPACITY;
  // ---- thresholds (:78-125)
  double min_in = 1e9, min_out = 1e9, min_mix = 1e9, w = 1e-4;
  const long long N = S->n_live;
  long long size;
  if (mode == PIA_MODE_INPUT) { w = 0.0; size = S->n_in; }
  else if (mode == PIA_MODE_OUTPUT) { w = 1.0; size = S->n_out; }
  else size = N;
  if (size > max_size) {
    if (S->hist_ovf) return PIA_ERR_CAPACITY;
    // python index k-1 with negative wrap: k == 0 -> the smallest value (rank N)
    if (need_in) {
      if (!kth_value(S, &S->hin, min_in_sz >= 1 ? min_in_sz : N, t_in)) return PIA_ERR_INDEX;
      min_in = __longlong_as_double((long long)S->thr_bits);
    }
    if (need_out) {
      if (!kth_value(S, &S->hout, min_out_sz >= 1 ? min_out_sz : N, t_out)) return PIA_ERR_INDEX;
      min_out = __longlong_as_double((long long)S->thr_bits);
    }
    // mix mode: the reference's refinement loop never lowers min_mix_freq (every record carries None in
    // slot 0, :100-123), so it stays 1e9
  } else {
    if (mode == PIA_MODE_INPUT) min_in = 0.0;
    else if (mode == PIA_MODE_OUTPUT) min_out = 0.0;
    else min_mix = 0.0;
  }
  PHASE(5);
  const double omw = __dsub_rn(1.0, w);
  // ---- _ravel (:248-293): DFS pre-order, iterative with one sorted frame per depth
  if (tid == 0) {
    const int mt = nq > 0 ? q[nq - 1] : 0;
    S->ids[0] = (nq > 0 && mt != 0) ? mt : tree_token;  // `match_token_id or self.token_id` (:129)
    for (int w2 = 0; w2 < W; ++w2) S->mask[0][w2] = 0;
    S->mask[0][0] = 1ull;
    S->n = 1;
    S->depth = -1;
  }
  __syncthreads();
  if (max_size > 1 && max_length > 0) {
    int cnt0 = build_frame(D, S, start, max_size - 1, idx, mode, omw, w, min_in, min_out, min_mix, S->fnode[0],
                           S->ftok[0], S->fflag[0], nv, ne);
    if (tid == 0) { S->fcnt[0] = cnt0; S->fcur[0] = 0; S->fpid[0] = -1; S->depth = 0; }
    PHASE(6);
    __syncthreads();
    while (true) {
      // thread 0 advances the DFS until a sorted frame must be built (state 1) or the walk ends (state 0).
      // Single-child nodes (n-gram chains, the common case below the first levels) are followed inline by thread 0:
      // one dependent record load per node instead of a CTA-wide frame construction.
      if (tid == 0) {
        int st = 0;
        while (S->depth >= 0 && S->n < max_size && st == 0) {
          const int d = S->depth;
          if (S->fcur[d] >= S->fcnt[d]) { S->depth = d - 1; continue; }
          const int e = S->fcur[d]++;
          int rid = S->n;
          S->ids[rid] = S->ftok[d][e];
          int fl = S->fflag[d][e];
          S->sizes0 += (fl & CF_FI) ? 1 : 0;
          S->sizes1 += (fl & CF_FO) ? 1 : 0;
          const int pid = S->fpid[d];
          for (int w2 = 0; w2 < W; ++w2) S->mask[rid][w2] = pid >= 0 ? S->mask[pid][w2] : (w2 == 0 ? 1ull : 0ull);
          S->mask[rid][rid >> 6] |= 1ull << (rid & 63);
          S->n = rid + 1;
          // recurse (:283-293): children exist, depth budget max_length-1-d > 0, room left
          int cur_node = S->fnode[d][e], cur_d = d;
          Node x;
          bool have_x = false;  // the record of cur_node is already in registers (it was the child of the last step)
          while ((fl & CF_KIDS) && (max_length - 1 - cur_d) > 0 && S->n < max_size && cur_d + 1 < MAXD) {
            if (!have_x) { x = load_node<true>(D.nodes + cur_node); ++nv; }
            if (x.n_child != 1) {  // several children: they must be ranked by fm -> build a frame
              S->best_node = cur_node;
              S->fpid[cur_d + 1] = rid;
              S->depth = cur_d;
              st = 1;
              break;
            }
            int cid;
            if (x.cap == 0) cid = x.child; else { cid = __ldg(&D.edges[x.child].y); ++ne; }
            const Node c = load_node<true>(D.nodes + cid);
            ++nv;
            const double fi = (double)load_fi(D, c, cid, idx), fo = c.fo;
            const double fm = mix_freq(omw, w, fi, fo);
            bool skip;
            if (mode == PIA_MODE_MIX) skip = (fi < min_in && fo < min_out && fm < min_mix);
            else if (mode == PIA_MODE_INPUT) skip = fi < min_in;
            else skip = fo < min_out;
            // an (already exhausted) frame at this depth keeps the unwinding uniform
            S->fcnt[cur_d + 1] = 0; S->fcur[cur_d + 1] = 0; S->fpid[cur_d + 1] = rid; S->depth = cur_d + 1;
            if (skip) break;
            const int prid = rid;
            rid = S->n;
            S->ids[rid] = c.token;
            S->sizes0 += fi > 0.0 ? 1 : 0;
            S->sizes1 += fo > 0.0 ? 1 : 0;
            for (int w2 = 0; w2 < W; ++w2) S->mask[rid][w2] = S->mask[prid][w2];
            S->mask[rid][rid >> 6] |= 1ull << (rid & 63);
            S->n = rid + 1;
            fl = c.n_child > 0 ? CF_KIDS : 0;
            cur_node = cid;
            cur_d = cur_d + 1;
            x = c; have_x = true;
          }
        }
        S->state = st;
      }
      __syncthreads();
      if (S->state == 0) break;
      const int d1 = S->depth + 1;
      const int cnt = build_frame(D, S, S->best_node, max_size - S->n, idx, mode, omw, w, min_in, min_out, min_mix,
                                  S->fnode[d1], S->ftok[d1], S->fflag[d1], nv, ne);
      if (tid == 0) { S->fcnt[d1] = cnt; S->fcur[d1] = 0; S->depth = d1; }
      __syncthreads();
    }
  }
  __syncthreads();
#ifdef PIA_TRIE_PHASES
  PHASE(7);
  if (tid == 0 && rank == 0)
    printf("tree_get phases ns: match %llu sync %llu bfs %llu merge %llu thr %llu frame0 %llu ravel %llu | n_live %lld n %d\n",
           ph[1] - ph[0], ph[2] - ph[1], ph[3] - ph[2], ph[4] - ph[3], ph[5] - ph[4], ph[6] - ph[5], ph[7] - ph[6],
           S->n_live, S->n);
#endif
  return PIA_OK;
}

// Tree.get_one_branch (lookahead_cache.py:171-222): greedy single chain
template <int MAXS, int MAXD>
__device__ int tree_get_one(const Dev &D, GetSmem<MAXS, MAXD> *S, int root, int tree_token, const int *q, int nq,
                            int max_length, int mode, int idx, int *miss, unsigned long long &nv,
                            unsigned long long &ne) {
  const int tid = threadIdx.x;
  if (tid < 32) {
    int cur = root;
    for (int j = 0; j < nq && cur >= 0; ++j) {
      const Node pn = D.nodes[cur];
      const int c = find_child(D, pn, q[j]);
      if (c < 0) { cur = -1; break; }
      const Node cn = D.nodes[c];
      const float fi = load_fi(D, cn, c, idx);
      bool live;
      if (mode == PIA_MODE_INPUT) live = fi > 0.f;
      else if (mode == PIA_MODE_OUTPUT) live = cn.fo > 0.0;
      else live = fi > 0.f || cn.fo > 0.0;
      cur = live ? c : -1;
    }
    if (cur >= 0 && D.nodes[cur].n_child == 0) cur = -1;
    if (tid == 0) S->match_node = cur;
  }
  __syncthreads();
  int cur = S->match_node;
  if (cur < 0) {
    if (tid == 0) { S->ids[0] = nq > 0 ? q[nq - 1] : tree_token; S->n = 1; }
    *miss = 1;
    __syncthreads();
    return PIA_OK;
  }
  *miss = 0;
  if (tid == 0) {
    const int mt = nq > 0 ? q[nq - 1] : 0;
    S->ids[0] = (nq > 0 && mt != 0) ? mt : tree_token;
    S->n = 1;
  }
  __syncthreads();
  for (int length = 0; length < max_length; ++length) {
    const Node p = D.nodes[cur];
    if (p.n_child == 0) break;
    if (tid == 0) { S->best_node = -1; S->best_key = 0; S->best_ord = 0x7fffffff; }
    __syncthreads();
    // argmax of freq over the children, strict '>' keeps the earliest child on ties, freq must be > 0
    for (int base = 0; base < p.n_child; base += NT) {
      const int i = base + tid;
      if (i < p.n_child) {
        int cid;
        if (p.cap == 0) cid = p.child; else { cid = D.edges[p.child + i].y; ++ne; }
        const Node c = D.nodes[cid];
        ++nv;
        const double a = (double)load_fi(D, c, cid, idx), b = c.fo;
        double freq; bool ok;
        if (mode == PIA_MODE_MIX) { ok = a > 0 || b > 0; freq = __dadd_rn(__dmul_rn(10000.0, b), a); }
        else if (mode == PIA_MODE_INPUT) { freq = a; ok = a > 0; }
        else { freq = b; ok = b > 0; }
        if (ok && freq > 0.0) {
          const unsigned long long k = dbits(freq);
          atomicMax(&S->best_key, k);
        }
      }
    }
    __syncthreads();
    const unsigned long long bk = S->best_key;
    if (bk == 0) break;
    for (int base = 0; base < p.n_child; base += NT) {
      const int i = base + tid;
      if (i < p.n_child) {
        int cid = p.cap == 0 ? p.child : D.edges[p.child + i].y;
        const Node c = D.nodes[cid];
        const double a = (double)load_fi(D, c, cid, idx), b = c.fo;
        double freq; bool ok;
        if (mode == PIA_MODE_MIX) { ok = a > 0 || b > 0; freq = __dadd_rn(__dmul_rn(10000.0, b), a); }
        else if (mode == PIA_MODE_INPUT) { freq = a; ok = a > 0; }
        else { freq = b; ok = b > 0; }
        if (ok && dbits(freq) == bk) atomicMin(&S->best_ord, i);
      }
    }
    __syncthreads();
    const int bo = S->best_ord;
    const int cid = p.cap == 0 ? p.child : D.edges[p.child + bo].y;
    if (tid == 0) { S->ids[S->n] = D.nodes[cid].token; S->n += 1; }
    cur = cid;
    __syncthreads();
  }
  __syncthreads();
  return PIA_OK;
}

// LookaheadCache.hier_get / one_get (lookahead_cache.py:408-439, 490-517): one CTA per query row
#ifndef PIA_GET_MINB
#define PIA_GET_MINB 2  // resident CTAs per SM the register budget is sized for (128 registers: no spills in the walk)
#endif
template <int MAXS, int MAXD>
__global__ void __launch_bounds__(NT, PIA_GET_MINB) k_get(Dev D, GetParams P) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  GetSmem<MAXS, MAXD> *S = reinterpret_cast<GetSmem<MAXS, MAXD> *>(smem_raw);
  constexpr int W = (MAXS + 63) / 64;
  const int tid = threadIdx.x;
  // a hier_get of few rows is launched as one thread-block cluster per row (the frequency walk below a hot match is
  // shared by its CTAs); rank 0 leads and owns the row's outputs
  const int CL = (int)cluster_size(), rank = (int)cluster_rank();
  int *fr0 = D.frontier + (long long)(blockIdx.x / CL) * 2 * D.fr_cap;
  int *fr1 = fr0 + D.fr_cap;
  unsigned long long nv = 0, ne = 0;
  const int Wout = (P.dl + 63) / 64;
  // rows are handed out by a ticket counter when there are more rows than CTAs (a batched scan: query cost varies by
  // three orders of magnitude with the matched subtree, a static stride leaves SMs idle behind the hot rows)
  const bool dynamic = CL == 1 && P.batch > (int)gridDim.x;
  for (int b = blockIdx.x / CL;; ) {
    if (dynamic) {
      __syncthreads();
      if (tid == 0) S->ticket = atomicAdd(&D.hdr->get_ticket, 1);
      __syncthreads();
      b = S->ticket;
    }
    if (b >= P.batch) break;
    __syncthreads();
    const int len = P.qlen[b];
    int nq, bl = P.bl;
    const int *qsrc;
    if (P.flags & PIA_GET_TAIL) {
      nq = len < P.max_query ? len : P.max_query;
      qsrc = P.queries + (long long)b * P.q_stride + (len - nq);
      const int max_seq = P.d_max_seq ? *P.d_max_seq : P.max_seq;
      if (max_seq > 0) { int lim = max_seq - len - 1; if (lim < 0) lim = 0; if (bl > lim) bl = lim; }
    } else {
      nq = len < P.q_stride ? len : P.q_stride;
      qsrc = P.queries + (long long)b * P.q_stride;
    }
    if (nq > 16) { qsrc += nq - 16; nq = 16; }
    if (nq < 0) nq = 0;
    if (tid < nq) S->q[tid] = qsrc[tid];
    if (tid == 0) { S->bfs.err = 0; }
    __syncthreads();
    const int idx = P.d_idx ? P.d_idx[b] : P.idx;
    int status = PIA_OK, n_out = 0, nsizes = 2, sz0 = 0, sz1 = 0;
    bool have = false;
    if (P.dl <= 1 || bl == 0) {  // (:413-414, :495-496)
      nsizes = 0;
    } else {
      const int n_iter = (P.flags & PIA_GET_FIRST_ONLY) ? (nq < 1 ? nq : 1) : nq;
      for (int i = 0; i < n_iter; ++i) {
        const int t = S->q[i];
        if (t < 0 || t >= D.vocab) continue;
        const int root = D.root_of[t];
        if (root < 0) continue;
        const int rest = nq - (i + 1);
        if (rest == 0 && is_stop(D, t)) continue;  // (:422-423)
        int rc, miss = 0;
        if (P.kind == PIA_GET_ONE) rc = tree_get_one<MAXS, MAXD>(D, S, root, t, S->q + i + 1, rest, bl, P.mode, idx, &miss, nv, ne);
        else rc = tree_get<MAXS, MAXD>(D, S, root, t, S->q + i + 1, rest, P.dl, bl, P.min_in, P.min_out, P.mode, idx, fr0, fr1, CL, rank, P.prune, nv, ne);
        int n_res = S->n;
        if (CL > 1) {  // the loop below must take the same turns in every CTA of the cluster: the leader's result decides
          if (rank == 0 && tid == 0) { S->pub_rc = rc; S->pub_n = S->n; }
          cluster_sync_all();
          const GetSmem<MAXS, MAXD> *L = map_to_rank(S, 0);
          rc = L->pub_rc; n_res = L->pub_n;
          cluster_sync_all();
        }
        if (rc != PIA_OK) { status = rc; break; }
        have = true;
        n_out = n_res;
        if (P.kind == PIA_GET_ONE) { if (miss) { nsizes = 2; sz0 = sz1 = 0; } else { nsizes = 1; sz0 = n_out - 1; sz1 = 0; } }
        else { nsizes = 2; sz0 = S->sizes0; sz1 = S->sizes1; }
        if (P.kind == PIA_GET_ONE ? (n_out >= bl / 2) : (n_out >= bl)) break;  // (:433-434, :512)
        __syncthreads();
      }
    }
    __syncthreads();
    int *oid = P.out_ids + (long long)b * P.dl;
    unsigned long long *om = P.out_mask + (long long)b * P.dl * Wout;
    if (rank != 0) break;  // followers of a cluster: one row, no outputs
    if (status == PIA_OK && have) {
      for (int i = tid; i < n_out; i += NT) {
        oid[i] = S->ids[i];
        if (P.kind == PIA_GET_ONE) {  // lower-triangular mask (:222)
          for (int w = 0; w < Wout; ++w) {
            unsigned long long v = 0;
            if (i >= 64 * (w + 1) - 1) v = ~0ull; else if (i >= 64 * w) v = (i - 64 * w) == 63 ? ~0ull : ((1ull << (i - 64 * w + 1)) - 1);
            om[(long long)i * Wout + w] = v;
          }
        } else {
          for (int w = 0; w < Wout; ++w) om[(long long)i * Wout + w] = w < W ? S->mask[i][w] : 0ull;
        }
      }
    } else if (status == PIA_OK) {  // token_ids[-1:], default mask (:414, :436-437)
      n_out = nq > 0 ? 1 : 0;
      if (tid == 0 && nq > 0) { oid[0] = S->q[nq - 1]; for (int w = 0; w < Wout; ++w) om[w] = w == 0 ? 1ull : 0ull; }
    } else {
      n_out = 0;
    }
    if (tid == 0) {
      P.out_n[b] = n_out;
      P.out_sizes[2 * b] = sz0; P.out_sizes[2 * b + 1] = sz1;
      P.out_nsizes[b] = nsizes;
      P.status[b] = status;
      if (status == PIA_ERR_CAPACITY) atomicOr(&D.hdr->err, S->hist_ovf ? ERR_HIST : ERR_FRONTIER);
    }
    if (!dynamic) break;  // one row per CTA
  }
  if (dynamic && tid == 0) {  // the last CTA to leave re-arms the ticket counter for the next launch
    __threadfence();
    if (atomicAdd(&D.hdr->get_done, 1) == (int)gridDim.x - 1) { D.hdr->get_ticket = 0; D.hdr->get_done = 0; __threadfence(); }
  }
  // roofline accounting: node records / child entries read
  for (int o = 16; o > 0; o >>= 1) { nv += __shfl_down_sync(FULL, nv, o); ne += __shfl_down_sync(FULL, ne, o); }
  if (lane_id() == 0) { if (nv) atomicAdd(&D.hdr->nodes_visited, nv); if (ne) atomicAdd(&D.hdr->edges_visited, ne); }
}

// ---------------------------------------------------------------------------------------------------
// reset_input_freqs (:320-333, :566-570)
// ---------------------------------------------------------------------------------------------------
// single_key >= 0: Tree.reset_input_freq(idx) of that one tree (:320-333), the touched-tree list is left alone
__global__ void __launch_bounds__(NT) k_reset_input(Dev D, int idx, int single_key) {
  __shared__ BfsShared sh;
  __shared__ ExpandTab xt;
  int *fr0 = D.frontier + (long long)blockIdx.x * 2 * D.fr_cap;
  int *fr1 = fr0 + D.fr_cap;
  unsigned long long nv = 0, ne = 0;
  const int n = single_key >= 0 ? 1 : D.hdr->n_updin;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const int key = single_key >= 0 ? single_key : D.updin_list[i];
    const int root = D.root_of[key];
    if (threadIdx.x == 0) { sh.err = 0; if (single_key < 0) D.tree_flags[key] &= ~FLAG_UPDIN; }
    __syncthreads();
    if (root < 0) continue;
    auto visit = [&](int id, const Node &nd, bool valid) -> bool {
      if (!valid) return false;
      const float f = load_fi(D, nd, id, idx);
      if (f == 0.f) return false;
      if (idx == 0) D.nodes[id].fi = 0.f; else D.fi_extra[(long long)(idx - 1) * D.node_cap + id] = 0.f;
      return true;
    };
    bfs_below<false>(D, root, fr0, fr1, nullptr, &xt, &sh, 1, 0, visit, [](int) {}, nv, ne);
    if (threadIdx.x == 0 && sh.err) atomicOr(&D.hdr->err, ERR_FRONTIER);
    __syncthreads();
  }
}
__global__ void k_reset_finish(Dev D) { D.hdr->n_updin = 0; }

// ---------------------------------------------------------------------------------------------------
// squeeze_branch_counts (:295-318, :572-576): one CTA per touched tree, one warp per surviving parent
// ---------------------------------------------------------------------------------------------------
// single_key >= 0: Tree.squeeze() of that one tree (:295-301), no 1024-trees threshold, lists left alone
__global__ void __launch_bounds__(NT) k_squeeze(Dev D, int single_key) {
  __shared__ int s_next, s_count, s_err;
  const int tid = threadIdx.x, lane = lane_id(), wid = warp_id();
  int *fr0 = D.frontier + (long long)blockIdx.x * 2 * D.fr_cap;
  int *fr1 = fr0 + D.fr_cap;
  const int n_listed = single_key >= 0 ? 1 : D.hdr->n_upd;
  if (single_key < 0 && n_listed + D.hdr->n_upd_stale < 1024) return;
  for (int i = blockIdx.x; i < n_listed; i += gridDim.x) {
    const int key = single_key >= 0 ? single_key : D.upd_list[i];
    const int root = D.root_of[key];
    __syncthreads();
    if (tid == 0) { s_next = 0; s_count = 0; s_err = 0; if (single_key < 0) D.tree_flags[key] &= ~FLAG_UPD; }
    __syncthreads();
    if (root < 0) continue;
    if (!(D.tree_n_node[key] > D.hdr->max_node || D.tree_n_out[key] > D.hdr->max_out)) continue;
    if (tid == 0) fr0[0] = root;
    __syncthreads();
    int cnt = 1;
    int *cur = fr0, *nxt = fr1;
    while (cnt > 0) {
      for (int e = wid; e < cnt; e += NT / 32) {
        const int pid = cur[e];
        const Node p = D.nodes[pid];
        if (p.cap == 0) {
          if (p.n_child == 1 && lane == 0) {
            const int c = p.child;
            const double fo = D.nodes[c].fo;
            if (fo > 1.0) {
              D.nodes[c].fo = fo * 0.5;
              atomicAdd(&s_count, 1);
              if (D.nodes[c].n_child > 0) { int pos = atomicAdd(&s_next, 1); if (pos < D.fr_cap) nxt[pos] = c; else s_err = 1; }
            } else {
              D.nodes[pid].n_child = 0; D.nodes[pid].child = -1;
            }
          }
        } else {
          int wr = 0;
          for (int base = 0; base < p.n_child; base += 32) {
            const int k = base + lane;
            int2 en = make_int2(-1, -1);
            bool keep = false; bool kids = false;
            if (k < p.n_child) {
              en = D.edges[p.child + k];
              const double fo = D.nodes[en.y].fo;
              keep = fo > 1.0;
              if (keep) { D.nodes[en.y].fo = fo * 0.5; kids = D.nodes[en.y].n_child > 0; }
            }
            const unsigned m = __ballot_sync(FULL, keep);
            const int off = __popc(m & ((1u << lane) - 1));
            __syncwarp();
            if (keep) D.edges[p.child + wr + off] = en;
            const unsigned mk = __ballot_sync(FULL, kids);
            int nb = 0;
            if (lane == 0 && mk) nb = atomicAdd(&s_next, __popc(mk));
            nb = __shfl_sync(FULL, nb, 0);
            if (kids) { int pos = nb + __popc(mk & ((1u << lane) - 1)); if (pos < D.fr_cap) nxt[pos] = en.y; else s_err = 1; }
            wr += __popc(m);
          }
          if (lane == 0) { D.nodes[pid].n_child = wr; atomicAdd(&s_count, wr); }
        }
      }
      __syncthreads();
      cnt = s_next;
      if (cnt > D.fr_cap) cnt = 0;
      __syncthreads();
      if (tid == 0) s_next = 0;
      __syncthreads();
      int *t = cur; cur = nxt; nxt = t;
    }
    if (tid == 0) {
      D.tree_n_node[key] = s_count; D.tree_n_out[key] = s_count;  // (:298-301)
      if (s_err) atomicOr(&D.hdr->err, ERR_FRONTIER);
    }
  }
}
__global__ void k_squeeze_finish(Dev D) {
  if (D.hdr->n_upd + D.hdr->n_upd_stale >= 1024) { D.hdr->n_upd = 0; D.hdr->n_upd_stale = 0; }
}

// fresh(): mem = {} (:563-564).  Trees pending in the update sets keep counting towards the 1024 threshold
// exactly as the orphaned Python objects do, but their storage is reclaimed.
__global__ void __launch_bounds__(NT) k_fresh(Dev D) {
  const int gid = blockIdx.x * NT + threadIdx.x;
  const int stride = gridDim.x * NT;
  for (int t = gid; t < D.vocab; t += stride) { D.root_of[t] = -1; D.tree_flags[t] = 0; D.tree_n_node[t] = 0; D.tree_n_out[t] = 0; }
}
__global__ void k_fresh_finish(Dev D) {
  Hdr *h = D.hdr;
  h->n_upd_stale += h->n_upd; h->n_upd = 0;
  h->n_updin = 0;  // resetting orphaned trees is unobservable
  h->node_top = 0; h->edge_top = 0; h->n_trees = 0;
}

}  // namespace trie
}  // namespace pia

// =====================================================================================================
// host side / C ABI
// =====================================================================================================
using namespace pia;
using namespace pia::trie;

struct pia_trie {
  Dev dev;
  pia_trie_config_t cfg;
  std::vector<void *> allocs;
  int n_sm;
  int get_cluster;  // CTAs per row of a small hier_get that cannot prune (PIA_TRIE_GET_CLUSTER, default 8; 1 = off)
  int prune;        // PIA_TRIE_PRUNE (default 1): pruned frequency walk (tree_get)
  int monotone;     // every node's fi / fo bound its children's: true for forests built by put, checked on import
};

template <class T>
static cudaError_t dalloc(pia_trie *t, T **p, size_t count, bool zero) {
  cudaError_t e = cudaMalloc((void **)p, count * sizeof(T));
  if (e != cudaSuccess) return e;
  t->allocs.push_back((void *)*p);
  if (zero) e = cudaMemset(*p, 0, count * sizeof(T));
  return e;
}

extern "C" int pia_trie_create(const pia_trie_config_t *c, pia_trie_t **out) {
  PIA_REQUIRE(c && out, "null argument");
  pia_trie_config_t cfg = *c;
  if (cfg.vocab_capacity <= 0) cfg.vocab_capacity = 65536;
  if (cfg.node_capacity <= 0) cfg.node_capacity = 1 << 24;
  if (cfg.edge_capacity <= 0) cfg.edge_capacity = cfg.node_capacity;
  if (cfg.n_input_slots <= 0) cfg.n_input_slots = 1;
  if (cfg.max_node <= 0) cfg.max_node = 65536;
  if (cfg.max_output_node <= 0) cfg.max_output_node = 512;
  if (cfg.max_put_tokens <= 0) cfg.max_put_tokens = 8192;
  if (cfg.frontier_capacity <= 0) cfg.frontier_capacity = 1 << 18;
  if (cfg.max_resident_queries <= 0) cfg.max_resident_queries = 296;
  PIA_REQUIRE(cfg.node_capacity < (1ll << 31) && cfg.edge_capacity < (1ll << 31), "pools are indexed with int32");
  pia_trie *t = new (std::nothrow) pia_trie();
  PIA_REQUIRE(t, "out of host memory");
  t->cfg = cfg;
  Dev &D = t->dev;
  memset(&D, 0, sizeof(D));
  cudaError_t e = cudaSuccess;
  auto ok = [&](cudaError_t x) { if (e == cudaSuccess) e = x; };
  ok(dalloc(t, &D.nodes, (size_t)cfg.node_capacity, false));
  ok(dalloc(t, &D.edges, (size_t)cfg.edge_capacity, false));
  if (cfg.n_input_slots > 1) ok(dalloc(t, &D.fi_extra, (size_t)(cfg.n_input_slots - 1) * cfg.node_capacity, false));
  ok(dalloc(t, &D.hdr, 1, true));
  ok(dalloc(t, &D.root_of, (size_t)cfg.vocab_capacity, false));
  ok(dalloc(t, &D.tree_n_node, (size_t)cfg.vocab_capacity, true));
  ok(dalloc(t, &D.tree_n_out, (size_t)cfg.vocab_capacity, true));
  ok(dalloc(t, &D.tree_flags, (size_t)cfg.vocab_capacity, true));
  ok(dalloc(t, &D.upd_list, (size_t)cfg.vocab_capacity, true));
  ok(dalloc(t, &D.updin_list, (size_t)cfg.vocab_capacity, true));
  ok(dalloc(t, &D.stop_bits, (size_t)(cfg.vocab_capacity + 31) / 32, true));
  D.out_cap = cfg.max_put_tokens + 128;
  ok(dalloc(t, &D.out_buf, (size_t)cfg.n_input_slots * D.out_cap, true));
  ok(dalloc(t, &D.out_len, (size_t)cfg.n_input_slots, true));
  ok(dalloc(t, &D.frontier, (size_t)cfg.max_resident_queries * 2 * cfg.frontier_capacity, false));
  if (e == cudaSuccess) e = cudaMemset(D.root_of, 0xff, sizeof(int) * (size_t)cfg.vocab_capacity);
  D.node_cap = cfg.node_capacity; D.edge_cap = cfg.edge_capacity; D.vocab = cfg.vocab_capacity;
  D.n_slots = cfg.n_input_slots; D.fr_cap = cfg.frontier_capacity; D.max_resident = cfg.max_resident_queries;
  if (e == cudaSuccess) {
    Hdr h; memset(&h, 0, sizeof(h));
    h.max_node = cfg.max_node; h.max_out = cfg.max_output_node; h.n_eos = 1; h.eos[0] = 2;
    e = cudaMemcpy(D.hdr, &h, sizeof(h), cudaMemcpyHostToDevice);
  }
  int dev_id = 0;
  if (e == cudaSuccess) e = cudaGetDevice(&dev_id);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&t->n_sm, cudaDevAttrMultiProcessorCount, dev_id);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_get<64, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GetSmem<64, 16>));
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_get<128, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GetSmem<128, 32>));
  {
    const char *ev = getenv("PIA_TRIE_GET_CLUSTER");
    int c = ev ? atoi(ev) : 8;
    t->get_cluster = (c == 2 || c == 4 || c == 8) ? c : 1;
    ev = getenv("PIA_TRIE_PRUNE");
    t->prune = ev ? atoi(ev) != 0 : 1;
    t->monotone = 1;
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error("pia_trie_create: %s", cudaGetErrorString(e));
    for (void *p : t->allocs) cudaFree(p);
    delete t;
    return PIA_ERR_CUDA;
  }
  *out = t;
  return PIA_OK;
}

extern "C" int pia_trie_destroy(pia_trie_t *t) {
  if (!t) return PIA_OK;
  cudaDeviceSynchronize();
  for (void *p : t->allocs) cudaFree(p);
  delete t;
  return PIA_OK;
}

extern "C" int pia_trie_set_eos(pia_trie_t *t, const int32_t *h_eos, int n) {
  PIA_REQUIRE(t && n >= 0 && n <= 8 && (n == 0 || h_eos), "eos: at most 8 ids");
  int buf[9]; buf[0] = n;
  for (int i = 0; i < 8; ++i) buf[1 + i] = i < n ? h_eos[i] : -1;
  PIA_CUDA_CHECK(cudaDeviceSynchronize());
  PIA_CUDA_CHECK(cudaMemcpy((char *)t->dev.hdr + offsetof(Hdr, n_eos), buf, sizeof(buf), cudaMemcpyHostToDevice));
  return PIA_OK;
}

extern "C" int pia_trie_set_stop_words(pia_trie_t *t, const int32_t *h_words, int n) {
  PIA_REQUIRE(t && n >= 0 && (n == 0 || h_words), "bad stop words");
  const size_t words = (size_t)(t->cfg.vocab_capacity + 31) / 32;
  std::vector<unsigned> bits(words, 0u);
  for (int i = 0; i < n; ++i) {
    PIA_REQUIRE(h_words[i] >= 0 && h_words[i] < t->cfg.vocab_capacity, "stop word %d outside vocab_capacity", h_words[i]);
    bits[h_words[i] >> 5] |= 1u << (h_words[i] & 31);
  }
  PIA_CUDA_CHECK(cudaDeviceSynchronize());
  PIA_CUDA_CHECK(cudaMemcpy(t->dev.stop_bits, bits.data(), words * sizeof(unsigned), cudaMemcpyHostToDevice));
  return PIA_OK;
}

extern "C" int pia_trie_set_limits(pia_trie_t *t, int max_node, int max_output_node) {
  PIA_REQUIRE(t, "null trie");
  int v[2] = {max_node, max_output_node};
  PIA_CUDA_CHECK(cudaDeviceSynchronize());
  PIA_CUDA_CHECK(cudaMemcpy((char *)t->dev.hdr + offsetof(Hdr, max_node), v, sizeof(v), cudaMemcpyHostToDevice));
  t->cfg.max_node = max_node; t->cfg.max_output_node = max_output_node;
  return PIA_OK;
}

static int launch_reset(pia_trie *t, int idx, cudaStream_t s) {
  const int grid = t->dev.max_resident < 4 * t->n_sm ? t->dev.max_resident : 4 * t->n_sm;
  k_reset_input<<<grid, NT, 0, s>>>(t->dev, idx, -1);
  PIA_LAUNCH_CHECK();
  k_reset_finish<<<1, 1, 0, s>>>(t->dev);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}
static int launch_squeeze(pia_trie *t, cudaStream_t s) {
  const int grid = t->dev.max_resident < 4 * t->n_sm ? t->dev.max_resident : 4 * t->n_sm;
  k_squeeze<<<grid, NT, 0, s>>>(t->dev, -1);
  PIA_LAUNCH_CHECK();
  k_squeeze_finish<<<1, 1, 0, s>>>(t->dev);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

static int put_common(pia_trie *t, const int32_t *d_tokens, int n, const int32_t *d_n, int B, int mode, int idx,
                      int final, int is_stream, cudaStream_t s, const int32_t *d_slot = nullptr) {
  PIA_REQUIRE(t, "null trie");
  PIA_REQUIRE(n >= 0 && n <= t->cfg.max_put_tokens, "token list of %d exceeds max_put_tokens=%d", n, t->cfg.max_put_tokens);
  PIA_REQUIRE(n == 0 || d_tokens, "null tokens");
  PIA_REQUIRE(B >= 1 && B <= 64, "branch_length %d outside [1,64]", B);
  PIA_REQUIRE(mode == PIA_MODE_INPUT || mode == PIA_MODE_OUTPUT, "put mode must be input or output");
  if (mode == PIA_MODE_INPUT) PIA_REQUIRE(idx >= 0 && idx < t->cfg.n_input_slots, "idx %d outside [0,%d)", idx, t->cfg.n_input_slots);
  const int slot = is_stream ? idx : 0;
  if (is_stream && !d_slot) PIA_REQUIRE(idx >= 0 && idx < t->cfg.n_input_slots, "stream idx %d outside [0,%d)", idx, t->cfg.n_input_slots);
  PIA_REQUIRE(!(d_slot && final), "a final stream_put needs the request idx on the host");
  k_put_prepare<<<1, NT, 0, s>>>(t->dev, d_tokens, n, d_n, B, is_stream, final, slot, d_slot);
  PIA_LAUNCH_CHECK();
  const int max_pos = is_stream ? n + 64 : n;
  if (max_pos > 0) {
    const int grid = (max_pos + (NT / 32) - 1) / (NT / 32);
    k_put_insert<<<grid, NT, 0, s>>>(t->dev, d_tokens, B, mode, idx, is_stream, slot, d_slot);
    PIA_LAUNCH_CHECK();
  }
  if (is_stream) {
    k_put_finish<<<1, 128, 0, s>>>(t->dev, B, final, slot, d_slot);
    PIA_LAUNCH_CHECK();
  }
  if (final) {
    int rc = launch_reset(t, idx < 0 ? 0 : idx, s);
    if (rc) return rc;
    rc = launch_squeeze(t, s);
    if (rc) return rc;
  }
  return PIA_OK;
}

extern "C" int pia_trie_put(pia_trie_t *t, const int32_t *d_tokens, int n, const int32_t *d_n, int branch_length,
                            int mode, int idx, int final, void *stream) {
  return put_common(t, d_tokens, n, d_n, branch_length, mode, idx, final, 0, (cudaStream_t)stream);
}
extern "C" int pia_trie_tree_put(pia_trie_t *t, int tree_token, const int32_t *d_tokens, int n, int mode, int idx,
                                 void *stream) {
  PIA_REQUIRE(t && tree_token >= 0 && tree_token < t->cfg.vocab_capacity, "bad tree token");
  PIA_REQUIRE(n >= 0 && (n == 0 || d_tokens), "bad tokens");
  PIA_REQUIRE(mode == PIA_MODE_INPUT || mode == PIA_MODE_OUTPUT, "put mode must be input or output");
  if (mode == PIA_MODE_INPUT) PIA_REQUIRE(idx >= 0 && idx < t->cfg.n_input_slots, "bad idx");
  k_tree_put<<<1, 32, 0, (cudaStream_t)stream>>>(t->dev, tree_token, d_tokens, n, mode, idx);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}
extern "C" int pia_trie_stream_put(pia_trie_t *t, const int32_t *d_tokens, int n, const int32_t *d_n,
                                   int branch_length, int idx, const int32_t *d_idx, int final, void *stream) {
  return put_common(t, d_tokens, n, d_n, branch_length, PIA_MODE_OUTPUT, idx, final, 1, (cudaStream_t)stream, d_idx);
}

extern "C" int pia_trie_get(pia_trie_t *t, const int32_t *d_queries, const int32_t *d_qlen, int batch, int q_stride,
                            int max_query_length, const int32_t *d_idx, int idx, int decoding_length,
                            int branch_length, int min_input_size, int min_output_size, int mode, int kind, int flags,
                            int max_seq_length, const int32_t *d_max_seq_length, int32_t *d_out_ids,
                            uint64_t *d_out_mask, int32_t *d_out_n, int32_t *d_out_sizes, int32_t *d_out_nsizes,
                            int32_t *d_status, void *stream) {
  PIA_REQUIRE(t, "null trie");
  PIA_REQUIRE(batch >= 1 && d_queries && d_qlen, "bad query batch");
  PIA_REQUIRE(decoding_length >= 1 && decoding_length <= 128, "decoding_length %d outside [1,128]", decoding_length);
  PIA_REQUIRE(branch_length >= 0 && branch_length <= 32, "branch_length %d outside [0,32]", branch_length);
  PIA_REQUIRE(mode >= 0 && mode <= 2 && (kind == PIA_GET_HIER || kind == PIA_GET_ONE), "bad mode/kind");
  PIA_REQUIRE(min_input_size >= 0 && min_output_size >= 0, "negative min sizes");
  PIA_REQUIRE(d_idx || (idx >= 0 && idx < t->cfg.n_input_slots), "idx %d outside [0,%d)", idx, t->cfg.n_input_slots);
  PIA_REQUIRE(d_out_ids && d_out_mask && d_out_n && d_out_sizes && d_out_nsizes && d_status, "null output");
  GetParams P;
  P.queries = d_queries; P.qlen = d_qlen; P.d_idx = d_idx; P.batch = batch; P.q_stride = q_stride;
  P.max_query = max_query_length > 0 ? max_query_length : q_stride; P.idx = idx; P.dl = decoding_length;
  P.bl = branch_length; P.min_in = min_input_size; P.min_out = min_output_size; P.mode = mode; P.kind = kind;
  P.flags = flags; P.max_seq = max_seq_length; P.d_max_seq = d_max_seq_length;
  P.out_ids = d_out_ids; P.out_mask = (unsigned long long *)d_out_mask; P.out_n = d_out_n; P.out_sizes = d_out_sizes;
  P.out_nsizes = d_out_nsizes; P.status = d_status;
  int grid = batch < t->dev.max_resident ? batch : t->dev.max_resident;
  cudaStream_t s = (cudaStream_t)stream;
  // The walk below the match is pruned (tree_get) whenever the forest's counts are known to be monotone along root
  // paths.  Otherwise, for few rows (the decode step: 1 row, the batched loop: <= 16), a cluster of GET_CLUSTER CTAs
  // per row shares the full walk; a batched scan keeps one CTA per row (rows are the parallelism there).
  P.prune = t->prune && t->monotone;
  int cl = 1;
  if (kind == PIA_GET_HIER && !P.prune && t->get_cluster > 1 && batch * t->get_cluster <= 128 &&
      batch * t->get_cluster <= t->dev.max_resident)
    cl = t->get_cluster;
  grid *= cl;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(NT); cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  // no programmatic-serialization attribute: the kernel has no griddepcontrol.wait; no cluster attribute either for the
  // ordinary one-CTA-per-row launch
  cfg.attrs = attr; cfg.numAttrs = cl > 1 ? 1 : 0;
  if (decoding_length <= 64 && branch_length <= 16) {
    cfg.dynamicSmemBytes = sizeof(GetSmem<64, 16>);
    PIA_CUDA_CHECK(cudaLaunchKernelEx(&cfg, k_get<64, 16>, t->dev, P));
  } else {
    cfg.dynamicSmemBytes = sizeof(GetSmem<128, 32>);
    PIA_CUDA_CHECK(cudaLaunchKernelEx(&cfg, k_get<128, 32>, t->dev, P));
  }
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

__global__ void k_copy_err(pia::trie::Dev D, int *out) { *out = D.hdr->err; }

extern "C" int pia_trie_copy_error_flags(pia_trie_t *t, int32_t *d_out, void *stream) {
  PIA_REQUIRE(t && d_out, "null argument");
  k_copy_err<<<1, 1, 0, (cudaStream_t)stream>>>(t->dev, d_out);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

// Tree.squeeze (:295-301) / Tree.reset_input_freq (:320-333) of the one tree keyed by `token`
extern "C" int pia_trie_tree_squeeze(pia_trie_t *t, int token, void *stream) {
  PIA_REQUIRE(t && token >= 0 && token < t->cfg.vocab_capacity, "bad tree token");
  k_squeeze<<<1, NT, 0, (cudaStream_t)stream>>>(t->dev, token);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}
extern "C" int pia_trie_tree_reset_input_freq(pia_trie_t *t, int token, int idx, void *stream) {
  PIA_REQUIRE(t && token >= 0 && token < t->cfg.vocab_capacity, "bad tree token");
  PIA_REQUIRE(idx >= 0 && idx < t->cfg.n_input_slots, "bad idx");
  k_reset_input<<<1, NT, 0, (cudaStream_t)stream>>>(t->dev, idx, token);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

extern "C" int pia_trie_reset_input_freqs(pia_trie_t *t, int idx, void *stream) {
  PIA_REQUIRE(t && idx >= 0 && idx < t->cfg.n_input_slots, "bad idx");
  return launch_reset(t, idx, (cudaStream_t)stream);
}
extern "C" int pia_trie_squeeze_branch_counts(pia_trie_t *t, void *stream) {
  PIA_REQUIRE(t, "null trie");
  return launch_squeeze(t, (cudaStream_t)stream);
}
extern "C" int pia_trie_fresh(pia_trie_t *t, void *stream) {
  PIA_REQUIRE(t, "null trie");
  cudaStream_t s = (cudaStream_t)stream;
  k_fresh<<<t->n_sm, NT, 0, s>>>(t->dev);
  PIA_LAUNCH_CHECK();
  k_fresh_finish<<<1, 1, 0, s>>>(t->dev);
  PIA_LAUNCH_CHECK();
  return PIA_OK;
}

extern "C" int pia_trie_stats(pia_trie_t *t, pia_trie_stats_t *o, void *stream) {
  PIA_REQUIRE(t && o, "null argument");
  Hdr h;
  PIA_CUDA_CHECK(cudaMemcpyAsync(&h, t->dev.hdr, sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  PIA_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  o->nodes_used = (int64_t)h.node_top; o->edges_used = (int64_t)h.edge_top; o->n_trees = h.n_trees;
  o->n_update_trees = h.n_upd + h.n_upd_stale; o->n_update_input_trees = h.n_updin; o->error_flags = h.err;
  o->nodes_visited = (int64_t)h.nodes_visited; o->edges_visited = (int64_t)h.edges_visited;
  return PIA_OK;
}

extern "C" int pia_trie_tree_counters(pia_trie_t *t, int token, int64_t *h_n_node, int64_t *h_n_output_node,
                                      void *stream) {
  PIA_REQUIRE(t && token >= 0 && token < t->cfg.vocab_capacity, "bad token");
  cudaStream_t s = (cudaStream_t)stream;
  int root = -1, a = 0, b = 0;
  PIA_CUDA_CHECK(cudaMemcpyAsync(&root, t->dev.root_of + token, sizeof(int), cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(&a, t->dev.tree_n_node + token, sizeof(int), cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(&b, t->dev.tree_n_out + token, sizeof(int), cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaStreamSynchronize(s));
  if (h_n_node) *h_n_node = root < 0 ? -1 : a;
  if (h_n_output_node) *h_n_output_node = root < 0 ? -1 : b;
  return PIA_OK;
}

// ---------------------------------------------------------------------------------------------------
// persistence (LookaheadCache.save_mem / load_mem, lookahead_cache.py:578-587): raw pools <-> host
// ---------------------------------------------------------------------------------------------------
extern "C" int pia_trie_export_sizes(pia_trie_t *t, int64_t *n_nodes, int64_t *n_edges, void *stream) {
  PIA_REQUIRE(t && n_nodes && n_edges, "null argument");
  Hdr h;
  PIA_CUDA_CHECK(cudaMemcpyAsync(&h, t->dev.hdr, sizeof(h), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  PIA_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  *n_nodes = (int64_t)h.node_top; *n_edges = (int64_t)h.edge_top;
  return PIA_OK;
}

extern "C" int pia_trie_export(pia_trie_t *t, void *h_nodes, int64_t n_nodes, void *h_edges, int64_t n_edges,
                               int32_t *h_root_of, int32_t *h_n_node, int32_t *h_n_out, void *stream) {
  PIA_REQUIRE(t && h_nodes && h_edges && h_root_of && h_n_node && h_n_out, "null argument");
  PIA_REQUIRE(n_nodes <= t->cfg.node_capacity && n_edges <= t->cfg.edge_capacity, "sizes exceed the pools");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t v = (size_t)t->cfg.vocab_capacity * sizeof(int);
  PIA_CUDA_CHECK(cudaMemcpyAsync(h_nodes, t->dev.nodes, (size_t)n_nodes * sizeof(Node), cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(h_edges, t->dev.edges, (size_t)n_edges * sizeof(int2), cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(h_root_of, t->dev.root_of, v, cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(h_n_node, t->dev.tree_n_node, v, cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(h_n_out, t->dev.tree_n_out, v, cudaMemcpyDeviceToHost, s));
  PIA_CUDA_CHECK(cudaStreamSynchronize(s));
  return PIA_OK;
}

// Storage reclamation.  The pools are bump allocators: squeeze unlinks subtrees (the reference pops them, :302-310, and
// Python frees them), grown child blocks are abandoned, and every request's input-mode prompt adds up to
// prompt_len * (branch_length + 1) nodes, so a long-running process would sooner or later exhaust a pool and stop
// learning.  pia_trie_compact copies the REACHABLE forest (host round trip: D2H, depth-first renumbering so that chains
// stay contiguous, child order kept, blocks trimmed to the next power of two >= 4, H2D) and resets the allocator tops.
// Nothing a query or an update can observe changes: same trees, children, order, counts, per-tree counters, touched-tree
// lists.  Synchronous; call it between requests (LookaheadCache.maybe_compact does, past a fill threshold).
extern "C" int pia_trie_compact(pia_trie_t *t, int64_t *h_nodes_before, int64_t *h_nodes_after, void *stream) {
  PIA_REQUIRE(t, "null trie");
  cudaStream_t s = (cudaStream_t)stream;
  PIA_CUDA_CHECK(cudaStreamSynchronize(s));
  Hdr h;
  PIA_CUDA_CHECK(cudaMemcpy(&h, t->dev.hdr, sizeof(h), cudaMemcpyDeviceToHost));
  const int64_t nn = (int64_t)(h.node_top < (unsigned long long)t->cfg.node_capacity ? h.node_top : t->cfg.node_capacity);
  const int64_t ne = (int64_t)(h.edge_top < (unsigned long long)t->cfg.edge_capacity ? h.edge_top : t->cfg.edge_capacity);
  const int V = t->cfg.vocab_capacity, extra = t->cfg.n_input_slots - 1;
  std::vector<Node> on((size_t)nn), nw;
  std::vector<int2> oe((size_t)ne), we;
  std::vector<int> root((size_t)V), newid((size_t)nn, -1), order;
  std::vector<float> ofx((size_t)extra * nn), nfx;
  if (nn) PIA_CUDA_CHECK(cudaMemcpy(on.data(), t->dev.nodes, (size_t)nn * sizeof(Node), cudaMemcpyDeviceToHost));
  if (ne) PIA_CUDA_CHECK(cudaMemcpy(oe.data(), t->dev.edges, (size_t)ne * sizeof(int2), cudaMemcpyDeviceToHost));
  PIA_CUDA_CHECK(cudaMemcpy(root.data(), t->dev.root_of, (size_t)V * sizeof(int), cudaMemcpyDeviceToHost));
  for (int e = 0; e < extra; ++e)
    if (nn) PIA_CUDA_CHECK(cudaMemcpy(ofx.data() + (size_t)e * nn, t->dev.fi_extra + (size_t)e * t->cfg.node_capacity,
                                      (size_t)nn * sizeof(float), cudaMemcpyDeviceToHost));
  auto child_of = [&](const Node &p, int k) -> int {
    if (p.cap == 0) return p.child;
    const long long o = (long long)p.child + k;
    return (o >= 0 && o < ne) ? oe[(size_t)o].y : -1;
  };
  // pass 1: depth-first pre-order numbering of everything reachable from a root
  order.reserve((size_t)nn);
  std::vector<int> stack;
  for (int tok = 0; tok < V; ++tok) {
    const int r = root[tok];
    if (r < 0 || r >= nn || newid[r] >= 0) continue;
    stack.push_back(r);
    while (!stack.empty()) {
      const int i = stack.back();
      stack.pop_back();
      if (i < 0 || i >= nn || newid[i] >= 0) continue;
      newid[i] = (int)order.size();
      order.push_back(i);
      const Node &p = on[i];
      for (int k = p.n_child - 1; k >= 0; --k) stack.push_back(child_of(p, k));  // first child numbered next
    }
  }
  // pass 2: records and trimmed child blocks
  const size_t live = order.size();
  nw.resize(live);
  nfx.resize((size_t)extra * live);
  for (size_t j = 0; j < live; ++j) {
    const int i = order[j];
    Node p = on[i];
    if (p.n_child <= 0) { p.n_child = 0; p.child = -1; p.cap = 0; }
    else if (p.cap == 0) { const int c = child_of(on[i], 0); p.child = (c >= 0 && c < nn) ? newid[c] : -1; if (p.child < 0) p.n_child = 0; }
    else {
      int cap = 4;
      while (cap < p.n_child) cap *= 2;
      const size_t off = we.size();
      we.resize(off + (size_t)cap, make_int2(-1, -1));
      for (int k = 0; k < p.n_child; ++k) {
        const long long o = (long long)on[i].child + k;
        int2 e = (o >= 0 && o < ne) ? oe[(size_t)o] : make_int2(-1, -1);
        e.y = (e.y >= 0 && e.y < nn) ? newid[e.y] : -1;
        we[off + k] = e;
      }
      p.child = (int)off; p.cap = cap;
    }
    nw[j] = p;
    for (int e = 0; e < extra; ++e) nfx[(size_t)e * live + j] = ofx[(size_t)e * nn + i];
  }
  PIA_REQUIRE((int64_t)we.size() <= t->cfg.edge_capacity, "compacted child blocks do not fit the edge pool");
  for (int tok = 0; tok < V; ++tok) if (root[tok] >= 0) root[tok] = root[tok] < nn ? newid[root[tok]] : -1;
  if (live) PIA_CUDA_CHECK(cudaMemcpy(t->dev.nodes, nw.data(), live * sizeof(Node), cudaMemcpyHostToDevice));
  if (!we.empty()) PIA_CUDA_CHECK(cudaMemcpy(t->dev.edges, we.data(), we.size() * sizeof(int2), cudaMemcpyHostToDevice));
  PIA_CUDA_CHECK(cudaMemcpy(t->dev.root_of, root.data(), (size_t)V * sizeof(int), cudaMemcpyHostToDevice));
  for (int e = 0; e < extra; ++e)
    if (live) PIA_CUDA_CHECK(cudaMemcpy(t->dev.fi_extra + (size_t)e * t->cfg.node_capacity, nfx.data() + (size_t)e * live,
                                        live * sizeof(float), cudaMemcpyHostToDevice));
  h.node_top = (unsigned long long)live; h.edge_top = (unsigned long long)we.size();
  h.err &= ~(ERR_NODE_POOL | ERR_EDGE_POOL);  // room again: inserts resume (what was dropped while full stays dropped)
  PIA_CUDA_CHECK(cudaMemcpy(t->dev.hdr, &h, sizeof(h), cudaMemcpyHostToDevice));
  if (h_nodes_before) *h_nodes_before = nn;
  if (h_nodes_after) *h_nodes_after = (int64_t)live;
  return PIA_OK;
}

// replaces the whole forest (like `self.mem = pickle.loads(...)`, :587); pending update sets are dropped
extern "C" int pia_trie_import(pia_trie_t *t, const void *h_nodes, int64_t n_nodes, const void *h_edges, int64_t n_edges,
                               const int32_t *h_root_of, const int32_t *h_n_node, const int32_t *h_n_out, void *stream) {
  PIA_REQUIRE(t && h_nodes && h_edges && h_root_of && h_n_node && h_n_out, "null argument");
  PIA_REQUIRE(n_nodes <= t->cfg.node_capacity && n_edges <= t->cfg.edge_capacity, "forest does not fit the pools");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t v = (size_t)t->cfg.vocab_capacity * sizeof(int);
  PIA_CUDA_CHECK(cudaMemcpyAsync(t->dev.nodes, h_nodes, (size_t)n_nodes * sizeof(Node), cudaMemcpyHostToDevice, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(t->dev.edges, h_edges, (size_t)n_edges * sizeof(int2), cudaMemcpyHostToDevice, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(t->dev.root_of, h_root_of, v, cudaMemcpyHostToDevice, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(t->dev.tree_n_node, h_n_node, v, cudaMemcpyHostToDevice, s));
  PIA_CUDA_CHECK(cudaMemcpyAsync(t->dev.tree_n_out, h_n_out, v, cudaMemcpyHostToDevice, s));
  PIA_CUDA_CHECK(cudaMemsetAsync(t->dev.tree_flags, 0, v, s));
  if (t->dev.fi_extra) PIA_CUDA_CHECK(cudaMemsetAsync(t->dev.fi_extra, 0, (size_t)(t->cfg.n_input_slots - 1) * t->cfg.node_capacity * sizeof(float), s));
  PIA_CUDA_CHECK(cudaStreamSynchronize(s));
  {  // the pruned query walk relies on parent counts bounding child counts; a forest written by put/squeeze/reset has
     // that property, an arbitrary file may not: check it once here (host, one pass) and fall back to full walks if not
    const Node *hn = static_cast<const Node *>(h_nodes);
    const int2 *he = static_cast<const int2 *>(h_edges);
    int mono = 1;
    for (int64_t i = 0; i < n_nodes && mono; ++i) {
      const Node &p = hn[i];
      for (int k = 0; k < p.n_child; ++k) {
        const int64_t c = p.cap == 0 ? p.child : (p.child + k < n_edges ? he[p.child + k].y : -1);
        if (c < 0 || c >= n_nodes) continue;
        if (hn[c].fo > p.fo || hn[c].fi > p.fi) { mono = 0; break; }
      }
    }
    t->monotone = mono;
  }
  Hdr h;
  PIA_CUDA_CHECK(cudaMemcpy(&h, t->dev.hdr, sizeof(h), cudaMemcpyDeviceToHost));
  h.node_top = (unsigned long long)n_nodes; h.edge_top = (unsigned long long)n_edges;
  h.n_upd = 0; h.n_updin = 0; h.n_upd_stale = 0;
  int trees = 0;
  for (int i = 0; i < t->cfg.vocab_capacity; ++i) trees += h_root_of[i] >= 0;
  h.n_trees = trees;
  PIA_CUDA_CHECK(cudaMemcpy(t->dev.hdr, &h, sizeof(h), cudaMemcpyHostToDevice));
  return PIA_OK;
}
