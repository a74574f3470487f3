// lfr_graph.cuh — the graph stage on the device (include/lfr_graph.h): node interning, CSR + edge
// records, constrained Kruskal, track ids and roots, the track meta-graph and its components, the
// dispatch list.  Each step reproduces one block of lfr_host.cc bit for bit, tie-breaks included;
// the comments name the block.  Only the recursive 2-way cut of oversized meta-components runs on the
// host (lfr_cut.h, the same code the host stage runs), on the downloaded edges of those components.
//
// Sorts and scans are CUB device primitives; every other step is a kernel of this file.  The host
// driver (build_graph_on_device) is in lfr_capi.cu.
#pragma once
#include <cstdint>

#include <cub/cub.cuh>

#include "../../include/lfr.h"

namespace lfr {
namespace graph {

constexpr uint32_t kListMax = 12;  // image sets of 2..12 images: a list of image ids (lfr_host.cc kListMax)

// lfr_host.cc sortable_bits: float -> uint32 whose unsigned order is the float order, -0.0 keyed as +0.0
// (equal under the reference's tuple sort, solve.cc:489)
__device__ __forceinline__ uint32_t sortable_bits(float f) {
  uint32_t u = __float_as_uint(f);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// double -> uint64 whose unsigned order is the order of the (finite) doubles.  -0.0 would key below +0.0,
// but the root scores it sees are sums that start at +0.0, and under round-to-nearest such a sum is never
// -0.0 (x + -x and +0.0 + -0.0 both give +0.0)
__device__ __forceinline__ unsigned long long sortable_bits64(double d) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(d);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

__global__ void iota_kernel(uint32_t* a, uint64_t n) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) a[i] = (uint32_t)i;
}

// ---- H1: the match list (lfr_host.cc "H1: node interning + directed edges") ---------------------
// kept matches of every pair (0 for a skipped pair); images of non-skipped pairs are range-checked
// and marked seen.  err[0] = 1: image id out of range.
__global__ void pair_count_kernel(const uint32_t* img1, const uint32_t* img2, const uint8_t* skip, const uint64_t* ptr,
                                  uint64_t n_pairs, uint32_t n_images, uint64_t* cnt, uint8_t* seen, int* err) {
  const uint64_t p = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (p >= n_pairs) return;
  if (skip && skip[p]) {
    cnt[p] = 0;
    return;
  }
  const uint32_t a = img1[p], b = img2[p];
  if (a >= n_images || b >= n_images) {
    err[0] = 1;
    cnt[p] = 0;
    return;
  }
  seen[a] = 1;
  seen[b] = 1;
  cnt[p] = ptr[p + 1] >= ptr[p] ? ptr[p + 1] - ptr[p] : 0;
}

// kept match k -> its match index and pair images; keys of both sides for interning
// (position 2k = side 1, 2k+1 = side 2: the order of first appearance).  err[1] = 1: non-finite sim.
__global__ void expand_matches_kernel(const uint64_t* off /* [n_pairs+1] exclusive sums of cnt */, uint64_t n_pairs,
                                      const uint32_t* img1, const uint32_t* img2, const uint64_t* ptr,
                                      const uint32_t* feat1, const uint32_t* feat2, const float* sim, uint64_t M,
                                      uint64_t* kept_m, unsigned long long* key, uint32_t* pos, int* err) {
  const uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (k >= M) return;
  uint64_t lo = 0, hi = n_pairs;  // the pair p with off[p] <= k < off[p+1]
  while (hi - lo > 1) {
    const uint64_t mid = (lo + hi) / 2;
    if (off[mid] <= k) lo = mid; else hi = mid;
  }
  const uint64_t p = lo;
  const uint64_t m = ptr[p] + (k - off[p]);
  kept_m[k] = m;
  if (!isfinite(sim[m])) err[1] = 1;
  key[2 * k] = ((unsigned long long)img1[p] << 32) | feat1[m];
  key[2 * k + 1] = ((unsigned long long)img2[p] << 32) | feat2[m];
  pos[2 * k] = (uint32_t)(2 * k);
  pos[2 * k + 1] = (uint32_t)(2 * k + 1);
}

// after a stable sort of (key, position): a run of equal keys starts with the key's first position
__global__ void first_flags_kernel(const unsigned long long* skey, const uint32_t* spos, uint64_t n, uint32_t* first,
                                   uint32_t* head_idx) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool head = i == 0 || skey[i] != skey[i - 1];
  first[spos[i]] = head ? 1u : 0u;
  head_idx[i] = head ? (uint32_t)i : 0u;
}

// node id of every position (= the source node of directed edge j = position j); node image / feature
__global__ void assign_nodes_kernel(const unsigned long long* skey, const uint32_t* spos, const uint32_t* head_of,
                                    const uint32_t* id_of_pos, uint64_t n, uint32_t* node_of_pos, uint32_t* node_image,
                                    uint32_t* node_feat) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t h = head_of[i];
  const uint32_t id = id_of_pos[spos[h]];
  node_of_pos[spos[i]] = id;
  if (h == i) {
    node_image[id] = (uint32_t)(skey[i] >> 32);
    node_feat[id] = (uint32_t)(skey[i] & 0xffffffffu);
  }
}

// CSR: row_ptr[v] = first slot of source v (every node has an out-edge); row_ptr[N] = E
__global__ void row_ptr_kernel(const uint32_t* ssrc, uint64_t E, uint32_t N, uint32_t* row_ptr) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= E) return;
  if (i == 0 || ssrc[i] != ssrc[i - 1]) row_ptr[ssrc[i]] = (uint32_t)i;
  if (i == 0) row_ptr[N] = (uint32_t)E;
}

// the 80-byte records in CSR order: slot i holds directed edge j = perm[i] of match k = j / 2;
// n1 -> n2 (j even) carries disp2, n2 -> n1 carries disp1; its destination is position j ^ 1
__global__ void edge_records_kernel(const uint32_t* perm, uint64_t E, const uint64_t* kept_m, const uint32_t* node_of_pos,
                                    const float* sim, const float* disp1, const float* disp2, lfr_edge* edges,
                                    uint32_t* cdst, float* csim) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= E) return;
  const uint32_t j = perm[i];
  const uint64_t m = kept_m[j >> 1];
  const float2* f = reinterpret_cast<const float2*>(((j & 1u) ? disp1 : disp2) + 18 * m);
  const uint32_t dst = node_of_pos[j ^ 1u];
  const float s = sim[m];
  float v[20];
#pragma unroll
  for (int q = 0; q < 9; ++q) {
    const float2 x = f[q];
    v[2 * q] = x.x;
    v[2 * q + 1] = x.y;
  }
  v[18] = s;
  v[19] = __uint_as_float(dst);
  float4* o = reinterpret_cast<float4*>(edges + i);
#pragma unroll
  for (int q = 0; q < 5; ++q) o[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  cdst[i] = dst;
  csim[i] = s;
}

// ---- H2: constrained Kruskal (lfr_host.cc "H2") ---------------------------------------------------
// sort keys: first pass by n2, second by (sortable_bits(sim), n1); stable, so ties end in (n2, k) order
__global__ void kruskal_keys_kernel(const uint32_t* node_of_pos, uint64_t M, uint32_t* n2key) {
  const uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (k >= M) return;
  n2key[k] = node_of_pos[2 * k + 1];
}

// (sortable_bits(sim), n1) packed into 32 + n1_bits bits
__global__ void kruskal_keys2_kernel(const uint32_t* perm, const uint64_t* kept_m, const uint32_t* node_of_pos,
                                     const float* sim, uint64_t M, int n1_bits, unsigned long long* key) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= M) return;
  const uint32_t k = perm[i];
  key[i] = ((unsigned long long)sortable_bits(sim[kept_m[k]]) << n1_bits) | node_of_pos[2 * k];
}

// Union-find state.  A root's image set: <= 64 images a 64-bit mask (small_sets); otherwise {its own
// image} while a singleton, a list of up to kListMax image ids in `lists` (per node), then a bitset of
// W words from `pool`.  Sets never share an image, so a set's size is also its node count and the
// union by size keeps every tree O(log N) deep: find() needs no path compression.
struct UfState {
  int32_t* parent;           // -1 = root
  uint32_t* size;            // images (= nodes) of a root's set
  unsigned long long* mask;  // small_sets
  uint16_t* lists;           // [N * kListMax]
  int32_t* slot;             // bitset slot of a root with more than kListMax images
  unsigned long long* pool;  // [slots * W]
  uint32_t* pool_next;
  uint32_t W;
  bool small_sets;
  const uint32_t* node_image;
  uint32_t* res;             // reservation: lowest rank of a pending edge touching the root
};

__global__ void uf_init_kernel(UfState S, uint32_t N) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  S.parent[v] = -1;
  S.size[v] = 1;
  S.res[v] = 0xffffffffu;
  if (S.small_sets) S.mask[v] = 1ull << S.node_image[v];
}

__device__ __forceinline__ uint32_t uf_find(const int32_t* parent, uint32_t x) {
  int32_t p;
  while ((p = parent[x]) != -1) x = (uint32_t)p;
  return x;
}

__device__ bool set_has(const UfState& S, uint32_t r, uint32_t img) {
  const uint32_t sz = S.size[r];
  if (sz == 1) return S.node_image[r] == img;
  if (sz <= kListMax) {
    const uint16_t* l = S.lists + (size_t)r * kListMax;
    for (uint32_t i = 0; i < sz; ++i)
      if (l[i] == img) return true;
    return false;
  }
  return (S.pool[(size_t)S.slot[r] * S.W + (img >> 6)] >> (img & 63)) & 1ull;
}

template <typename F>
__device__ void for_each_image(const UfState& S, uint32_t r, F&& fn) {
  const uint32_t sz = S.size[r];
  if (sz == 1) {
    fn(S.node_image[r]);
  } else if (sz <= kListMax) {
    const uint16_t* l = S.lists + (size_t)r * kListMax;
    for (uint32_t i = 0; i < sz; ++i) fn((uint32_t)l[i]);
  } else {
    const unsigned long long* b = S.pool + (size_t)S.slot[r] * S.W;
    for (uint32_t w = 0; w < S.W; ++w)
      for (unsigned long long m = b[w]; m; m &= m - 1) fn(64 * w + (uint32_t)__ffsll((long long)m) - 1);
  }
}

__device__ bool sets_clash(const UfState& S, uint32_t a, uint32_t b) {  // a = the smaller set
  if (S.size[a] > kListMax && S.size[b] > kListMax) {
    const unsigned long long* x = S.pool + (size_t)S.slot[a] * S.W;
    const unsigned long long* y = S.pool + (size_t)S.slot[b] * S.W;
    for (uint32_t w = 0; w < S.W; ++w)
      if (x[w] & y[w]) return true;
    return false;
  }
  bool clash = false;
  for_each_image(S, a, [&](uint32_t img) { clash = clash || set_has(S, b, img); });
  return clash;
}

// dst <- dst U src (disjoint)
__device__ void absorb(const UfState& S, uint32_t dst, uint32_t src) {
  const uint32_t sd = S.size[dst], new_size = sd + S.size[src];
  if (new_size <= kListMax) {
    uint16_t* l = S.lists + (size_t)dst * kListMax;
    if (sd == 1) l[0] = (uint16_t)S.node_image[dst];
    uint32_t n = sd;
    for_each_image(S, src, [&](uint32_t img) { l[n++] = (uint16_t)img; });
  } else {
    if (sd <= kListMax) {  // singleton / list -> a fresh (zeroed) bitset
      const uint32_t sl = atomicAdd(S.pool_next, 1u);
      unsigned long long* b = S.pool + (size_t)sl * S.W;
      for_each_image(S, dst, [&](uint32_t img) { b[img >> 6] |= 1ull << (img & 63); });
      S.slot[dst] = (int32_t)sl;
    }
    unsigned long long* b = S.pool + (size_t)S.slot[dst] * S.W;
    if (S.size[src] > kListMax) {
      const unsigned long long* c = S.pool + (size_t)S.slot[src] * S.W;
      for (uint32_t w = 0; w < S.W; ++w) b[w] |= c[w];
    } else {
      for_each_image(S, src, [&](uint32_t img) { b[img >> 6] |= 1ull << (img & 63); });
    }
  }
  S.size[dst] = new_size;
  S.size[src] = 0;
}

// Deterministic reservations over a window of the pending edges, in rank order (rank r = the r-th
// edge the sequential loop visits).  Round: (1) every window edge finds its two roots; equal roots
// reject it, otherwise it reserves both with atomicMin(rank).  (2) an edge holding both reservations
// is the lowest-ranked pending edge on either root, so it sees exactly the sets the sequential loop
// would: it rejects on an image clash or unions.  (3) reservations are cleared, finished edges leave.
// win_state: 0 pending, 1 done.
__global__ void kr_reserve_kernel(UfState S, const uint32_t* win, uint32_t n_win, const uint32_t* order, uint32_t M,
                                  const uint32_t* node_of_pos, uint32_t* wr1, uint32_t* wr2, uint8_t* win_state) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_win) return;
  const uint32_t r = win[i];
  const uint32_t k = order[M - 1 - r];
  const uint32_t r1 = uf_find(S.parent, node_of_pos[2 * (size_t)k]), r2 = uf_find(S.parent, node_of_pos[2 * (size_t)k + 1]);
  wr1[i] = r1;
  wr2[i] = r2;
  if (r1 == r2) {
    win_state[i] = 1;
    return;
  }
  win_state[i] = 0;
  atomicMin(&S.res[r1], r);
  atomicMin(&S.res[r2], r);
}

__global__ void kr_decide_kernel(UfState S, const uint32_t* win, uint32_t n_win, const uint32_t* wr1, const uint32_t* wr2,
                                 uint8_t* win_state) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_win || win_state[i]) return;
  const uint32_t r = win[i], r1 = wr1[i], r2 = wr2[i];
  if (S.res[r1] != r || S.res[r2] != r) return;
  win_state[i] = 2;  // decided (cleared to 1 by kr_release_kernel, after every decision has read `res`)
  if (S.small_sets) {
    const unsigned long long m1 = S.mask[r1], m2 = S.mask[r2];
    if (m1 & m2) return;  // set_intersection non-empty (solve.cc:507-511)
    if (__popcll(m1) < __popcll(m2)) {  // solve.cc:513-521
      S.parent[r1] = (int32_t)r2;
      S.mask[r2] = m1 | m2;
      S.mask[r1] = 0;
    } else {
      S.parent[r2] = (int32_t)r1;
      S.mask[r1] = m1 | m2;
      S.mask[r2] = 0;
    }
    return;
  }
  // smaller set under larger, tie: root2 under root1
  const bool r1_smaller = S.size[r1] < S.size[r2];
  if (sets_clash(S, r1_smaller ? r1 : r2, r1_smaller ? r2 : r1)) return;
  if (r1_smaller) {
    S.parent[r1] = (int32_t)r2;
    absorb(S, r2, r1);
  } else {
    S.parent[r2] = (int32_t)r1;
    absorb(S, r1, r2);
  }
}

__global__ void kr_release_kernel(UfState S, uint32_t n_win, const uint32_t* wr1, const uint32_t* wr2, uint8_t* win_state,
                                  uint32_t* keep) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_win) return;
  const uint8_t st = win_state[i];
  if (st != 1) {  // it reserved both roots this round
    S.res[wr1[i]] = 0xffffffffu;
    S.res[wr2[i]] = 0xffffffffu;
  }
  keep[i] = st == 0 ? 1u : 0u;
}

// survivors (in order) first, then the next ranks of the sequence
__global__ void kr_refill_kernel(uint32_t* win, uint32_t ns, uint32_t n_add, uint32_t next) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_add) win[ns + t] = next + t;
}

// ---- H3: track ids and roots (lfr_host.cc "H3") ---------------------------------------------------
__global__ void root_flags_kernel(const int32_t* parent, uint32_t N, uint32_t* flag) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < N) flag[v] = parent[v] == -1 ? 1u : 0u;
}

__global__ void track_ids_kernel(const int32_t* parent, const uint32_t* tid_of_root, uint32_t N, uint32_t* track,
                                 uint32_t* nodes_in_track) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  const uint32_t t = tid_of_root[uf_find(parent, v)];
  track[v] = t;
  atomicAdd(&nodes_in_track[t], 1u);
}

// score of node v: its intra-track out-edges' similarities summed in CSR order (one thread, the host's
// order, so the double is bit-identical); per track the max score
__global__ void root_score_kernel(const uint32_t* row_ptr, const uint32_t* cdst, const float* csim, const uint32_t* track,
                                  uint32_t N, double* score, unsigned long long* best) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  const uint32_t t = track[v];
  double s = 0.0;
  for (uint32_t e = row_ptr[v]; e < row_ptr[v + 1]; ++e)
    if (track[cdst[e]] == t) s += (double)csim[e];
  score[v] = s;
  atomicMax(&best[t], sortable_bits64(s));
}

// the root: lexicographic max of (score, node)
__global__ void root_pick_kernel(const double* score, const unsigned long long* best, const uint32_t* track, uint32_t N,
                                 uint32_t* best_node) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  const uint32_t t = track[v];
  if (sortable_bits64(score[v]) == best[t]) atomicMax(&best_node[t], v);
}

__global__ void root_mark_kernel(const uint32_t* best_node, uint32_t T, uint8_t* is_root) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) is_root[best_node[t]] = 1;
}

// ---- H4: meta-graph, components, cut (lfr_host.cc "H4") -------------------------------------------
// key of every directed edge: (source track, destination track); inter-track flag
__global__ void meta_keys_kernel(const uint32_t* ssrc, const uint32_t* cdst, const uint32_t* track, uint64_t E, uint32_t T,
                                 unsigned long long* key, uint32_t* inter) {
  const uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint32_t ts = track[ssrc[e]], tt = track[cdst[e]];
  key[e] = (unsigned long long)ts * T + tt;
  inter[e] = ts != tt ? 1u : 0u;
}

__global__ void seg_heads_kernel(const unsigned long long* key, uint64_t n, uint32_t* head) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) head[i] = (i == 0 || key[i] != key[i - 1]) ? 1u : 0u;
}

// one meta-edge per run of equal keys: its weight summed left to right (the host's double sum)
__global__ void meta_sum_kernel(const unsigned long long* key, const float* sim, const uint32_t* seg_start, uint32_t n_seg,
                                uint64_t n, uint32_t T, uint32_t* ma, uint32_t* mb, double* wsum) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg) return;
  const uint64_t lo = seg_start[s], hi = s + 1 < n_seg ? seg_start[s + 1] : n;
  double sum = (double)sim[lo];
  for (uint64_t i = lo + 1; i < hi; ++i) sum += (double)sim[i];
  const unsigned long long k = key[lo];
  ma[s] = (uint32_t)(k / T);
  mb[s] = (uint32_t)(k % T);
  wsum[s] = sum;
}

// connected components: every tree is hooked under its smaller root, so a component's root is its
// lowest member; `gc` (optional) keeps only the edges inside one cut group
__device__ __forceinline__ uint32_t cc_find(uint32_t* p, uint32_t x) {
  uint32_t y;
  while ((y = p[x]) != x) {
    const uint32_t z = p[y];
    if (z != y) atomicCAS(&p[x], y, z);  // path halving
    x = y;
  }
  return x;
}

__global__ void cc_hook_kernel(const uint32_t* ma, const uint32_t* mb, uint32_t n, const uint32_t* gc, uint32_t* p) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (gc && gc[ma[i]] != gc[mb[i]]) return;
  uint32_t a = ma[i], b = mb[i];
  for (;;) {
    a = cc_find(p, a);
    b = cc_find(p, b);
    if (a == b) return;
    if (a < b) {
      const uint32_t t = a;
      a = b;
      b = t;
    }
    if (atomicCAS(&p[a], a, b) == a) return;
  }
}

__global__ void cc_flatten_kernel(uint32_t* p, uint32_t n, uint32_t* is_rep) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t r = cc_find(p, i);
  p[i] = r;
  is_rep[i] = r == i ? 1u : 0u;
}

__global__ void cc_label_kernel(const uint32_t* p, const uint32_t* label_of_rep, uint32_t n, uint32_t* label) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) label[i] = label_of_rep[p[i]];
}

__global__ void cc_weight_kernel(const uint32_t* cc, const uint32_t* nodes_in_track, uint32_t T, unsigned long long* cc_nodes) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) atomicAdd(&cc_nodes[cc[t]], (unsigned long long)nodes_in_track[t]);
}

// cap (may be NULL: max_nodes for all): the cut cap of each meta-component (sub-scenes, lfr_host_input::image_group)
__global__ void oversized_kernel(const unsigned long long* cc_nodes, uint32_t n_cc, uint32_t max_nodes, const uint32_t* cap,
                                 uint32_t* big) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n_cc) big[c] = cc_nodes[c] > (cap ? cap[c] : max_nodes) ? 1u : 0u;
}

// undirected meta-edges (ma < mb) of oversized components, weight int(100 * sum) (solve.cc:327-330)
__global__ void cut_edges_flag_kernel(const uint32_t* ma, const uint32_t* mb, const uint32_t* cc, const uint32_t* big,
                                      uint32_t n, uint32_t* flag) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = (ma[i] < mb[i] && big[cc[ma[i]]]) ? 1u : 0u;
}

struct CutRec {
  uint32_t a, b, comp, pad;
  double wsum;  // the weight int(100 * wsum) is taken on the host, lfr::cut_weight (lfr_cut.h)
};

__global__ void cut_edges_gather_kernel(const uint32_t* idx, uint32_t n, const uint32_t* ma, const uint32_t* mb,
                                        const double* wsum, const uint32_t* cc, CutRec* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e = idx[i];
  out[i] = CutRec{ma[e], mb[e], cc[ma[e]], 0u, wsum[e]};
}

__global__ void scatter_kernel(const uint32_t* idx, const uint32_t* val, uint32_t n, uint32_t* dst) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[idx[i]] = val[i];
}

// sub-scenes: cc_cap[meta-component of node v] = the image count of v's sub-scene (every node of a
// meta-component writes the same value)
__global__ void cc_cap_kernel(const uint32_t* node_image, const uint32_t* track, const uint32_t* cc, const uint32_t* image_cap,
                              uint32_t n, uint32_t* cc_cap) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) cc_cap[cc[track[v]]] = image_cap[node_image[v]];
}

__global__ void gather_kernel(const uint32_t* idx, const uint32_t* src, uint32_t n, uint32_t* dst) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

// ---- H5: dispatch list (lfr_host.cc "H5") ---------------------------------------------------------
__global__ void comp_size_kernel(const uint32_t* comp, uint32_t N, uint32_t* size) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < N) atomicAdd(&size[comp[v]], 1u);
}

// sort + reverse on (size, id): a descending sort of size << 32 | id
__global__ void comp_keys_kernel(const uint32_t* size, uint32_t C, unsigned long long* key) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) key[c] = ((unsigned long long)size[c] << 32) | c;
}

__global__ void comp_slots_kernel(const unsigned long long* skey, uint32_t C, uint32_t* comp_order, uint32_t* slot_of,
                                  uint32_t* slot_size) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= C) return;
  const uint32_t c = (uint32_t)(skey[s] & 0xffffffffu);
  comp_order[s] = c;
  slot_of[c] = s;
  slot_size[s] = (uint32_t)(skey[s] >> 32);
}

__global__ void node_slot_kernel(const uint32_t* comp, const uint32_t* slot_of, uint32_t N, uint32_t* node_slot) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < N) node_slot[v] = slot_of[comp[v]];
}

}  // namespace graph
}  // namespace lfr
