// lfr_diff.cuh — which components of a device-resident plan pose the problem an earlier plan posed
// (lfr_plan_update_solution_since, include/lfr_graph.h, which states the rule), over both plans' arrays in
// HBM.  Keypoints are keyed as the start-point join keys them (image id << 32 | feature_idx, lfr_start.cuh),
// the earlier plan's image ids mapped to this plan's by name on the host.
//
//   prev_key_kernel + radix sort   the earlier nodes by key
//   node_kernel                    each node's earlier node (binary search), its inverse, the nodes without
//                                  one and the root flags that differ; per component the lowest and highest
//                                  earlier component and the size
//   size_kernel / comp_kernel      one earlier component of the same size
//   edge_key_kernel (twice) + radix sort   the kept edges of both plans keyed (source, destination) in this
//                                  plan's node ids, the value naming the plan, the record and the kind
//   run_kernel                     every run of one key compared as a multiset, exactly: kind and the bits of
//                                  sim and of the 18 flow floats
// A failure sets changed[c] of this plan's component c; stores are idempotent.
#pragma once

#include <cstdint>

namespace lfr {
namespace diff {

constexpr uint32_t kNone = 0xffffffffu;

__device__ __forceinline__ unsigned long long node_key(uint32_t image, uint32_t feat) {
  return (unsigned long long)image << 32 | feat;
}

// the last u with row_ptr[u] <= e: the source of edge e
__device__ __forceinline__ uint32_t source_of(const uint32_t* row_ptr, uint32_t n, uint32_t e) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (row_ptr[mid] <= e) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void prev_key_kernel(const uint32_t* __restrict__ node_image, const uint32_t* __restrict__ node_feat, uint32_t M,
                                const uint32_t* __restrict__ image_map, unsigned long long* __restrict__ key,
                                uint32_t* __restrict__ idx) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= M) return;
  key[u] = node_key(image_map[node_image[u]], node_feat[u]);
  idx[u] = u;
}

// m[v] = the earlier node with v's key (kNone without one), inv[m[v]] = v (inv starts all kNone)
__global__ void node_kernel(const uint32_t* __restrict__ node_image, const uint32_t* __restrict__ node_feat,
                            const uint32_t* __restrict__ comp, const uint8_t* __restrict__ is_root, uint32_t N,
                            const unsigned long long* __restrict__ key_s, const uint32_t* __restrict__ idx_s, uint32_t M,
                            const uint32_t* __restrict__ prev_comp, const uint8_t* __restrict__ prev_root,
                            uint32_t* __restrict__ inv, uint32_t* __restrict__ lo_pc, uint32_t* __restrict__ hi_pc,
                            uint32_t* __restrict__ size, uint8_t* __restrict__ changed) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  const uint32_t c = comp[v];
  atomicAdd(&size[c], 1u);
  const unsigned long long k = node_key(node_image[v], node_feat[v]);
  uint32_t lo = 0, hi = M;  // the first earlier key >= k
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (key_s[mid] < k) lo = mid + 1; else hi = mid;
  }
  if (lo == M || key_s[lo] != k) {
    changed[c] = 1;
    return;
  }
  const uint32_t u = idx_s[lo];
  inv[u] = v;
  if ((is_root[v] != 0) != (prev_root[u] != 0)) changed[c] = 1;
  atomicMin(&lo_pc[c], prev_comp[u]);
  atomicMax(&hi_pc[c], prev_comp[u]);
}

__global__ void size_kernel(const uint32_t* __restrict__ comp, uint32_t n, uint32_t* __restrict__ size) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) atomicAdd(&size[comp[v]], 1u);
}

// every node of c maps into one earlier component, whose size is c's: then the two hold the same keypoints
__global__ void comp_kernel(const uint32_t* __restrict__ lo_pc, const uint32_t* __restrict__ hi_pc,
                            const uint32_t* __restrict__ size, const uint32_t* __restrict__ prev_size, uint32_t C,
                            uint8_t* __restrict__ changed) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C || changed[c]) return;
  if (lo_pc[c] != hi_pc[c] || lo_pc[c] == kNone || size[c] != prev_size[lo_pc[c]]) changed[c] = 1;
}

// Edge e of one plan (n nodes, `to_cur` maps its node ids to this plan's, NULL for this plan itself): a kept
// edge gets key = source << 32 | destination in this plan's ids (kNone for a destination without one) and
// value = side << 34 | kind << 32 | e; a skipped edge, or one whose source has no node here, gets `sentinel`,
// which sorts after every kept key.
__global__ void edge_key_kernel(const uint32_t* __restrict__ row_ptr, const float4* __restrict__ edges,
                                const uint32_t* __restrict__ track, const uint32_t* __restrict__ comp, uint32_t n, uint32_t E,
                                const uint32_t* __restrict__ to_cur, unsigned long long side, unsigned long long sentinel,
                                unsigned long long* __restrict__ key, unsigned long long* __restrict__ val) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint32_t s = source_of(row_ptr, n, e);
  const uint32_t d = __float_as_uint(edges[5 * (size_t)e + 4].w);  // lfr_edge.dst, the record's last word
  const uint32_t kind = track[s] == track[d] ? LFR_EDGE_CAUCHY : (comp[s] == comp[d] ? LFR_EDGE_TUKEY : LFR_EDGE_SKIP);
  const uint32_t sc = to_cur ? to_cur[s] : s, dc = to_cur ? to_cur[d] : d;
  key[e] = (kind == LFR_EDGE_SKIP || sc == kNone) ? sentinel : ((unsigned long long)sc << 32 | dc);
  val[e] = side << 34 | (unsigned long long)kind << 32 | e;
}

// whether the records of two sorted values are equal: kind, then the bits of flow[18] and sim
__device__ __forceinline__ bool same_record(unsigned long long a, unsigned long long b, const uint32_t* __restrict__ cur,
                                            const uint32_t* __restrict__ prev) {
  if (((a >> 32) & 3u) != ((b >> 32) & 3u)) return false;
  const uint32_t* ra = ((a >> 34) ? prev : cur) + 20 * (size_t)(uint32_t)a;
  const uint32_t* rb = ((b >> 34) ? prev : cur) + 20 * (size_t)(uint32_t)b;
  for (int i = 0; i < 19; ++i)
    if (ra[i] != rb[i]) return false;
  return true;
}

// One thread per run of equal keys (its first slot): the run's records of this plan and of the earlier one
// must be equal multisets.  A run is short (the edges between one pair of keypoints: one per side unless a
// match is repeated), so each record's multiplicity is counted by a scan of the run.
__global__ void run_kernel(const unsigned long long* __restrict__ key_s, const unsigned long long* __restrict__ val_s,
                           uint32_t n, unsigned long long sentinel, const uint32_t* __restrict__ cur_edges,
                           const uint32_t* __restrict__ prev_edges, const uint32_t* __restrict__ comp,
                           uint8_t* __restrict__ changed) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned long long k = key_s[j];
  if (k == sentinel || (j > 0 && key_s[j - 1] == k)) return;
  uint32_t end = j + 1;
  while (end < n && key_s[end] == k) ++end;
  const uint32_t c = comp[(uint32_t)(k >> 32)];
  if (changed[c]) return;
  int balance = 0;
  for (uint32_t i = j; i < end; ++i) balance += (val_s[i] >> 34) ? -1 : 1;
  bool same = balance == 0;
  for (uint32_t i = j; same && i < end; ++i) {
    if (val_s[i] >> 34) continue;
    int count = 0;  // this plan's copies minus the earlier plan's
    for (uint32_t q = j; q < end; ++q)
      if (same_record(val_s[i], val_s[q], cur_edges, prev_edges)) count += (val_s[q] >> 34) ? -1 : 1;
    same = count == 0;
  }
  if (!same) changed[c] = 1;
}

}  // namespace diff
}  // namespace lfr
