// lfr_record.cuh — the problem record of a device-resident plan (lfr_plan_problem_record,
// lfr_plan_update_solution_since_record; include/lfr_graph.h states the rule), over the plan's arrays in
// HBM.  The element hashes are lfr_record.h's, the code the host library runs.
//
//   digest_kernel   one thread per node element and per out-edge (nodes, then edges in CSR order): its
//                   element hash when it is a node or a kept edge; equal components in consecutive lanes
//                   are summed in a segmented warp scan, and the last lane of each run adds the run to
//                   digest[c] with one 64-bit atomic per lane of the hash.  Sums are exact mod 2^64, so
//                   the order of the atomics does not matter.
//   two stable radix sorts (by d1, then by d0) order the digests; lookup_kernel marks the components
//   whose digest an earlier record lacks (binary search).
//   Many scenes of one plan: component_group_kernel gives every component its scene, group_lookup_kernel searches
//   only that scene's slice of the concatenated records, and record_group_off_kernel / record_write_kernel lay out
//   every scene's record after a third stable radix pass by scene.
#pragma once

#include <cstdint>

#include "lfr_record.h"

namespace lfr {
namespace record {

constexpr uint32_t kNoComp = 0xffffffffu;

// the last u with row_ptr[u] <= e: the source of edge e
__device__ __forceinline__ uint32_t edge_source(const uint32_t* __restrict__ row_ptr, uint32_t n, uint32_t e) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (row_ptr[mid] <= e) lo = mid; else hi = mid;
  }
  return lo;
}

// `ids` = the name id of every image, (id.0, id.1)
__global__ void __launch_bounds__(256) digest_kernel(
    const uint32_t* __restrict__ row_ptr, const float4* __restrict__ edges, const uint32_t* __restrict__ track,
    const uint32_t* __restrict__ comp, const uint8_t* __restrict__ is_root, const uint32_t* __restrict__ node_image,
    const uint32_t* __restrict__ node_feat, const ulonglong2* __restrict__ ids, uint32_t N, uint64_t E,
    unsigned long long* __restrict__ d0, unsigned long long* __restrict__ d1) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t c = kNoComp;
  uint64_t h0 = 0, h1 = 0;
  if (i < N) {
    const uint32_t v = (uint32_t)i;
    const ulonglong2 id = ids[node_image[v]];
    node_element(id.x, id.y, node_feat[v], is_root[v] != 0, h0, h1);
    c = comp[v];
  } else if (i < N + E) {
    const uint32_t e = (uint32_t)(i - N);
    const uint32_t v = edge_source(row_ptr, N, e);
    const float4* r = edges + 5 * (size_t)e;
    uint32_t w[20];
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const float4 f = r[q];
      w[4 * q] = __float_as_uint(f.x);
      w[4 * q + 1] = __float_as_uint(f.y);
      w[4 * q + 2] = __float_as_uint(f.z);
      w[4 * q + 3] = __float_as_uint(f.w);
    }
    const uint32_t d = w[19];  // lfr_edge.dst
    const uint32_t cv = comp[v];
    const uint32_t kind = edge_kind(track[v], track[d], cv, comp[d]);
    if (kind != LFR_EDGE_SKIP) {
      const ulonglong2 iv = ids[node_image[v]], iw = ids[node_image[d]];
      edge_element(iv.x, iv.y, iw.x, iw.y, node_feat[v], node_feat[d], kind, w, h0, h1);
      c = cv;
    }
  }
  // segmented inclusive scan over runs of equal c in consecutive lanes
  const unsigned lane = threadIdx.x & 31u;
  const uint32_t c_prev = __shfl_up_sync(0xffffffffu, c, 1);
  const unsigned heads = __ballot_sync(0xffffffffu, lane == 0 || c_prev != c);
  const unsigned head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));  // first lane of this lane's run
#pragma unroll
  for (unsigned off = 1; off < 32; off <<= 1) {
    const uint64_t a0 = __shfl_up_sync(0xffffffffu, h0, off), a1 = __shfl_up_sync(0xffffffffu, h1, off);
    if (lane >= head + off) {
      h0 += a0;
      h1 += a1;
    }
  }
  const uint32_t c_next = __shfl_down_sync(0xffffffffu, c, 1);
  if (c != kNoComp && (lane == 31 || c_next != c)) {
    atomicAdd(&d0[c], (unsigned long long)h0);
    atomicAdd(&d1[c], (unsigned long long)h1);
  }
}

// changed[c] = 1 unless (d0[c], d1[c]) is among the R earlier digests `rec` ((d0, d1) pairs, ascending)
__global__ void lookup_kernel(const unsigned long long* __restrict__ d0, const unsigned long long* __restrict__ d1,
                              uint32_t C, const ulonglong2* __restrict__ rec, uint64_t R, uint8_t* __restrict__ changed) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const unsigned long long a = d0[c], b = d1[c];
  uint64_t lo = 0, hi = R;  // the first earlier digest >= (a, b)
  while (lo < hi) {
    const uint64_t mid = (lo + hi) / 2;
    const ulonglong2 m = rec[mid];
    if (m.x < a || (m.x == a && m.y < b)) lo = mid + 1; else hi = mid;
  }
  changed[c] = (lo < R && rec[lo].x == a && rec[lo].y == b) ? 0 : 1;
}

// ---- many scenes in one plan (lfr_plan_update_solution_groups, lfr_plan_problem_record_groups) --------------
// A component lies in one scene: cgroup[comp[v]] = the group of v's image (the stores of one component agree).
__global__ void component_group_kernel(const uint32_t* __restrict__ comp, const uint32_t* __restrict__ node_image,
                                       const uint32_t* __restrict__ group_of_image, uint32_t N, uint32_t* __restrict__ cgroup) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < N) cgroup[comp[v]] = group_of_image[node_image[v]];
}

// lookup_kernel within each component's own scene: rec holds every scene's earlier digests back to back, scene g's
// in [rec_off[g], rec_off[g + 1]), ascending.  A component of a scene without a record (has_rec[g] == 0) is not
// changed: the plain update rule.
__global__ void group_lookup_kernel(const unsigned long long* __restrict__ d0, const unsigned long long* __restrict__ d1,
                                    const uint32_t* __restrict__ cgroup, uint32_t C, const ulonglong2* __restrict__ rec,
                                    const uint64_t* __restrict__ rec_off, const uint8_t* __restrict__ has_rec,
                                    uint8_t* __restrict__ changed) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const uint32_t g = cgroup[c];
  if (!has_rec[g]) {
    changed[c] = 0;
    return;
  }
  const unsigned long long a = d0[c], b = d1[c];
  const uint64_t R = rec_off[g + 1];
  uint64_t lo = rec_off[g], hi = R;  // the first earlier digest of the scene >= (a, b)
  while (lo < hi) {
    const uint64_t mid = (lo + hi) / 2;
    const ulonglong2 m = rec[mid];
    if (m.x < a || (m.x == a && m.y < b)) lo = mid + 1; else hi = mid;
  }
  changed[c] = (lo < R && rec[lo].x == a && rec[lo].y == b) ? 0 : 1;
}

// out[i] = src[idx[i]]
__global__ void gather_u64_kernel(const unsigned long long* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t n,
                                  unsigned long long* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[idx[i]];
}

// out[i] = src[idx[i]]
__global__ void gather_u32_kernel(const uint32_t* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t n,
                                  uint32_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[idx[i]];
}

// goff[g] (g <= G) = the byte offset of scene g's record: 16 per record header and per digest before it; `gs` = the
// C component groups in ascending order
__global__ void record_group_off_kernel(const uint32_t* __restrict__ gs, uint32_t C, uint32_t G, uint64_t* __restrict__ goff) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g > G) return;
  uint32_t lo = 0, hi = C;  // the first component of a group >= g
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (gs[mid] < g) lo = mid + 1; else hi = mid;
  }
  goff[g] = kHeaderBytes * (uint64_t)g + 16 * (uint64_t)lo;
}

// Every scene's record into `out`: thread i < C writes the i-th digest in (group, d0, d1) order (component
// perm[i], of group gs[i]) after the headers of groups 0..gs[i]; thread C + g writes scene g's header.
__global__ void record_write_kernel(const unsigned long long* __restrict__ d0, const unsigned long long* __restrict__ d1,
                                    const uint32_t* __restrict__ perm, const uint32_t* __restrict__ gs, uint32_t C, uint32_t G,
                                    const uint64_t* __restrict__ goff, uint8_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < C) {
    const uint32_t c = perm[i];
    *reinterpret_cast<ulonglong2*>(out + kHeaderBytes * ((uint64_t)gs[i] + 1) + 16 * (uint64_t)i) = make_ulonglong2(d0[c], d1[c]);
  } else if (i < C + G) {
    const uint32_t g = i - C;
    const uint64_t n = (goff[g + 1] - goff[g]) / 16 - 1;
    *reinterpret_cast<ulonglong2*>(out + goff[g]) = make_ulonglong2(kMagic, n);
  }
}

}  // namespace record
}  // namespace lfr
