// lfr_start.cuh — fixed images, kept and updated solutions and start points of a device-resident plan
// (lfr_plan_fix_images, lfr_plan_keep_solution, lfr_plan_update_solution, lfr_plan_start_from_solution;
// include/lfr_graph.h), over the node ids the plan keeps in HBM.
//
// A constant node is what a root is to every tier (lfr_setup.cuh: kept at its start value, no bounds, a
// block between two constant nodes dropped), so fixing images and keeping a solution only widen the mask
// the tiers read as `is_root`.  The start point is a sorted join: the SolutionFile's displacements keyed as the encoder keys
// nodes (image id << 32 | feature, lfr_join.h), radix-sorted stably so the last of a run of equal keys is
// the last occurrence, then one binary search per node.
#ifndef LFR_START_CUH_
#define LFR_START_CUH_

#include <cstdint>

namespace lfr {
namespace start {

// constant[v] = reference root OR node of a fixed image OR kept node; `fixed` (per image) and `kept` (per
// node) may each be NULL, for a plan never given that input
__global__ void constant_mask_kernel(const uint8_t* __restrict__ is_root, const uint32_t* __restrict__ node_image,
                                     const uint8_t* __restrict__ fixed, const uint8_t* __restrict__ kept, uint32_t N,
                                     uint8_t* __restrict__ constant) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < N) constant[v] = (is_root[v] || (fixed && fixed[node_image[v]]) || (kept && kept[v])) ? 1 : 0;
}

// key of displacement d: its Image message i = the last with img_ptr[i] <= d (img_ptr[0] = 0), keyed when
// that message is the one its scene image takes (image_id[i] != kNoImage)
__global__ void solution_key_kernel(const uint64_t* __restrict__ img_ptr, const uint32_t* __restrict__ image_id,
                                    uint32_t n_msgs, const uint32_t* __restrict__ feature_idx, uint32_t D,
                                    unsigned long long* __restrict__ key, uint32_t* __restrict__ idx) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  uint32_t lo = 0, hi = n_msgs;  // img_ptr[lo] <= d < img_ptr[hi]
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (img_ptr[mid] <= d) lo = mid; else hi = mid;
  }
  const uint32_t im = image_id[lo];
  key[d] = im == 0xffffffffu ? ~0ull : ((unsigned long long)im << 32 | feature_idx[d]);
  idx[d] = d;
}

// positions of node v from the last entry with its key (0 without one), into the start and working arrays;
// has_entry[v] (may be NULL) = whether it has one
__global__ void join_kernel(const uint32_t* __restrict__ node_image, const uint32_t* __restrict__ node_feat, uint32_t N,
                            const unsigned long long* __restrict__ key_s, const uint32_t* __restrict__ idx_s, uint32_t D,
                            const float* __restrict__ di, const float* __restrict__ dj, double* __restrict__ pos_init,
                            double* __restrict__ pos, unsigned long long* __restrict__ n_started,
                            uint8_t* __restrict__ has_entry) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  const unsigned long long k = (unsigned long long)node_image[v] << 32 | node_feat[v];
  uint32_t lo = 0, hi = D;  // upper bound: the first entry with a key > k
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (key_s[mid] <= k) lo = mid + 1; else hi = mid;
  }
  double a = 0.0, b = 0.0;
  const bool hit = lo > 0 && key_s[lo - 1] == k;
  if (hit) {
    const uint32_t e = idx_s[lo - 1];
    a = (double)di[e];
    b = (double)dj[e];
    atomicAdd(n_started, 1ull);
  }
  if (has_entry) has_entry[v] = hit ? 1 : 0;
  pos_init[2 * (size_t)v] = a;
  pos_init[2 * (size_t)v + 1] = b;
  pos[2 * (size_t)v] = a;
  pos[2 * (size_t)v + 1] = b;
}

// lfr_plan_update_solution: touched[comp[v]] = 1 for every node without an entry.  Reads are coalesced; the
// lanes of a warp that name the same component store once (the stores are idempotent across warps).
__global__ void touch_kernel(const uint8_t* __restrict__ has_entry, const uint32_t* __restrict__ comp, uint32_t N,
                             uint8_t* __restrict__ touched) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool miss = v < N && !has_entry[v];
  const unsigned active = __ballot_sync(0xffffffffu, miss);
  if (!miss) return;
  const uint32_t c = comp[v];
  const unsigned same = __match_any_sync(active, c);
  if ((uint32_t)(__ffs(same) - 1) == (threadIdx.x & 31u)) touched[c] = 1;
}

// lfr_plan_update_solution after the join and touch_kernel: held[v] (has_entry in, held out) = entry AND
// component not touched; a touched component's nodes start at 0 in the start and working arrays.
// n_held += the held nodes.
__global__ void update_kernel(const uint32_t* __restrict__ comp, const uint8_t* __restrict__ touched, uint32_t N,
                              uint8_t* __restrict__ held, double* __restrict__ pos_init, double* __restrict__ pos,
                              unsigned long long* __restrict__ n_held) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  bool h = false;
  if (v < N) {
    h = held[v] && !touched[comp[v]];
    held[v] = h ? 1 : 0;
    if (!h) {
      pos_init[2 * (size_t)v] = 0.0;
      pos_init[2 * (size_t)v + 1] = 0.0;
      pos[2 * (size_t)v] = 0.0;
      pos[2 * (size_t)v + 1] = 0.0;
    }
  }
  const unsigned n = __popc(__ballot_sync(0xffffffffu, h));
  if ((threadIdx.x & 31u) == 0 && n) atomicAdd(n_held, (unsigned long long)n);
}

// n_touched += the components with touched[c] != 0
__global__ void count_touched_kernel(const uint8_t* __restrict__ touched, uint32_t C, unsigned long long* __restrict__ n_touched) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned n = __popc(__ballot_sync(0xffffffffu, c < C && touched[c]));
  if ((threadIdx.x & 31u) == 0 && n) atomicAdd(n_touched, (unsigned long long)n);
}

}  // namespace start
}  // namespace lfr

#endif  // LFR_START_CUH_
