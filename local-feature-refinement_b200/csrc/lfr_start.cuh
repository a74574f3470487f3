// lfr_start.cuh — fixed images, kept solutions and start points of a device-resident plan
// (lfr_plan_fix_images, lfr_plan_keep_solution, lfr_plan_start_from_solution; include/lfr_graph.h), over the
// node ids the plan keeps in HBM.
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

}  // namespace start
}  // namespace lfr

#endif  // LFR_START_CUH_
