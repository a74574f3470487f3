// lfr_solution.cuh — the SolutionFile of a device-resident plan encoded on the device
// (lfr_plan_encode_solution, include/lfr_graph.h).  The byte layout is lfr_wire_encode_solution's
// (lfr_wire.cc) on the output assembly of solve.cc:643-679: images in order of their lowest node index,
// within an image the displacements in ascending node index, di / dj the float32 of the fp64 positions,
// proto3 scalars omitted when their bit pattern is zero, minimal varints.
//
//   first_node_kernel   first[img] = lowest node of the image; the "> 0.5" count
//   (sort images by first)  rank_kernel: rank of every present image, their count
//   node_key_kernel     key[v] = rank of v's image  (stable sort by key -> perm, the output node order)
//   record_size_kernel  bytes of each Displacement record; img_ptr[r] = first output slot of image r
//   (exclusive scan of the record sizes -> node_off)
//   image_size_kernel   body and record size of each image  (exclusive scan -> img_off; img_off[end] = total)
//   write_images_kernel / write_records_kernel   the bytes, one thread per image / per node
// With `written` (lfr_plan_encode_solution_images, --query_images) an image without the flag is absent: its
// nodes count towards "> 0.5" but sort after every written node and get no record.
//
// lfr_plan_encode_solution_groups (--additional_scenes) writes one SolutionFile per image group in the same
// pass: the images are sorted once by (group, first node) and ranked densely over the present ones, so every
// later kernel above runs unchanged and group g's bytes are one contiguous range of the output:
//   group_first_node_kernel   first[img]; the "> 0.5" count of every group
//   group_key_kernel          key[img] = group << 32 | first[img]  (sort -> img_s, by group then first node)
//   group_present_kernel      present[r] of the sorted images, present images per group
//   (exclusive scan of present -> dense ranks)  group_rank_kernel: rank, the present images in order
//   (node_key .. write_records as above; exclusive scan of the per-group counts -> first rank of each group)
//   group_off_kernel          group_off[g] = byte offset of the group's first image
#pragma once

#include <cstdint>

namespace lfr {
namespace solution {

// SolutionFile.images = 1 (LEN); Image.image_name = 1 (LEN), fact = 2 (I32), displacements = 3 (LEN);
// Displacement.feature_idx = 1 (VARINT), di = 2 (I32), dj = 3 (I32)
constexpr uint8_t kTagImage = (1 << 3) | 2, kTagName = (1 << 3) | 2, kTagFact = (2 << 3) | 5, kTagDisp = (3 << 3) | 2;
constexpr uint8_t kTagFeat = (1 << 3) | 0, kTagDi = (2 << 3) | 5, kTagDj = (3 << 3) | 5;

// (float)d as x86 cvtsd2ss rounds it (round to nearest, denormals kept, overflow to +-inf): a NaN keeps its
// sign and the top 23 bits of its payload, with the quiet bit set — spelled out rather than left to the
// device conversion's NaN handling
__device__ __forceinline__ uint32_t f32_bits(double d) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(d);
  if (d != d) return ((uint32_t)(b >> 32) & 0x80000000u) | 0x7FC00000u | (uint32_t)((b >> 29) & 0x7FFFFFu);
  return __float_as_uint(__double2float_rn(d));
}

__device__ __forceinline__ uint32_t varint_size(uint64_t v) {
  uint32_t n = 1;
  while (v >= 0x80) { v >>= 7; ++n; }
  return n;
}
__device__ __forceinline__ uint32_t u32_field_size(uint32_t v) { return v ? 1 + varint_size(v) : 0; }
__device__ __forceinline__ uint32_t f32_field_size(uint32_t bits) { return bits ? 5 : 0; }
__device__ __forceinline__ uint64_t str_field_size(uint64_t len) { return len ? 1 + varint_size(len) + len : 0; }

__device__ __forceinline__ uint8_t* put_varint(uint8_t* p, uint64_t v) {
  while (v >= 0x80) {
    *p++ = (uint8_t)(v | 0x80);
    v >>= 7;
  }
  *p++ = (uint8_t)v;
  return p;
}
__device__ __forceinline__ uint8_t* put_fixed32(uint8_t* p, uint32_t bits) {
  for (int i = 0; i < 4; ++i) p[i] = (uint8_t)(bits >> (8 * i));
  return p + 4;
}

__device__ __forceinline__ uint32_t disp_size(uint32_t feat, uint32_t di, uint32_t dj) {
  return u32_field_size(feat) + f32_field_size(di) + f32_field_size(dj);
}

// image headers: the size of the name and fact fields of image `img`
__device__ __forceinline__ uint64_t header_size(const uint64_t* name_off, const float* fact, uint32_t img) {
  return str_field_size(name_off[img + 1] - name_off[img]) + f32_field_size(__float_as_uint(fact[img]));
}

__global__ void init_images_kernel(uint32_t* first, uint32_t* iota, uint32_t n_images, uint32_t n_nodes) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_images) return;
  first[i] = n_nodes;  // "no node": sorts after every present image
  iota[i] = i;
}

// first[img] = min node index over the image's nodes (one atomic per run of equal images in a warp, from
// its lowest lane, which holds the run's lowest node); *n_outside += |pos| > 0.5 on either coordinate
__global__ void first_node_kernel(const uint32_t* node_image, const double* pos, uint32_t n, uint32_t* first,
                                  unsigned long long* n_outside, const uint8_t* written) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = v < n;
  const unsigned mask = __ballot_sync(0xffffffffu, live);
  bool outside = false;
  if (live) {
    const uint32_t img = node_image[v];
    const unsigned peers = __match_any_sync(mask, img);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1) && (!written || written[img])) atomicMin(first + img, v);
    outside = fabs(pos[2 * (size_t)v + 1]) > 0.5 || fabs(pos[2 * (size_t)v]) > 0.5;  // solve.cc:666-669
  }
  const int c = __syncthreads_count(outside);
  if (threadIdx.x == 0 && c) atomicAdd(n_outside, (unsigned long long)c);
}

// from the images sorted by first node: rank[img] of every present image and *n_present
__global__ void rank_kernel(const uint32_t* first_sorted, const uint32_t* img_sorted, uint32_t n_images,
                            uint32_t n_nodes, uint32_t* rank, uint32_t* n_present) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_images || first_sorted[r] >= n_nodes) return;
  rank[img_sorted[r]] = r;
  if (r + 1 == n_images || first_sorted[r + 1] >= n_nodes) *n_present = r + 1;
}

// key[v] = rank of v's image, or n_images (after every written image) for a node of an absent image;
// *n_written (with `written`) = the nodes of written images
__global__ void node_key_kernel(const uint32_t* node_image, const uint32_t* rank, uint32_t n, uint32_t* key,
                                uint32_t* iota, const uint8_t* written, uint32_t n_images, uint32_t* n_written) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  bool w = false;
  if (v < n) {
    const uint32_t img = node_image[v];
    w = !written || written[img];
    key[v] = w ? rank[img] : n_images;
    iota[v] = v;
  }
  if (written) {
    const int c = __syncthreads_count(w);
    if (threadIdx.x == 0 && c) atomicAdd(n_written, (uint32_t)c);
  }
}

// output slot k holds node perm[k] of the image of rank key_sorted[k]: its record's size (tag, 1-byte length —
// a Displacement body is at most 16 bytes — and body), and the image boundaries img_ptr[0..I]
__global__ void record_size_kernel(const uint32_t* perm, const uint32_t* key_sorted, const uint32_t* node_feat,
                                   const double* pos, uint32_t n, uint64_t* rec_size, uint32_t* img_ptr) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t v = perm[k], r = key_sorted[k];
  rec_size[k] = 2 + disp_size(node_feat[v], f32_bits(pos[2 * (size_t)v]), f32_bits(pos[2 * (size_t)v + 1]));
  if (k == 0 || key_sorted[k - 1] != r) img_ptr[r] = k;
  if (k + 1 == n) {
    img_ptr[r + 1] = n;
    rec_size[n] = 0;
  }
}

// body[r] (name, fact, records) and img_size[r] = its whole Image record; 0 past the present images, so
// that the exclusive scan over n_images + 1 entries ends on the total
__global__ void image_size_kernel(const uint32_t* img_sorted, const uint32_t* img_ptr, const uint64_t* node_off,
                                  const uint64_t* name_off, const float* fact, const uint32_t* n_present,
                                  uint32_t n_images, uint64_t* body, uint64_t* img_size) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_images) return;
  if (r >= *n_present) {
    img_size[r] = 0;
    return;
  }
  const uint64_t b = header_size(name_off, fact, img_sorted[r]) + node_off[img_ptr[r + 1]] - node_off[img_ptr[r]];
  body[r] = b;
  img_size[r] = 1 + varint_size(b) + b;
}

__global__ void write_images_kernel(const uint32_t* img_sorted, const uint64_t* body, const uint64_t* img_off,
                                    const uint8_t* names, const uint64_t* name_off, const float* fact,
                                    const uint32_t* n_present, uint8_t* out) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *n_present) return;
  const uint32_t img = img_sorted[r];
  uint8_t* p = out + img_off[r];
  *p++ = kTagImage;
  p = put_varint(p, body[r]);
  const uint64_t nl = name_off[img + 1] - name_off[img];
  if (nl) {
    *p++ = kTagName;
    p = put_varint(p, nl);
    const uint8_t* s = names + name_off[img];
    for (uint64_t i = 0; i < nl; ++i) p[i] = s[i];
    p += nl;
  }
  const uint32_t fb = __float_as_uint(fact[img]);
  if (fb) {
    *p++ = kTagFact;
    put_fixed32(p, fb);
  }
}

// an image's records are the tail of its Image record: slot k's record ends the image's bytes minus the
// records after it
__global__ void write_records_kernel(const uint32_t* perm, const uint32_t* key_sorted, const uint32_t* node_feat,
                                     const double* pos, const uint32_t* img_ptr, const uint64_t* node_off,
                                     const uint64_t* img_off, uint32_t n, uint8_t* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t v = perm[k], r = key_sorted[k];
  const uint32_t feat = node_feat[v];
  const uint32_t di = f32_bits(pos[2 * (size_t)v]), dj = f32_bits(pos[2 * (size_t)v + 1]);
  uint8_t* p = out + (img_off[r + 1] - node_off[img_ptr[r + 1]] + node_off[k]);
  *p++ = kTagDisp;
  *p++ = (uint8_t)disp_size(feat, di, dj);
  if (feat) {
    *p++ = kTagFeat;
    p = put_varint(p, feat);
  }
  if (di) {
    *p++ = kTagDi;
    p = put_fixed32(p, di);
  }
  if (dj) {
    *p++ = kTagDj;
    put_fixed32(p, dj);
  }
}

// first_node_kernel without `written`, the "> 0.5" count kept per group (one atomic per run of equal groups
// in a warp)
__global__ void group_first_node_kernel(const uint32_t* node_image, const double* pos, uint32_t n, const uint32_t* group,
                                        uint32_t* first, unsigned long long* n_outside) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = v < n;
  const unsigned mask = __ballot_sync(0xffffffffu, live);
  if (!live) return;
  const uint32_t img = node_image[v];
  const unsigned peers = __match_any_sync(mask, img);
  if ((threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicMin(first + img, v);
  const bool outside = fabs(pos[2 * (size_t)v + 1]) > 0.5 || fabs(pos[2 * (size_t)v]) > 0.5;  // solve.cc:666-669
  const uint32_t g = group[img];
  const unsigned same = __match_any_sync(mask, g), out = __ballot_sync(mask, outside) & same;
  if ((threadIdx.x & 31) == (unsigned)(__ffs(same) - 1) && out) atomicAdd(n_outside + g, (unsigned long long)__popc(out));
}

// an image without a node keeps first = n_nodes and sorts after its group's present images
__global__ void group_key_kernel(const uint32_t* first, const uint32_t* group, uint32_t n_images, unsigned long long* key) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_images) key[i] = (unsigned long long)group[i] << 32 | first[i];
}

// present[r] of the sorted images (present[n_images] = 0, so that the exclusive scan ends on their count) and
// the present images of every group
__global__ void group_present_kernel(const unsigned long long* key_sorted, uint32_t n_images, uint32_t n_nodes,
                                     uint32_t* present, uint32_t* group_count) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_images) return;
  const bool p = r < n_images && (uint32_t)key_sorted[r] < n_nodes;
  present[r] = p;
  if (p) atomicAdd(group_count + (uint32_t)(key_sorted[r] >> 32), 1u);
}

// rank[img] and img_dense[rank] of every present image, ranks dense in (group, first node) order; *n_present
__global__ void group_rank_kernel(const uint32_t* img_sorted, const uint32_t* present, const uint32_t* dense,
                                  uint32_t n_images, uint32_t* rank, uint32_t* img_dense, uint32_t* n_present) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) *n_present = dense[n_images];
  if (r >= n_images || !present[r]) return;
  rank[img_sorted[r]] = dense[r];
  img_dense[dense[r]] = img_sorted[r];
}

// group_off[g] = the byte offset of group g's first present image (its rank group_rank[g]); past the last
// present image the scan of the image sizes holds the total
__global__ void group_off_kernel(const uint32_t* group_rank, const uint64_t* img_off, uint32_t n_groups, uint64_t* group_off) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g <= n_groups) group_off[g] = img_off[group_rank[g]];
}

}  // namespace solution
}  // namespace lfr
