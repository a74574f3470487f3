// lfr_carry.cuh — the SolutionFile of a device-resident plan merged with an earlier SolutionFile, encoded on
// the device (lfr_plan_encode_solution_carried, include/lfr_graph.h).  The bytes are those of
// lfr_wire_encode_solution_carried() (lfr_wire.cc) on the plan's host assembly: the scene images in order of
// their lowest node, each with its nodes' displacements and then its carried entries, then the file's
// other winning Image messages in file order.  The file is decoded on the host (lfr_join.h); every entry is
// handled here.  Records come from two sources: node v (slot source v < N, di / dj the float32 of the fp64
// positions, as lfr_solution.cuh writes them) and carried entry c (source N + c, the file's float bits).
//
//   (lfr_solution.cuh) init_images / first_node / sort / rank   present scene images, their ranks, "> 0.5"
//   (lfr_start.cuh) solution_key_kernel + stable radix sort     entries keyed (image << 32 | feature)
//   consume_kernel       the run of a node's key: the node has that entry, it is not carried
//   carry_flag_kernel    the last entry of each run (the winner), not consumed  (exclusive scan -> slot)
//   carry_compact_kernel carried entries in (image, feature) order, with their Image message
//   group2_flag_kernel   winning messages whose name has no node  (exclusive scan -> rank after the present)
//   group2_scatter_kernel  the message of each such output image
//   record_key_kernel    output image rank of every record  (stable sort -> the output record order)
//   record_size_kernel   bytes of each Displacement record  (exclusive scan -> rec_off)
//   image_size_kernel    records, body and size of each output image  (exclusive scan -> img_off)
//   write_images_kernel / write_records_kernel   the bytes, one thread per image / per record
#pragma once

#include <cstdint>

#include "lfr_solution.cuh"

namespace lfr {
namespace carry {

using solution::disp_size;
using solution::f32_bits;
using solution::f32_field_size;
using solution::put_fixed32;
using solution::put_varint;
using solution::str_field_size;
using solution::varint_size;

constexpr uint32_t kNoImage = 0xffffffffu;

// the last message lo with msg_ptr[lo] <= e (msg_ptr[0] = 0)
__device__ __forceinline__ uint32_t message_of(const uint64_t* msg_ptr, uint32_t n_msgs, uint32_t e) {
  uint32_t lo = 0, hi = n_msgs;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (msg_ptr[mid] <= e) lo = mid; else hi = mid;
  }
  return lo;
}

// the first slot in key_s[0, n) with a key >= r
__device__ __forceinline__ uint32_t lower_bound(const uint32_t* key_s, uint32_t n, uint32_t r) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (key_s[mid] < r) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// node v has the entry at the end of its key's run: mark it consumed (node keys are distinct)
__global__ void consume_kernel(const uint32_t* __restrict__ node_image, const uint32_t* __restrict__ node_feat, uint32_t N,
                               const unsigned long long* __restrict__ key_s, uint32_t D, uint8_t* __restrict__ consumed) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= N) return;
  const unsigned long long k = (unsigned long long)node_image[v] << 32 | node_feat[v];
  uint32_t lo = 0, hi = D;  // upper bound: the first entry with a key > k
  while (lo < hi) {
    const uint32_t mid = (lo + hi) / 2;
    if (key_s[mid] <= k) lo = mid + 1; else hi = mid;
  }
  if (lo > 0 && key_s[lo - 1] == k) consumed[lo - 1] = 1;
}

// flag[j] = 1 when sorted entry j is the last of its key's run (the effective entry of its name and
// feature) and no node consumed it; flag[D] = 0 so that the exclusive scan ends on the count
__global__ void carry_flag_kernel(const unsigned long long* __restrict__ key_s, const uint8_t* __restrict__ consumed,
                                  uint32_t D, uint32_t* __restrict__ flag) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j > D) return;
  if (j == D) {
    flag[D] = 0;
    return;
  }
  const unsigned long long k = key_s[j];
  flag[j] = (k != ~0ull && (j + 1 == D || key_s[j + 1] != k) && !consumed[j]) ? 1u : 0u;
}

__global__ void carry_compact_kernel(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ slot,
                                     const uint32_t* __restrict__ idx_s, const uint64_t* __restrict__ msg_ptr,
                                     uint32_t n_msgs, uint32_t D, uint32_t* __restrict__ carried_e,
                                     uint32_t* __restrict__ carried_msg) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D || !flag[j]) return;
  const uint32_t e = idx_s[j], c = slot[j];
  carried_e[c] = e;
  carried_msg[c] = message_of(msg_ptr, n_msgs, e);
}

// g2[i] = 1 for a winning message (msg_pid != kNoImage) whose name is not a present scene image: a name
// outside the scene (pid >= n_images) or a scene image without a node; g2[n_msgs] = 0
__global__ void group2_flag_kernel(const uint32_t* __restrict__ msg_pid, uint32_t n_msgs, const uint32_t* __restrict__ first,
                                   uint32_t n_images, uint32_t N, uint32_t* __restrict__ g2) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_msgs) return;
  if (i == n_msgs) {
    g2[n_msgs] = 0;
    return;
  }
  const uint32_t p = msg_pid[i];
  g2[i] = (p != kNoImage && (p >= n_images || first[p] >= N)) ? 1u : 0u;
}

__global__ void group2_scatter_kernel(const uint32_t* __restrict__ g2, const uint32_t* __restrict__ g2_off, uint32_t n_msgs,
                                      uint32_t* __restrict__ g2_msg) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_msgs && g2[i]) g2_msg[g2_off[i]] = i;
}

// record k < N is node k, record N + c carried entry c: key = the rank of its output image
__global__ void record_key_kernel(const uint32_t* __restrict__ node_image, const uint32_t* __restrict__ rank, uint32_t N,
                                  const uint32_t* __restrict__ carried_msg, const uint32_t* __restrict__ msg_pid,
                                  const uint32_t* __restrict__ g2, const uint32_t* __restrict__ g2_off,
                                  const uint32_t* __restrict__ n_present, uint32_t n_rec, uint32_t* __restrict__ key,
                                  uint32_t* __restrict__ iota) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_rec) return;
  uint32_t r;
  if (k < N) {
    r = rank[node_image[k]];
  } else {
    const uint32_t m = carried_msg[k - N];
    r = g2[m] ? *n_present + g2_off[m] : rank[msg_pid[m]];
  }
  key[k] = r;
  iota[k] = k;
}

struct Record {
  uint32_t feat, di, dj;
};

__device__ __forceinline__ Record record_of(uint32_t src, uint32_t N, const uint32_t* node_feat, const double* pos,
                                            const uint32_t* carried_e, const uint32_t* feat, const float* di, const float* dj) {
  if (src < N) return Record{node_feat[src], f32_bits(pos[2 * (size_t)src]), f32_bits(pos[2 * (size_t)src + 1])};
  const uint32_t e = carried_e[src - N];
  return Record{feat[e], __float_as_uint(di[e]), __float_as_uint(dj[e])};
}

// rec_size[k] = the bytes of slot k's record (tag, 1-byte length, body); rec_size[n_rec] = 0
__global__ void record_size_kernel(const uint32_t* __restrict__ perm, uint32_t n_rec, uint32_t N,
                                   const uint32_t* __restrict__ node_feat, const double* __restrict__ pos,
                                   const uint32_t* __restrict__ carried_e, const uint32_t* __restrict__ feat,
                                   const float* __restrict__ di, const float* __restrict__ dj, uint64_t* __restrict__ rec_size) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > n_rec) return;
  if (k == n_rec) {
    rec_size[n_rec] = 0;
    return;
  }
  const Record x = record_of(perm[k], N, node_feat, pos, carried_e, feat, di, dj);
  rec_size[k] = 2 + disp_size(x.feat, x.di, x.dj);
}

// the header of output image r: the scene's name and fact for a present image, the message's otherwise
struct Header {
  const uint8_t* name;
  uint64_t len;
  uint32_t fact;
};

__device__ __forceinline__ Header header_of(uint32_t r, uint32_t n_present, const uint32_t* img_sorted, const uint8_t* names,
                                            const uint64_t* name_off, const float* fact, const uint32_t* g2_msg,
                                            const uint8_t* msg_names, const uint64_t* msg_name_off, const float* msg_fact) {
  if (r < n_present) {
    const uint32_t img = img_sorted[r];
    return Header{names + name_off[img], name_off[img + 1] - name_off[img], __float_as_uint(fact[img])};
  }
  const uint32_t m = g2_msg[r - n_present];
  return Header{msg_names + msg_name_off[m], msg_name_off[m + 1] - msg_name_off[m], __float_as_uint(msg_fact[m])};
}

// for r < n_present + n_g2 (n_out): img_end[r] = its last record slot + 1, body[r], img_size[r] = its whole
// Image record; 0 up to n_max, so that the exclusive scan over n_max + 1 entries ends on the total
__global__ void image_size_kernel(const uint32_t* __restrict__ key_s, uint32_t n_rec, const uint64_t* __restrict__ rec_off,
                                  const uint32_t* __restrict__ n_present, const uint32_t* __restrict__ g2_off, uint32_t n_msgs,
                                  const uint32_t* __restrict__ img_sorted, const uint8_t* __restrict__ names,
                                  const uint64_t* __restrict__ name_off, const float* __restrict__ fact,
                                  const uint32_t* __restrict__ g2_msg, const uint8_t* __restrict__ msg_names,
                                  const uint64_t* __restrict__ msg_name_off, const float* __restrict__ msg_fact, uint32_t n_max,
                                  uint32_t* __restrict__ img_end, uint64_t* __restrict__ body, uint64_t* __restrict__ img_size) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_max) return;
  const uint32_t np = *n_present;
  if (r >= np + g2_off[n_msgs]) {
    img_size[r] = 0;
    return;
  }
  const uint32_t lo = lower_bound(key_s, n_rec, r), hi = lower_bound(key_s, n_rec, r + 1);
  const Header h = header_of(r, np, img_sorted, names, name_off, fact, g2_msg, msg_names, msg_name_off, msg_fact);
  const uint64_t b = str_field_size(h.len) + f32_field_size(h.fact) + rec_off[hi] - rec_off[lo];
  img_end[r] = hi;
  body[r] = b;
  img_size[r] = 1 + varint_size(b) + b;
}

__global__ void write_images_kernel(const uint32_t* __restrict__ n_present, const uint32_t* __restrict__ g2_off, uint32_t n_msgs,
                                    const uint32_t* __restrict__ img_sorted, const uint8_t* __restrict__ names,
                                    const uint64_t* __restrict__ name_off, const float* __restrict__ fact,
                                    const uint32_t* __restrict__ g2_msg, const uint8_t* __restrict__ msg_names,
                                    const uint64_t* __restrict__ msg_name_off, const float* __restrict__ msg_fact,
                                    const uint64_t* __restrict__ body, const uint64_t* __restrict__ img_off, uint32_t n_max,
                                    uint8_t* __restrict__ out) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t np = *n_present;
  if (r >= n_max || r >= np + g2_off[n_msgs]) return;
  const Header h = header_of(r, np, img_sorted, names, name_off, fact, g2_msg, msg_names, msg_name_off, msg_fact);
  uint8_t* p = out + img_off[r];
  *p++ = solution::kTagImage;
  p = put_varint(p, body[r]);
  if (h.len) {
    *p++ = solution::kTagName;
    p = put_varint(p, h.len);
    for (uint64_t i = 0; i < h.len; ++i) p[i] = h.name[i];
    p += h.len;
  }
  if (h.fact) {
    *p++ = solution::kTagFact;
    put_fixed32(p, h.fact);
  }
}

// an image's records are the tail of its Image record: slot k's record ends the image's bytes minus the
// records after it
__global__ void write_records_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ key_s, uint32_t n_rec,
                                     uint32_t N, const uint32_t* __restrict__ node_feat, const double* __restrict__ pos,
                                     const uint32_t* __restrict__ carried_e, const uint32_t* __restrict__ feat,
                                     const float* __restrict__ di, const float* __restrict__ dj,
                                     const uint32_t* __restrict__ img_end, const uint64_t* __restrict__ rec_off,
                                     const uint64_t* __restrict__ img_off, uint8_t* __restrict__ out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_rec) return;
  const uint32_t r = key_s[k];
  const Record x = record_of(perm[k], N, node_feat, pos, carried_e, feat, di, dj);
  uint8_t* p = out + (img_off[r + 1] - rec_off[img_end[r]] + rec_off[k]);
  *p++ = solution::kTagDisp;
  *p++ = (uint8_t)disp_size(x.feat, x.di, x.dj);
  if (x.feat) {
    *p++ = solution::kTagFeat;
    p = put_varint(p, x.feat);
  }
  if (x.di) {
    *p++ = solution::kTagDi;
    p = put_fixed32(p, x.di);
  }
  if (x.dj) {
    *p++ = solution::kTagDj;
    put_fixed32(p, x.dj);
  }
}

}  // namespace carry
}  // namespace lfr
