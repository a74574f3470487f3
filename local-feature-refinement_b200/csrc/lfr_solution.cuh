// lfr_solution.cuh — the SolutionFile of a device-resident plan encoded on the device, by every
// lfr_plan_encode_solution* call (include/lfr_graph.h).  The byte layout is lfr_wire_encode_solution's
// (lfr_wire.cc) on the output assembly of solve.cc:643-679: images in order of their lowest node index,
// within an image the displacements in ascending node index, di / dj the float32 of the fp64 positions,
// proto3 scalars omitted when their bit pattern is zero, minimal varints.
//
// One pipeline serves every call; they differ only in its inputs.  An image may have a group below G (without
// groups every image is in group 0 of G = 1): the images are ordered by (group, first node), so that each
// group's SolutionFile is one contiguous range of the output.  A group of G or more marks an image that is not
// written: its nodes count towards "> 0.5" but get no record.  With an earlier SolutionFile (G = 1), the
// output is lfr_wire_encode_solution_carried()'s: each scene image's nodes, then its carried entries (those no
// node refines), then the file's other winning Image messages in file order.  The file is decoded on the host
// (lfr_join.h); every entry is handled here.
//
//   init_images_kernel   key[img] = absent, which sorts after every present image of every group
//   first_node_kernel    key[img] = group << shift | lowest node of a written image; "> 0.5" per group
//   (sort images by key)  rank_kernel: rank of every present image, their count
// with a file:
//   solution_key_kernel (lfr_start.cuh) + stable radix sort    entries keyed (image << 32 | feature)
//   consume_kernel       the run of a node's key: the node has that entry, it is not carried
//   carry_flag_kernel    the last entry of each run (the winner), not consumed  (exclusive scan -> slot)
//   carry_compact_kernel carried entries in (image, feature) order, with their Image message
//   group2_flag_kernel   winning messages whose name has no node  (exclusive scan -> rank after the present)
//   group2_scatter_kernel  the message of each such output image; the output image count
// the records, node v < N and carried entry N + c:
//   record_key_kernel    output image rank of every record  (stable sort -> the output record order)
//   record_size_kernel   bytes of each record; img_ptr[r] = first slot of output image r  (exclusive scan -> rec_off)
//   image_size_kernel    body and size of each output image  (exclusive scan -> img_off; img_off[end] = total)
//   group_off_kernel     (G > 1) the byte offset of each group's first image
//   write_images_kernel / write_records_kernel   the bytes, one thread per image / per record
#pragma once

#include <cstdint>

namespace lfr {
namespace solution {

// SolutionFile.images = 1 (LEN); Image.image_name = 1 (LEN), fact = 2 (I32), displacements = 3 (LEN);
// Displacement.feature_idx = 1 (VARINT), di = 2 (I32), dj = 3 (I32)
constexpr uint8_t kTagImage = (1 << 3) | 2, kTagName = (1 << 3) | 2, kTagFact = (2 << 3) | 5, kTagDisp = (3 << 3) | 2;
constexpr uint8_t kTagFeat = (1 << 3) | 0, kTagDi = (2 << 3) | 5, kTagDj = (3 << 3) | 5;

constexpr uint32_t kNoImage = 0xffffffffu;

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

// one Displacement record: node src < N (the float32 of its fp64 position) or carried entry src - N (the
// file's float bits)
struct Record {
  uint32_t feat, di, dj;
};

struct Records {
  uint32_t N;
  const uint32_t* node_feat;
  const double* pos;
  const uint32_t* carried_e;  // per carried record: its entry in feat / di / dj
  const uint32_t* feat;
  const float* di;
  const float* dj;

  __device__ __forceinline__ Record operator()(uint32_t src) const {
    if (src < N) return Record{node_feat[src], f32_bits(pos[2 * (size_t)src]), f32_bits(pos[2 * (size_t)src + 1])};
    const uint32_t e = carried_e[src - N];
    return Record{feat[e], __float_as_uint(di[e]), __float_as_uint(dj[e])};
  }
};

// the header of output image r: the scene's name and fact for a present image, the file's Image message's
// after them
struct Header {
  const uint8_t* name;
  uint64_t len;
  uint32_t fact;
};

struct Headers {
  const uint32_t* n_present;
  const uint32_t* img_sorted;
  const uint8_t* names;
  const uint64_t* name_off;
  const float* fact;
  const uint32_t* g2_msg;  // per output image past the present ones: its message
  const uint8_t* msg_names;
  const uint64_t* msg_name_off;
  const float* msg_fact;

  __device__ __forceinline__ Header operator()(uint32_t r) const {
    const uint32_t np = *n_present;
    if (r < np) {
      const uint32_t img = img_sorted[r];
      return Header{names + name_off[img], name_off[img + 1] - name_off[img], __float_as_uint(fact[img])};
    }
    const uint32_t m = g2_msg[r - np];
    return Header{msg_names + msg_name_off[m], msg_name_off[m + 1] - msg_name_off[m], __float_as_uint(msg_fact[m])};
  }
};

__global__ void init_images_kernel(unsigned long long* key, uint32_t* iota, uint32_t n_images, unsigned long long absent) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_images) return;
  key[i] = absent;
  iota[i] = i;
}

// key[img] = group << shift | the image's lowest node, for a written image (one atomic per run of equal images
// in a warp, from its lowest lane, which holds the run's lowest node); n_outside[slot] += |pos| > 0.5 on either
// coordinate, where the slot is the image's group, or G for an image not written.  Without groups one atomic
// per block, otherwise one per run of equal slots in a warp.
__global__ void first_node_kernel(const uint32_t* node_image, const double* pos, uint32_t n, const uint32_t* group,
                                  uint32_t G, int shift, unsigned long long* key, unsigned long long* n_outside) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = v < n;
  const unsigned mask = __ballot_sync(0xffffffffu, live);
  uint32_t slot = 0;
  bool outside = false;
  if (live) {
    const uint32_t img = node_image[v];
    if (group) slot = min(group[img], G);
    const unsigned peers = __match_any_sync(mask, img);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1) && slot < G)
      atomicMin(key + img, (unsigned long long)slot << shift | v);
    outside = fabs(pos[2 * (size_t)v + 1]) > 0.5 || fabs(pos[2 * (size_t)v]) > 0.5;  // solve.cc:666-669
  }
  if (!group) {
    const int c = __syncthreads_count(outside);
    if (threadIdx.x == 0 && c) atomicAdd(n_outside, (unsigned long long)c);
  } else if (live) {
    const unsigned same = __match_any_sync(mask, slot), out = __ballot_sync(mask, outside) & same;
    if ((threadIdx.x & 31) == (unsigned)(__ffs(same) - 1) && out) atomicAdd(n_outside + slot, (unsigned long long)__popc(out));
  }
}

// from the images sorted by key: rank[img] of every present image and *n_present
__global__ void rank_kernel(const unsigned long long* key_sorted, const uint32_t* img_sorted, uint32_t n_images,
                            unsigned long long absent, uint32_t* rank, uint32_t* n_present) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_images || key_sorted[r] == absent) return;
  rank[img_sorted[r]] = r;
  if (r + 1 == n_images || key_sorted[r + 1] == absent) *n_present = r + 1;
}

// the last message lo with msg_ptr[lo] <= e (msg_ptr[0] = 0)
__device__ __forceinline__ uint32_t message_of(const uint64_t* msg_ptr, uint32_t n_msgs, uint32_t e) {
  uint32_t lo = 0, hi = n_msgs;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (msg_ptr[mid] <= e) lo = mid; else hi = mid;
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
__global__ void group2_flag_kernel(const uint32_t* __restrict__ msg_pid, uint32_t n_msgs, const unsigned long long* __restrict__ key,
                                   uint32_t n_images, unsigned long long absent, uint32_t* __restrict__ g2) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_msgs) return;
  if (i == n_msgs) {
    g2[n_msgs] = 0;
    return;
  }
  const uint32_t p = msg_pid[i];
  g2[i] = (p != kNoImage && (p >= n_images || key[p] == absent)) ? 1u : 0u;
}

// g2_msg[] = the message of each output image past the present ones; *n_out = the output images
__global__ void group2_scatter_kernel(const uint32_t* __restrict__ g2, const uint32_t* __restrict__ g2_off, uint32_t n_msgs,
                                      const uint32_t* __restrict__ n_present, uint32_t* __restrict__ g2_msg,
                                      uint32_t* __restrict__ n_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_msgs && g2[i]) g2_msg[g2_off[i]] = i;
  if (i == n_msgs) *n_out = *n_present + g2_off[n_msgs];
}

// record k < N is node k, record N + c carried entry c: key = the rank of its output image, or n_max (after
// every output image) for a node of an image that is not written
__global__ void record_key_kernel(const uint32_t* __restrict__ node_image, const uint32_t* __restrict__ group, uint32_t G,
                                  const uint32_t* __restrict__ rank, uint32_t N, const uint32_t* __restrict__ carried_msg,
                                  const uint32_t* __restrict__ msg_pid, const uint32_t* __restrict__ g2,
                                  const uint32_t* __restrict__ g2_off, const uint32_t* __restrict__ n_present, uint32_t n_rec,
                                  uint32_t n_max, uint32_t* __restrict__ key, uint32_t* __restrict__ iota) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_rec) return;
  uint32_t r;
  if (k < N) {
    const uint32_t img = node_image[k];
    r = (!group || group[img] < G) ? rank[img] : n_max;
  } else {
    const uint32_t m = carried_msg[k - N];
    r = g2[m] ? *n_present + g2_off[m] : rank[msg_pid[m]];
  }
  key[k] = r;
  iota[k] = k;
}

// rec_size[k] = the bytes of slot k's record (tag, 1-byte length — a Displacement body is at most 16 bytes —
// and body; 0 for a node that is not written), rec_size[n_rec] = 0; and img_ptr[r] = the first slot of output
// image r for r <= *n_out: slot k is the first of the images (key_s[k - 1], key_s[k]], those between having no
// record
__global__ void record_size_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ key_s, uint32_t n_rec,
                                   Records rec, const uint32_t* __restrict__ n_out, uint64_t* __restrict__ rec_size,
                                   uint32_t* __restrict__ img_ptr) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > n_rec) return;
  const uint32_t no = *n_out, r = k < n_rec ? key_s[k] : no;
  for (uint32_t i = k ? key_s[k - 1] + 1 : 0; i <= min(r, no); ++i) img_ptr[i] = k;
  if (k == n_rec) {
    rec_size[n_rec] = 0;
    return;
  }
  const Record x = rec(perm[k]);
  rec_size[k] = r < no ? 2 + disp_size(x.feat, x.di, x.dj) : 0;
}

// for r < *n_out: body[r] (name, fact, records) and img_size[r] = its whole Image record; 0 from there to
// n_max, so that the exclusive scan over n_max + 1 entries ends on the total
__global__ void image_size_kernel(Headers hdr, const uint32_t* __restrict__ img_ptr, const uint64_t* __restrict__ rec_off,
                                  const uint32_t* __restrict__ n_out, uint32_t n_max, uint64_t* __restrict__ body,
                                  uint64_t* __restrict__ img_size) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_max) return;
  if (r >= *n_out) {
    img_size[r] = 0;
    return;
  }
  const Header h = hdr(r);
  const uint64_t b = str_field_size(h.len) + f32_field_size(h.fact) + rec_off[img_ptr[r + 1]] - rec_off[img_ptr[r]];
  body[r] = b;
  img_size[r] = 1 + varint_size(b) + b;
}

// group_off[g] = the byte offset of group g's first image: img_off at the first rank whose group is g or more
// (an absent image's is G), so that every g <= G is written once
__global__ void group_off_kernel(const unsigned long long* key_sorted, uint32_t n_images, int shift, uint32_t G,
                                 const uint64_t* img_off, uint64_t* group_off) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_images) return;
  const uint32_t lo = r ? (uint32_t)(key_sorted[r - 1] >> shift) + 1 : 0, hi = r < n_images ? (uint32_t)(key_sorted[r] >> shift) : G;
  for (uint32_t g = lo; g <= hi; ++g) group_off[g] = img_off[r];
}

__global__ void write_images_kernel(Headers hdr, const uint64_t* __restrict__ body, const uint64_t* __restrict__ img_off,
                                    const uint32_t* __restrict__ n_out, uint32_t n_max, uint8_t* __restrict__ out) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_max || r >= *n_out) return;
  const Header h = hdr(r);
  uint8_t* p = out + img_off[r];
  *p++ = kTagImage;
  p = put_varint(p, body[r]);
  if (h.len) {
    *p++ = kTagName;
    p = put_varint(p, h.len);
    for (uint64_t i = 0; i < h.len; ++i) p[i] = h.name[i];
    p += h.len;
  }
  if (h.fact) {
    *p++ = kTagFact;
    put_fixed32(p, h.fact);
  }
}

// an image's records are the tail of its Image record: slot k's record ends the image's bytes minus the
// records after it
__global__ void write_records_kernel(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ key_s, uint32_t n_rec,
                                     Records rec, const uint32_t* __restrict__ img_ptr, const uint64_t* __restrict__ rec_off,
                                     const uint64_t* __restrict__ img_off, const uint32_t* __restrict__ n_out,
                                     uint8_t* __restrict__ out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_rec) return;
  const uint32_t r = key_s[k];
  if (r >= *n_out) return;
  const Record x = rec(perm[k]);
  uint8_t* p = out + (img_off[r + 1] - rec_off[img_ptr[r + 1]] + rec_off[k]);
  *p++ = kTagDisp;
  *p++ = (uint8_t)disp_size(x.feat, x.di, x.dj);
  if (x.feat) {
    *p++ = kTagFeat;
    p = put_varint(p, x.feat);
  }
  if (x.di) {
    *p++ = kTagDi;
    p = put_fixed32(p, x.di);
  }
  if (x.dj) {
    *p++ = kTagDj;
    put_fixed32(p, x.dj);
  }
}

}  // namespace solution
}  // namespace lfr
