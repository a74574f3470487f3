// lfr_wire.cuh — the Match messages of a MatchingFile decoded on the device (lfr_plan_create_from_wire,
// include/lfr_graph.h).  One thread per match: it reads the match's length prefix at the offset the host
// walk recorded (lfr_wire_walk_matches) and decodes the payload straight into the graph stage's flat
// arrays at the match's global index.  The semantics are those of read_match / read_disp in lfr_wire.cc,
// field for field; every read is bounds-checked against its own message, and a malformed match sets
// *err instead of trapping.
#pragma once

#include <cstdint>

namespace lfr {
namespace wire {

struct DevReader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok;
  __device__ __forceinline__ bool done() const { return p >= end; }
  __device__ __forceinline__ uint64_t varint() {  // at most 10 bytes, as Reader::varint
    uint64_t v = 0;
    for (int shift = 0; shift < 64; shift += 7) {
      if (p >= end) { ok = false; return 0; }
      const uint8_t b = *p++;
      v |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
    }
    ok = false;
    return 0;
  }
  __device__ __forceinline__ uint32_t fixed32() {
    if (end - p < 4) { ok = false; return 0; }
    const uint32_t v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
    p += 4;
    return v;
  }
  __device__ __forceinline__ float f32() { return __uint_as_float(fixed32()); }
  __device__ __forceinline__ DevReader sub() {  // length-delimited payload
    const uint64_t n = varint();
    if (!ok || n > (uint64_t)(end - p)) { ok = false; return DevReader{p, p, true}; }
    DevReader r{p, p + n, true};
    p += n;
    return r;
  }
  __device__ __forceinline__ void skip(uint32_t wire_type) {
    switch (wire_type) {
      case 0: varint(); break;
      case 1: if (end - p < 8) ok = false; else p += 8; break;
      case 2: sub(); break;
      case 5: if (end - p < 4) ok = false; else p += 4; break;
      default: ok = false;
    }
  }
};

// Displacement { float di = 1; float dj = 2; } -> out2 (NULL: parsed and ignored, past the 9th entry)
__device__ __forceinline__ bool read_disp(DevReader r, float* out2) {
  float di = 0.f, dj = 0.f;
  while (!r.done() && r.ok) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
    if (field == 1 && wt == 5) di = r.f32();
    else if (field == 2 && wt == 5) dj = r.f32();
    else r.skip(wt);
  }
  if (out2) { out2[0] = di; out2[1] = dj; }
  return r.ok;
}

// Match { uint32 feature_idx1 = 1; uint32 feature_idx2 = 2; float similarity = 3;
//         repeated Displacement disp1 = 4; repeated Displacement disp2 = 5; }
// disp1 / disp2 rows must be zero on entry (missing entries stay 0).
__device__ __forceinline__ bool read_match(DevReader r, uint64_t m, uint32_t* feat1, uint32_t* feat2, float* sim,
                                           float* disp1, float* disp2) {
  uint32_t f1 = 0, f2 = 0;
  float s = 0.f;
  int n1 = 0, n2 = 0;
  while (!r.done() && r.ok) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
    if (field == 1 && wt == 0) f1 = (uint32_t)r.varint();
    else if (field == 2 && wt == 0) f2 = (uint32_t)r.varint();
    else if (field == 3 && wt == 5) s = r.f32();
    else if ((field == 4 || field == 5) && wt == 2) {
      int& n = field == 4 ? n1 : n2;
      float* dst = n < 9 ? (field == 4 ? disp1 : disp2) + 18 * m + 2 * n : nullptr;
      // speed path for the form every writer emits for two non-zero floats: length 10, 0x0D <di>, 0x15 <dj>
      if (r.end - r.p >= 11 && r.p[0] == 10 && r.p[1] == 0x0D && r.p[6] == 0x15) {
        DevReader d{r.p + 2, r.p + 11, true};
        const float di = d.f32();
        d.p += 1;
        const float dj = d.f32();
        if (dst) { dst[0] = di; dst[1] = dj; }
        r.p += 11;
      } else {
        DevReader d = r.sub();
        if (!r.ok) return false;
        if (!read_disp(d, dst)) return false;
      }
      ++n;
    } else r.skip(wt);
  }
  feat1[m] = f1;
  feat2[m] = f2;
  sim[m] = s;
  return r.ok;
}

// Match i of one part: its length prefix at buf[off[i]], decoded to global index m0 + i.
__global__ void __launch_bounds__(256) decode_matches_kernel(const uint8_t* __restrict__ buf, uint64_t len,
                                                             const uint64_t* __restrict__ off, uint64_t n, uint64_t m0,
                                                             uint32_t* feat1, uint32_t* feat2, float* sim, float* disp1,
                                                             float* disp2, int* err) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t o = off[i];
  if (o >= len) { *err = 1; return; }
  DevReader r{buf + o, buf + len, true};
  const DevReader mm = r.sub();
  if (!r.ok || !read_match(mm, m0 + i, feat1, feat2, sim, disp1, disp2)) *err = 1;
}

}  // namespace wire
}  // namespace lfr
