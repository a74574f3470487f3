// lfr_record.h — the problem record of a run (include/lfr_graph.h states it exactly, next to
// lfr_plan_update_solution_since): one 128-bit digest per component, the sum of SipHash-2-4 element
// hashes over its nodes and their kept out-edges, written sorted after an 8-byte magic and the count.
// One definition, included by the host library (lfr_wire.cc: lfr_host_problem_record and the host
// update since a record) and by the kernels (lfr_record.cuh), so both compute the same bits.
//
//   S(k, m)      SipHash-2-4 (Aumasson and Bernstein) with the 16-byte key k, m read as little-endian bytes
//   H(m)         (S(K0, m), S(K1, m)), K0 = "lfr problem rec0", K1 = "lfr problem rec1"
//   name id      H(exact name bytes)
//   node element [0x4e, id.0, id.1, feat | root << 32]                                       (32 bytes)
//   edge element [0x45, id(v).0, id(v).1, id(w).0, id(w).1, feat(v) | feat(w) << 32,
//                 kind | bits(sim) << 32, bits(flow[2i]) | bits(flow[2i+1]) << 32 (i = 0..8)]   (128 bytes)
//   digest(C)    (sum H(x).0, sum H(x).1) mod 2^64 over C's node elements and kept out-edge elements
//   record       "LFRPREC1", u64 C, C digests as (d0, d1) u64 pairs ascending in (d0, d1)
#pragma once
#include <cstdint>
#include <cstring>

#include "../../include/lfr.h"

#ifdef __CUDACC__
#define LFR_REC_HD __host__ __device__ __forceinline__
#else
#define LFR_REC_HD inline
#endif

namespace lfr {
namespace record {

// the two keys as little-endian u64 halves: "lfr prob" "lem rec0" / "lem rec1"
constexpr uint64_t kKeyLo = 0x626f72702072666cull;
constexpr uint64_t kKey0Hi = 0x30636572206d656cull;
constexpr uint64_t kKey1Hi = 0x31636572206d656cull;
constexpr uint64_t kMagic = 0x314345525052464cull;  // "LFRPREC1"
constexpr uint64_t kNodeTag = 0x4e, kEdgeTag = 0x45;
constexpr uint64_t kHeaderBytes = 16;

LFR_REC_HD uint64_t rotl(uint64_t x, int b) { return (x << b) | (x >> (64 - b)); }

// SipHash-2-4 of one key, fed 8-byte words
struct Sip {
  uint64_t v0, v1, v2, v3;
  LFR_REC_HD void init(uint64_t k0, uint64_t k1) {
    v0 = k0 ^ 0x736f6d6570736575ull;
    v1 = k1 ^ 0x646f72616e646f6dull;
    v2 = k0 ^ 0x6c7967656e657261ull;
    v3 = k1 ^ 0x7465646279746573ull;
  }
  LFR_REC_HD void round() {
    v0 += v1; v1 = rotl(v1, 13); v1 ^= v0; v0 = rotl(v0, 32);
    v2 += v3; v3 = rotl(v3, 16); v3 ^= v2;
    v0 += v3; v3 = rotl(v3, 21); v3 ^= v0;
    v2 += v1; v1 = rotl(v1, 17); v1 ^= v2; v2 = rotl(v2, 32);
  }
  LFR_REC_HD void absorb(uint64_t m) {
    v3 ^= m;
    round();
    round();
    v0 ^= m;
  }
  // the last block: the message length in its top byte over the 0..7 bytes that remain
  LFR_REC_HD uint64_t finish(uint64_t len, uint64_t tail) {
    absorb(len << 56 | tail);
    v2 ^= 0xff;
    round();
    round();
    round();
    round();
    return v0 ^ v1 ^ v2 ^ v3;
  }
};

// H over a message of whole words: both lanes in one pass
struct Lanes {
  Sip a, b;
  uint64_t n = 0;
  LFR_REC_HD Lanes() {
    a.init(kKeyLo, kKey0Hi);
    b.init(kKeyLo, kKey1Hi);
  }
  LFR_REC_HD void word(uint64_t m) {
    a.absorb(m);
    b.absorb(m);
    n += 8;
  }
  LFR_REC_HD void finish(uint64_t& h0, uint64_t& h1) {
    h0 = a.finish(n, 0);
    h1 = b.finish(n, 0);
  }
};

// H(bytes): the name id of an image
inline void hash_bytes(const uint8_t* p, uint64_t n, uint64_t& h0, uint64_t& h1) {
  Sip a, b;
  a.init(kKeyLo, kKey0Hi);
  b.init(kKeyLo, kKey1Hi);
  uint64_t i = 0;
  for (; i + 8 <= n; i += 8) {
    uint64_t m = 0;
    for (int k = 0; k < 8; ++k) m |= (uint64_t)p[i + k] << (8 * k);
    a.absorb(m);
    b.absorb(m);
  }
  uint64_t tail = 0;
  for (int k = 0; i + k < n; ++k) tail |= (uint64_t)p[i + k] << (8 * k);
  h0 = a.finish(n, tail);
  h1 = b.finish(n, tail);
}

// kind of the out-edge v -> w, as the solve classifies it (same track: Cauchy, same component: Tukey)
LFR_REC_HD uint32_t edge_kind(uint32_t track_v, uint32_t track_w, uint32_t comp_v, uint32_t comp_w) {
  return track_v == track_w ? LFR_EDGE_CAUCHY : (comp_v == comp_w ? LFR_EDGE_TUKEY : LFR_EDGE_SKIP);
}

LFR_REC_HD void node_element(uint64_t id0, uint64_t id1, uint32_t feat, bool root, uint64_t& h0, uint64_t& h1) {
  Lanes l;
  l.word(kNodeTag);
  l.word(id0);
  l.word(id1);
  l.word((uint64_t)feat | (uint64_t)(root ? 1u : 0u) << 32);
  l.finish(h0, h1);
}

// `w` = the 19 leading words of the lfr_edge record: flow[18], then sim
LFR_REC_HD void edge_element(uint64_t iv0, uint64_t iv1, uint64_t iw0, uint64_t iw1, uint32_t feat_v, uint32_t feat_w,
                             uint32_t kind, const uint32_t* w, uint64_t& h0, uint64_t& h1) {
  Lanes l;
  l.word(kEdgeTag);
  l.word(iv0);
  l.word(iv1);
  l.word(iw0);
  l.word(iw1);
  l.word((uint64_t)feat_v | (uint64_t)feat_w << 32);
  l.word((uint64_t)kind | (uint64_t)w[18] << 32);
  // constant trip count: nvcc unrolls it, and `w` stays in registers
  for (int i = 0; i < 9; ++i) l.word((uint64_t)w[2 * i] | (uint64_t)w[2 * i + 1] << 32);
  l.finish(h0, h1);
}

inline uint64_t record_bytes(uint64_t n_components) { return kHeaderBytes + 16 * n_components; }

inline uint64_t load_u64(const uint8_t* p) {
  uint64_t x = 0;
  for (int k = 0; k < 8; ++k) x |= (uint64_t)p[k] << (8 * k);
  return x;
}

inline void store_u64(uint8_t* p, uint64_t x) {
  for (int k = 0; k < 8; ++k) p[k] = (uint8_t)(x >> (8 * k));
}

// Whether `r` is a well-formed record: the magic, the length 16 + 16 C and the digests in ascending
// (d0, d1) order (equal pairs allowed).  *n_digests = C.
inline bool check(const uint8_t* r, uint64_t len, uint64_t* n_digests) {
  if (len < kHeaderBytes || !r || load_u64(r) != kMagic) return false;
  const uint64_t C = load_u64(r + 8);
  if (C > (len - kHeaderBytes) / 16 || record_bytes(C) != len) return false;
  for (uint64_t c = 1; c < C; ++c) {
    const uint8_t* a = r + kHeaderBytes + 16 * (c - 1);
    const uint64_t a0 = load_u64(a), a1 = load_u64(a + 8), b0 = load_u64(a + 16), b1 = load_u64(a + 24);
    if (b0 < a0 || (b0 == a0 && b1 < a1)) return false;
  }
  if (n_digests) *n_digests = C;
  return true;
}

}  // namespace record
}  // namespace lfr
