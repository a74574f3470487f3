// lfr_wire.cc — protobuf wire codec for types.proto (MatchingFile,
// SolutionFile) without libprotobuf.  Replaces the parse loop of
// solve.cc:426-480 and the writer of solve.cc:643-679.  Host code only.
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/lfr.h"
#include "../../include/lfr_wire.h"

namespace {

struct Reader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  bool done() const { return p >= end; }
  uint64_t varint() {
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
  uint32_t fixed32() {
    if (end - p < 4) { ok = false; return 0; }
    uint32_t v;
    std::memcpy(&v, p, 4);
    p += 4;
    return v;
  }
  float f32() {
    const uint32_t v = fixed32();
    float f;
    std::memcpy(&f, &v, 4);
    return f;
  }
  Reader sub() {  // length-delimited payload
    const uint64_t n = varint();
    if (!ok || n > (uint64_t)(end - p)) { ok = false; return Reader{p, p}; }
    Reader r{p, p + n};
    p += n;
    return r;
  }
  void skip(uint32_t wire_type) {
    switch (wire_type) {
      case 0: varint(); break;
      case 1: if (end - p < 8) ok = false; else p += 8; break;
      case 2: sub(); break;
      case 5: if (end - p < 4) ok = false; else p += 4; break;
      default: ok = false;
    }
  }
};

// Displacement { float di = 1; float dj = 2; }
bool read_disp(Reader r, float* out2) {
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
bool read_match(Reader r, lfr_wire_matches* o, uint64_t m) {
  uint32_t f1 = 0, f2 = 0;
  float sim = 0.f;
  int n1 = 0, n2 = 0;
  if (o) {
    std::memset(o->disp1 + 18 * m, 0, 18 * sizeof(float));
    std::memset(o->disp2 + 18 * m, 0, 18 * sizeof(float));
  }
  while (!r.done() && r.ok) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
    if (field == 1 && wt == 0) f1 = (uint32_t)r.varint();
    else if (field == 2 && wt == 0) f2 = (uint32_t)r.varint();
    else if (field == 3 && wt == 5) sim = r.f32();
    else if ((field == 4 || field == 5) && wt == 2) {
      int& n = field == 4 ? n1 : n2;
      float* dst = (o && n < 9) ? (field == 4 ? o->disp1 : o->disp2) + 18 * m + 2 * n : nullptr;
      // the form every writer of this schema emits for a displacement with two non-zero floats:
      // length 10, 0x0D <di>, 0x15 <dj> — taken without the generic field loop
      if (r.end - r.p >= 11 && r.p[0] == 10 && r.p[1] == 0x0D && r.p[6] == 0x15) {
        if (dst) {
          std::memcpy(dst, r.p + 2, 4);
          std::memcpy(dst + 1, r.p + 7, 4);
        }
        r.p += 11;
      } else {
        Reader d = r.sub();
        if (!r.ok) return false;
        if (!read_disp(d, dst)) return false;
      }
      ++n;
    } else r.skip(wt);
  }
  if (o) {
    o->feat1[m] = f1;
    o->feat2[m] = f2;
    o->sim[m] = sim;
  }
  return r.ok;
}

// ImagePair { string image_name1 = 1; float fact1 = 2; string image_name2 = 3;
//             float fact2 = 4; repeated Match matches = 5; }
// count_only: match payloads are skipped by their length (their contents are validated by the decode);
// match_off (header_only): the byte offset of every match's length prefix is recorded instead
bool read_pair(Reader r, const uint8_t* base, lfr_wire_matches* o, uint64_t pair, uint64_t* m, bool count_only = false,
               bool header_only = false, uint64_t* match_off = nullptr) {
  if (o) {
    o->fact1[pair] = o->fact2[pair] = 0.f;
    o->name1_off[pair] = o->name2_off[pair] = 0;
    o->name1_len[pair] = o->name2_len[pair] = 0;
  }
  while (!r.done() && r.ok) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
    if ((field == 1 || field == 3) && wt == 2) {
      Reader s = r.sub();
      if (!r.ok) return false;
      if (o) {
        if (field == 1) { o->name1_off[pair] = (uint64_t)(s.p - base); o->name1_len[pair] = (uint32_t)(s.end - s.p); }
        else { o->name2_off[pair] = (uint64_t)(s.p - base); o->name2_len[pair] = (uint32_t)(s.end - s.p); }
      }
    } else if (field == 2 && wt == 5) { const float f = r.f32(); if (o) o->fact1[pair] = f; }
    else if (field == 4 && wt == 5) { const float f = r.f32(); if (o) o->fact2[pair] = f; }
    else if (field == 5 && wt == 2) {
      const uint64_t at = (uint64_t)(r.p - base);
      Reader mm = r.sub();
      if (!r.ok) return false;
      if (match_off) {
        if (*m >= o->n_matches) return false;
        match_off[*m] = at;
      }
      if (count_only || header_only) {
        ++*m;
        continue;
      }
      if (o && *m >= o->n_matches) return false;
      if (!read_match(mm, o, *m)) return false;
      ++*m;
    } else r.skip(wt);
  }
  return r.ok;
}

// MatchingFile { repeated ImagePair image_pairs = 1; }
// Matches of one pair only (its header fields were taken by the serial walk): used by the workers.
bool read_pair_matches(Reader r, lfr_wire_matches* o, uint64_t m, uint64_t m_end) {
  while (!r.done() && r.ok) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
    if (field == 5 && wt == 2) {
      Reader mm = r.sub();
      if (!r.ok || m >= m_end) return false;
      if (!read_match(mm, o, m)) return false;
      ++m;
    } else r.skip(wt);
  }
  return r.ok && m == m_end;
}

// o == NULL: counts only.  match_off: the pair level of `o` and the match offsets only, no match decoded.
int walk_matching_file(const uint8_t* buf, uint64_t len, lfr_wire_matches* o, uint64_t* n_pairs,
                       uint64_t* n_matches, uint64_t* match_off = nullptr) {
  // serial walk over the pairs: header fields, match counts (match payloads skipped by length)
  Reader r{buf, buf + len};
  uint64_t pairs = 0, m = 0;
  std::vector<Reader> pair_payload;
  while (!r.done() && r.ok) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
    if (field == 1 && wt == 2) {
      Reader pr = r.sub();
      if (!r.ok) return LFR_EINVAL;
      if (o) {
        if (pairs >= o->n_pairs) return LFR_EINVAL;
        o->pair_ptr[pairs] = m;
        pair_payload.push_back(pr);
      }
      if (!read_pair(pr, buf, o, pairs, &m, /*count_only=*/o == nullptr, /*header_only=*/o != nullptr, match_off))
        return LFR_EINVAL;
      ++pairs;
    } else r.skip(wt);
  }
  if (!r.ok) return LFR_EINVAL;
  if (n_pairs) *n_pairs = pairs;
  if (n_matches) *n_matches = m;
  if (!o) return LFR_OK;
  if (m > o->n_matches) return LFR_EINVAL;
  o->pair_ptr[pairs] = m;
  if (match_off) return LFR_OK;
  // the matches of every pair, pairs dealt to worker threads (a pair's matches land at pair_ptr[pair]:
  // the output does not depend on the thread count)
  unsigned n_thr = 1;
  if (len >= (4u << 20) && pairs > 1) {
    const unsigned hw = std::thread::hardware_concurrency();
    n_thr = (unsigned)std::min<uint64_t>(std::min<uint64_t>(pairs, 8), hw ? hw : 1);
    if (const char* e = std::getenv("LFR_WIRE_THREADS")) n_thr = (unsigned)std::max(1, std::min(64, std::atoi(e)));
  }
  std::atomic<uint64_t> next{0};
  std::atomic<int> bad{0};
  auto work = [&] {
    for (;;) {
      const uint64_t p = next.fetch_add(1);
      if (p >= pairs || bad.load(std::memory_order_relaxed)) return;
      if (!read_pair_matches(pair_payload[p], o, o->pair_ptr[p], o->pair_ptr[p + 1])) bad.store(1);
    }
  };
  std::vector<std::thread> helpers;
  for (unsigned t = 1; t < n_thr; ++t) helpers.emplace_back(work);
  work();
  for (std::thread& h : helpers) h.join();
  return bad.load() ? LFR_EINVAL : LFR_OK;
}

// ---- encoder ----------------------------------------------------------------------
struct Writer {
  uint8_t* out;
  uint64_t cap;
  uint64_t n = 0;
  void byte(uint8_t b) {
    if (out && n < cap) out[n] = b;
    ++n;
  }
  void varint(uint64_t v) {
    while (v >= 0x80) {
      byte((uint8_t)(v | 0x80));
      v >>= 7;
    }
    byte((uint8_t)v);
  }
  void bytes(const uint8_t* p, uint64_t len) {
    if (out && n + len <= cap) std::memcpy(out + n, p, len);
    n += len;
  }
  void f32_field(uint32_t field, float f) {  // proto3: zero (bit pattern) is omitted
    uint32_t bits;
    std::memcpy(&bits, &f, 4);
    if (bits == 0) return;
    varint((field << 3) | 5);
    bytes((const uint8_t*)&bits, 4);
  }
  void u32_field(uint32_t field, uint32_t v) {
    if (v == 0) return;
    varint((field << 3) | 0);
    varint(v);
  }
  void str_field(uint32_t field, const uint8_t* p, uint64_t len) {
    if (len == 0) return;
    varint((field << 3) | 2);
    varint(len);
    bytes(p, len);
  }
};

inline int varint_size(uint64_t v) {
  int n = 1;
  while (v >= 0x80) { v >>= 7; ++n; }
  return n;
}
inline int f32_field_size(float f) {
  uint32_t bits;
  std::memcpy(&bits, &f, 4);
  return bits ? 5 : 0;
}
inline int u32_field_size(uint32_t v) { return v ? 1 + varint_size(v) : 0; }
inline uint64_t str_field_size(uint64_t len) { return len ? 1 + varint_size(len) + len : 0; }
inline int disp_size(const float* d) { return f32_field_size(d[0]) + f32_field_size(d[1]); }
inline int match_size(uint32_t f1, uint32_t f2, float sim, const float* d1, const float* d2) {
  int s = u32_field_size(f1) + u32_field_size(f2) + f32_field_size(sim);
  for (int g = 0; g < 9; ++g) s += 2 + disp_size(d1 + 2 * g);  // tag + 1-byte length (payload <= 10)
  for (int g = 0; g < 9; ++g) s += 2 + disp_size(d2 + 2 * g);
  return s;
}

}  // namespace

extern "C" {

int lfr_wire_scan_matches(const uint8_t* buf, uint64_t len, uint64_t* n_pairs, uint64_t* n_matches) {
  if (!buf && len) return LFR_EINVAL;
  return walk_matching_file(buf, len, nullptr, n_pairs, n_matches);
}

int lfr_wire_decode_matches(const uint8_t* buf, uint64_t len, lfr_wire_matches* out) {
  if ((!buf && len) || !out) return LFR_EINVAL;
  uint64_t np = 0, nm = 0;
  const int rc = walk_matching_file(buf, len, out, &np, &nm);
  if (rc) return rc;
  if (np != out->n_pairs || nm != out->n_matches) return LFR_EINVAL;
  return LFR_OK;
}

int lfr_wire_walk_matches(const uint8_t* buf, uint64_t len, lfr_wire_matches* out, uint64_t* match_off) {
  if ((!buf && len) || !out || (!match_off && out->n_matches)) return LFR_EINVAL;
  uint64_t np = 0, nm = 0;
  const int rc = walk_matching_file(buf, len, out, &np, &nm, match_off);
  if (rc) return rc;
  if (np != out->n_pairs || nm != out->n_matches) return LFR_EINVAL;
  return LFR_OK;
}

int64_t lfr_wire_encode_matches(uint64_t n_pairs, const uint64_t* pair_ptr, const uint32_t* pair_name1,
                                const uint32_t* pair_name2, const float* fact1, const float* fact2,
                                const uint8_t* names, const uint64_t* name_off, const uint32_t* feat1,
                                const uint32_t* feat2, const float* sim, const float* disp1,
                                const float* disp2, uint8_t* out, uint64_t cap) {
  Writer w{out, cap};
  for (uint64_t p = 0; p < n_pairs; ++p) {
    const uint64_t l1 = name_off[pair_name1[p] + 1] - name_off[pair_name1[p]];
    const uint64_t l2 = name_off[pair_name2[p] + 1] - name_off[pair_name2[p]];
    uint64_t body = str_field_size(l1) + f32_field_size(fact1[p]) + str_field_size(l2) + f32_field_size(fact2[p]);
    for (uint64_t m = pair_ptr[p]; m < pair_ptr[p + 1]; ++m) {
      const int ms = match_size(feat1[m], feat2[m], sim[m], disp1 + 18 * m, disp2 + 18 * m);
      body += 1 + varint_size(ms) + ms;
    }
    w.varint((1 << 3) | 2);
    w.varint(body);
    w.str_field(1, names + name_off[pair_name1[p]], l1);
    w.f32_field(2, fact1[p]);
    w.str_field(3, names + name_off[pair_name2[p]], l2);
    w.f32_field(4, fact2[p]);
    for (uint64_t m = pair_ptr[p]; m < pair_ptr[p + 1]; ++m) {
      const float* d1 = disp1 + 18 * m;
      const float* d2 = disp2 + 18 * m;
      w.varint((5 << 3) | 2);
      w.varint(match_size(feat1[m], feat2[m], sim[m], d1, d2));
      w.u32_field(1, feat1[m]);
      w.u32_field(2, feat2[m]);
      w.f32_field(3, sim[m]);
      for (int g = 0; g < 9; ++g) {
        w.varint((4 << 3) | 2);
        w.varint(disp_size(d1 + 2 * g));
        w.f32_field(1, d1[2 * g]);
        w.f32_field(2, d1[2 * g + 1]);
      }
      for (int g = 0; g < 9; ++g) {
        w.varint((5 << 3) | 2);
        w.varint(disp_size(d2 + 2 * g));
        w.f32_field(1, d2[2 * g]);
        w.f32_field(2, d2[2 * g + 1]);
      }
    }
  }
  return (int64_t)w.n;
}

int64_t lfr_wire_encode_solution(uint64_t n_images, const uint64_t* img_ptr, const uint8_t* names,
                                 const uint64_t* name_off, const float* fact, const uint32_t* feature_idx,
                                 const float* di, const float* dj, uint8_t* out, uint64_t cap) {
  // SolutionFile { repeated Image images = 1; }
  // Image { string image_name = 1; float fact = 2; repeated Displacement displacements = 3; }
  // Displacement { uint32 feature_idx = 1; float di = 2; float dj = 3; }
  Writer w{out, cap};
  for (uint64_t i = 0; i < n_images; ++i) {
    const uint64_t nl = name_off[i + 1] - name_off[i];
    uint64_t body = str_field_size(nl) + f32_field_size(fact[i]);
    for (uint64_t k = img_ptr[i]; k < img_ptr[i + 1]; ++k)
      body += 2 + u32_field_size(feature_idx[k]) + f32_field_size(di[k]) + f32_field_size(dj[k]);
    w.varint((1 << 3) | 2);
    w.varint(body);
    w.str_field(1, names + name_off[i], nl);
    w.f32_field(2, fact[i]);
    for (uint64_t k = img_ptr[i]; k < img_ptr[i + 1]; ++k) {
      w.varint((3 << 3) | 2);
      w.varint(u32_field_size(feature_idx[k]) + f32_field_size(di[k]) + f32_field_size(dj[k]));
      w.u32_field(1, feature_idx[k]);
      w.f32_field(2, di[k]);
      w.f32_field(3, dj[k]);
    }
  }
  return (int64_t)w.n;
}

int lfr_wire_decode_solution(const uint8_t* buf, uint64_t len, uint64_t* n_images, uint64_t* n_disp,
                             uint64_t* img_ptr, uint64_t* name_off, uint32_t* name_len, float* fact,
                             uint32_t* feature_idx, float* di, float* dj) {
  if (!buf && len) return LFR_EINVAL;
  Reader r{buf, buf + len};
  uint64_t ni = 0, nd = 0;
  while (!r.done() && r.ok) {
    const uint64_t tag = r.varint();
    const uint32_t field = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
    if (field == 1 && wt == 2) {
      Reader im = r.sub();
      if (!r.ok) return LFR_EINVAL;
      if (img_ptr) img_ptr[ni] = nd;
      if (name_off) { name_off[ni] = 0; name_len[ni] = 0; }
      if (fact) fact[ni] = 0.f;
      while (!im.done() && im.ok) {
        const uint64_t t2 = im.varint();
        const uint32_t f2 = (uint32_t)(t2 >> 3), w2 = (uint32_t)(t2 & 7);
        if (f2 == 1 && w2 == 2) {
          Reader s = im.sub();
          if (!im.ok) return LFR_EINVAL;
          if (name_off) { name_off[ni] = (uint64_t)(s.p - buf); name_len[ni] = (uint32_t)(s.end - s.p); }
        } else if (f2 == 2 && w2 == 5) { const float f = im.f32(); if (fact) fact[ni] = f; }
        else if (f2 == 3 && w2 == 2) {
          Reader d = im.sub();
          if (!im.ok) return LFR_EINVAL;
          uint32_t fi = 0;
          float a = 0.f, b = 0.f;
          while (!d.done() && d.ok) {
            const uint64_t t3 = d.varint();
            const uint32_t f3 = (uint32_t)(t3 >> 3), w3 = (uint32_t)(t3 & 7);
            if (f3 == 1 && w3 == 0) fi = (uint32_t)d.varint();
            else if (f3 == 2 && w3 == 5) a = d.f32();
            else if (f3 == 3 && w3 == 5) b = d.f32();
            else d.skip(w3);
          }
          if (!d.ok) return LFR_EINVAL;
          if (feature_idx) { feature_idx[nd] = fi; di[nd] = a; dj[nd] = b; }
          ++nd;
        } else im.skip(w2);
      }
      if (!im.ok) return LFR_EINVAL;
      ++ni;
    } else r.skip(wt);
  }
  if (!r.ok) return LFR_EINVAL;
  if (img_ptr) img_ptr[ni] = nd;
  if (n_images) *n_images = ni;
  if (n_disp) *n_disp = nd;
  return LFR_OK;
}

}  // extern "C"
