// lfr_wire.cc — protobuf wire codec for types.proto (MatchingFile,
// SolutionFile) without libprotobuf.  Replaces the parse loop of
// solve.cc:426-480 and the writer of solve.cc:643-679.  Host code only.
#include <algorithm>
#include <array>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <unordered_set>
#include <vector>

#include "../../include/lfr.h"
#include "../../include/lfr_host.h"
#include "../../include/lfr_wire.h"
#include "lfr_join.h"
#include "lfr_record.h"

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

int lfr_wire_join_solution(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names,
                           const uint64_t* name_off, uint32_t n_nodes, const uint32_t* node_image,
                           const uint32_t* node_feat, double* positions, uint64_t* n_started) {
  return lfr::join::join_nodes(buf, len, n_images, names, name_off, n_nodes, node_image, node_feat, positions, nullptr,
                               n_started);
}

int lfr_wire_join_solution_entries(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names,
                                   const uint64_t* name_off, uint32_t n_nodes, const uint32_t* node_image,
                                   const uint32_t* node_feat, double* positions, uint64_t* n_started, uint8_t* has_entry) {
  if (n_nodes && !has_entry) return LFR_EINVAL;
  return lfr::join::join_nodes(buf, len, n_images, names, name_off, n_nodes, node_image, node_feat, positions, has_entry,
                               n_started);
}

int lfr_wire_update_solution(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names,
                             const uint64_t* name_off, uint32_t n_nodes, const uint32_t* node_image,
                             const uint32_t* node_feat, const uint32_t* node_comp, uint32_t n_components,
                             double* positions, uint8_t* held, uint64_t* n_held, uint32_t* n_touched) {
  return lfr::join::update_nodes(buf, len, n_images, names, name_off, n_nodes, node_image, node_feat, node_comp,
                                 n_components, positions, held, n_held, n_touched);
}

namespace {

// The graph arrays the "unchanged" test reads (lfr_problem's plus the node ids)
struct Graph {
  uint32_t N = 0;
  const uint32_t *row_ptr, *track, *comp, *node_image, *node_feat;
  const uint8_t* is_root;
  const lfr_edge* edges;
};

// kept out-edge of node v (solve.cc:105-125: same track -> Cauchy, same component -> Tukey, else skipped)
uint32_t edge_kind(const Graph& g, uint32_t v, uint32_t w) {
  if (g.track[v] == g.track[w]) return LFR_EDGE_CAUCHY;
  return g.comp[v] == g.comp[w] ? LFR_EDGE_TUKEY : LFR_EDGE_SKIP;
}

// {destination in this run's node ids, kind, bits of the 18 flow floats and of sim}
using EdgeRec = std::array<uint32_t, 21>;

void kept_edges(const Graph& g, uint32_t v, const uint32_t* to_cur, std::vector<EdgeRec>& out) {
  out.clear();
  for (uint32_t e = g.row_ptr[v]; e < g.row_ptr[v + 1]; ++e) {
    const uint32_t w = g.edges[e].dst, kind = edge_kind(g, v, w);
    if (kind == LFR_EDGE_SKIP) continue;
    EdgeRec r;
    r[0] = to_cur ? to_cur[w] : w;
    r[1] = kind;
    std::memcpy(&r[2], &g.edges[e], 19 * sizeof(uint32_t));  // flow[18], sim
    out.push_back(r);
  }
  std::sort(out.begin(), out.end());
}

// changed[c] = 1 for every component c of `cur` that fails the "unchanged" test against `prev`
// (include/lfr_host.h); prev's image ids are mapped by `map`.  Returns the count.
uint32_t changed_components(const Graph& cur, uint32_t C, const Graph& prev, uint32_t prev_C, const std::vector<uint32_t>& map,
                            uint8_t* changed) {
  constexpr uint32_t kNone = 0xffffffffu;
  std::unordered_map<uint64_t, uint32_t> prev_of;
  prev_of.reserve(prev.N);
  for (uint32_t u = 0; u < prev.N; ++u) prev_of.emplace(lfr::join::node_key(map[prev.node_image[u]], prev.node_feat[u]), u);
  std::vector<uint32_t> m(cur.N, kNone), inv(prev.N, kNone), pc_of(C, kNone), size(C, 0), prev_size(prev_C, 0);
  std::fill(changed, changed + C, 0);
  for (uint32_t v = 0; v < cur.N; ++v) {
    const uint32_t c = cur.comp[v];
    ++size[c];
    const auto it = prev_of.find(lfr::join::node_key(cur.node_image[v], cur.node_feat[v]));
    if (it == prev_of.end()) {
      changed[c] = 1;
      continue;
    }
    const uint32_t u = it->second, pc = prev.comp[u];
    m[v] = u;
    inv[u] = v;
    if ((cur.is_root[v] != 0) != (prev.is_root[u] != 0)) changed[c] = 1;
    if (pc_of[c] == kNone) pc_of[c] = pc;
    else if (pc_of[c] != pc) changed[c] = 1;
  }
  for (uint32_t u = 0; u < prev.N; ++u) ++prev_size[prev.comp[u]];
  for (uint32_t c = 0; c < C; ++c)
    if (!changed[c] && (pc_of[c] == kNone || size[c] != prev_size[pc_of[c]])) changed[c] = 1;
  std::vector<EdgeRec> a, b;
  for (uint32_t v = 0; v < cur.N; ++v) {
    if (changed[cur.comp[v]]) continue;
    kept_edges(cur, v, nullptr, a);
    kept_edges(prev, m[v], inv.data(), b);
    if (a != b) changed[cur.comp[v]] = 1;
  }
  return (uint32_t)std::count(changed, changed + C, (uint8_t)1);
}

}  // namespace

int lfr_wire_update_solution_since(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names,
                                   const uint64_t* name_off, const lfr_problem* p, const uint32_t* node_image,
                                   const uint32_t* node_feat, const lfr_host_input* previous, const uint8_t* prev_names,
                                   const uint64_t* prev_name_off, double* positions, uint8_t* held, uint64_t* n_held,
                                   uint32_t* n_touched, uint32_t* n_changed) {
  if (!p || !previous) return LFR_EINVAL;
  const uint32_t N = p->n_nodes, C = p->n_components;
  if (N && (!p->row_ptr || !p->track || !p->comp || !p->is_root || !node_image || !node_feat)) return LFR_EINVAL;
  if (N && (p->row_ptr[N] != p->n_edges || (p->n_edges && !p->edges))) return LFR_EINVAL;
  for (uint32_t v = 0; v < N; ++v)
    if (p->comp[v] >= C || node_image[v] >= n_images) return LFR_EINVAL;
  for (uint64_t e = 0; e < p->n_edges; ++e)
    if (p->edges[e].dst >= N) return LFR_EINVAL;
  std::vector<uint32_t> map;
  if (lfr::join::map_previous_images(n_images, names, name_off, previous->n_images, prev_names, prev_name_off, map) != LFR_OK)
    return LFR_EINVAL;
  // the earlier run: the graph stage over every pair of the earlier file, no image banned
  lfr_host_input in = *previous;
  in.pair_skip = nullptr;
  in.edges_out = nullptr;
  in.edges_out_capacity = 0;
  lfr_host_stage* hs = nullptr;
  lfr_host_sizes sz;
  const int rc = lfr_host_stage_create(&in, &hs, &sz);
  if (rc != LFR_OK) return rc;
  const uint32_t M = sz.n_nodes;
  std::vector<uint32_t> row_ptr((size_t)M + 1, 0), track(M), comp(M), node_image_b(M), node_feat_b(M);
  std::vector<uint8_t> is_root(M);
  std::vector<lfr_edge> edges(sz.n_edges);
  const int rc2 = lfr_host_stage_export(hs, row_ptr.data(), edges.data(), track.data(), comp.data(), is_root.data(), nullptr,
                                        nullptr, nullptr, node_image_b.data(), node_feat_b.data());
  lfr_host_stage_destroy(hs);
  if (rc2 != LFR_OK) return rc2;
  Graph cur{N, p->row_ptr, p->track, p->comp, node_image, node_feat, p->is_root, p->edges};
  Graph prev{M, row_ptr.data(), track.data(), comp.data(), node_image_b.data(), node_feat_b.data(), is_root.data(), edges.data()};
  std::vector<uint8_t> changed(C, 0);
  const uint32_t nc = changed_components(cur, C, prev, sz.n_components, map, changed.data());
  const int rc3 = lfr::join::update_nodes(buf, len, n_images, names, name_off, N, node_image, node_feat, p->comp, C,
                                          positions, held, n_held, n_touched, changed.data());
  if (rc3 == LFR_OK && n_changed) *n_changed = nc;
  return rc3;
}

namespace {

using Digest = std::pair<uint64_t, uint64_t>;

// The checks of lfr_host_problem_record(): a problem whose arrays are consistent, node ids within the names
bool record_input_ok(const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat, uint32_t n_images,
                     const uint8_t* names, const uint64_t* name_off) {
  if (!p) return false;
  const uint32_t N = p->n_nodes, C = p->n_components;
  if (N && (!p->row_ptr || !p->track || !p->comp || !p->is_root || !node_image || !node_feat)) return false;
  if (N && (p->row_ptr[0] != 0 || p->row_ptr[N] != p->n_edges || (p->n_edges && !p->edges))) return false;
  if (!N && p->n_edges) return false;
  for (uint32_t v = 0; v < N; ++v)
    if (p->comp[v] >= C || node_image[v] >= n_images || p->row_ptr[v + 1] < p->row_ptr[v]) return false;
  for (uint64_t e = 0; e < p->n_edges; ++e)
    if (p->edges[e].dst >= N) return false;
  if (n_images && !name_off) return false;
  for (uint32_t k = 0; k < n_images; ++k)
    if (name_off[k + 1] < name_off[k]) return false;
  return !(n_images && name_off[n_images] && !names);
}

// digest[c] of every component c of `p` (include/lfr_graph.h; lfr_record.h has the elements).  Components
// are dealt to helper threads in blocks; each digest is one thread's exact sum, so the result does not
// depend on the thread count (LFR_HOST_THREADS overrides it).
std::vector<Digest> component_digests(const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat,
                                      uint32_t n_images, const uint8_t* names, const uint64_t* name_off) {
  namespace rec = lfr::record;
  const uint32_t N = p->n_nodes, C = p->n_components;
  std::vector<Digest> id(n_images);
  for (uint32_t k = 0; k < n_images; ++k)
    rec::hash_bytes(names + name_off[k], name_off[k + 1] - name_off[k], id[k].first, id[k].second);
  std::vector<uint32_t> start((size_t)C + 1, 0), order(N);  // nodes by component
  for (uint32_t v = 0; v < N; ++v) ++start[p->comp[v] + 1];
  for (uint32_t c = 0; c < C; ++c) start[c + 1] += start[c];
  {
    std::vector<uint32_t> fill(start.begin(), start.end() - 1);
    for (uint32_t v = 0; v < N; ++v) order[fill[p->comp[v]]++] = v;
  }
  std::vector<Digest> digest(C, Digest(0, 0));
  auto one = [&](uint32_t c) {
    uint64_t s0 = 0, s1 = 0, h0, h1;
    for (uint32_t k = start[c]; k < start[c + 1]; ++k) {
      const uint32_t v = order[k];
      const Digest& iv = id[node_image[v]];
      rec::node_element(iv.first, iv.second, node_feat[v], p->is_root[v] != 0, h0, h1);
      s0 += h0;
      s1 += h1;
      for (uint32_t e = p->row_ptr[v]; e < p->row_ptr[v + 1]; ++e) {
        const lfr_edge& r = p->edges[e];
        const uint32_t w = r.dst, kind = rec::edge_kind(p->track[v], p->track[w], p->comp[v], p->comp[w]);
        if (kind == LFR_EDGE_SKIP) continue;
        uint32_t words[19];
        std::memcpy(words, &r, sizeof words);  // flow[18], sim
        const Digest& iw = id[node_image[w]];
        rec::edge_element(iv.first, iv.second, iw.first, iw.second, node_feat[v], node_feat[w], kind, words, h0, h1);
        s0 += h0;
        s1 += h1;
      }
    }
    digest[c] = Digest(s0, s1);
  };
  unsigned n_thr = 1;
  if ((uint64_t)N + p->n_edges >= (1u << 16)) {
    const unsigned hw = std::thread::hardware_concurrency();
    n_thr = std::min(8u, hw ? hw : 1u);
  }
  if (const char* e = std::getenv("LFR_HOST_THREADS")) n_thr = (unsigned)std::max(1, std::min(64, std::atoi(e)));
  constexpr uint32_t kBlock = 64;
  std::atomic<uint32_t> next{0};
  auto work = [&] {
    for (;;) {
      const uint32_t b = next.fetch_add(1);
      if ((uint64_t)b * kBlock >= C) return;
      for (uint32_t c = b * kBlock; c < std::min<uint64_t>(C, (uint64_t)(b + 1) * kBlock); ++c) one(c);
    }
  };
  std::vector<std::thread> helpers;
  for (unsigned t = 1; t < n_thr; ++t) helpers.emplace_back(work);
  work();
  for (std::thread& h : helpers) h.join();
  return digest;
}

}  // namespace

int64_t lfr_host_problem_record(const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat,
                                uint32_t n_images, const uint8_t* names, const uint64_t* name_off, uint8_t* out,
                                uint64_t cap) {
  namespace rec = lfr::record;
  if (!record_input_ok(p, node_image, node_feat, n_images, names, name_off)) return LFR_EINVAL;
  const uint64_t need = rec::record_bytes(p->n_components);
  if (!out || cap < need) return (int64_t)need;
  std::vector<Digest> d = component_digests(p, node_image, node_feat, n_images, names, name_off);
  std::sort(d.begin(), d.end());
  rec::store_u64(out, rec::kMagic);
  rec::store_u64(out + 8, d.size());
  for (size_t c = 0; c < d.size(); ++c) {
    rec::store_u64(out + rec::kHeaderBytes + 16 * c, d[c].first);
    rec::store_u64(out + rec::kHeaderBytes + 16 * c + 8, d[c].second);
  }
  return (int64_t)need;
}

int lfr_wire_update_solution_since_record(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names,
                                          const uint64_t* name_off, const lfr_problem* p, const uint32_t* node_image,
                                          const uint32_t* node_feat, const uint8_t* record, uint64_t record_len,
                                          double* positions, uint8_t* held, uint64_t* n_held, uint32_t* n_touched,
                                          uint32_t* n_changed) {
  namespace rec = lfr::record;
  if (!record_input_ok(p, node_image, node_feat, n_images, names, name_off)) return LFR_EINVAL;
  uint64_t R = 0;
  if (!rec::check(record, record_len, &R)) return LFR_EINVAL;
  const uint32_t C = p->n_components;
  const std::vector<Digest> d = component_digests(p, node_image, node_feat, n_images, names, name_off);
  std::vector<Digest> earlier(R);
  for (uint64_t k = 0; k < R; ++k)
    earlier[k] = Digest(rec::load_u64(record + rec::kHeaderBytes + 16 * k), rec::load_u64(record + rec::kHeaderBytes + 16 * k + 8));
  std::vector<uint8_t> changed(C, 0);
  uint32_t nc = 0;
  for (uint32_t c = 0; c < C; ++c)
    if (!std::binary_search(earlier.begin(), earlier.end(), d[c])) {
      changed[c] = 1;
      ++nc;
    }
  const int rc = lfr::join::update_nodes(buf, len, n_images, names, name_off, p->n_nodes, node_image, node_feat, p->comp, C,
                                         positions, held, n_held, n_touched, changed.data());
  if (rc == LFR_OK && n_changed) *n_changed = nc;
  return rc;
}

namespace {

// The group of every component of `p`: its nodes' (one scene per component); LFR_EINVAL when a node's image has
// no group below G or a component's nodes span two groups
int component_groups(const lfr_problem* p, const uint32_t* node_image, uint32_t n_images, const uint32_t* group_of_image,
                     uint32_t G, std::vector<uint32_t>& group) {
  constexpr uint32_t kNone = 0xffffffffu;
  if (n_images && !group_of_image) return LFR_EINVAL;
  for (uint32_t k = 0; k < n_images; ++k)
    if (group_of_image[k] >= G) return LFR_EINVAL;
  group.assign(p->n_components, kNone);
  for (uint32_t v = 0; v < p->n_nodes; ++v) {
    uint32_t& g = group[p->comp[v]];
    const uint32_t gv = group_of_image[node_image[v]];
    if (g != kNone && g != gv) return LFR_EINVAL;
    g = gv;
  }
  return LFR_OK;
}

}  // namespace

int lfr_wire_update_solution_groups(uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                                    const uint32_t* group_of_image, uint32_t n_groups, const uint8_t* const* files,
                                    const uint64_t* file_len, const uint8_t* const* records, const uint64_t* record_len,
                                    const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat,
                                    double* positions, uint8_t* held, uint64_t* n_held, uint32_t* n_touched,
                                    uint32_t* n_changed) {
  namespace rec = lfr::record;
  namespace join = lfr::join;
  if (!record_input_ok(p, node_image, node_feat, n_images, names, name_off)) return LFR_EINVAL;
  const uint32_t N = p->n_nodes, C = p->n_components, G = n_groups;
  if (N && (!positions || !held)) return LFR_EINVAL;
  if (G && ((files && !file_len) || (records && !record_len))) return LFR_EINVAL;
  std::vector<uint32_t> cgroup;
  if (component_groups(p, node_image, n_images, group_of_image, G, cgroup) != LFR_OK) return LFR_EINVAL;
  // every record checked, and its digests as (group, d0, d1), ascending
  std::vector<std::array<uint64_t, 3>> earlier;
  std::vector<uint8_t> has_record(G, 0);
  for (uint32_t g = 0; records && g < G; ++g) {
    if (!records[g]) continue;
    uint64_t R = 0;
    if (!rec::check(records[g], record_len[g], &R)) return LFR_EINVAL;
    has_record[g] = 1;
    for (uint64_t k = 0; k < R; ++k)
      earlier.push_back({g, rec::load_u64(records[g] + rec::kHeaderBytes + 16 * k),
                         rec::load_u64(records[g] + rec::kHeaderBytes + 16 * k + 8)});
  }
  join::Decoded d;
  const uint8_t no_name = 0;
  if (join::decode_groups(G, files, file_len, n_images, names ? names : &no_name, name_off, group_of_image, d) != LFR_OK)
    return LFR_EINVAL;
  // a component of a scene with a record is changed when its digest is not in that scene's record
  std::vector<uint8_t> changed(C, 0);
  uint32_t nc = 0;
  if (std::find(has_record.begin(), has_record.end(), (uint8_t)1) != has_record.end()) {
    const std::vector<Digest> dg = component_digests(p, node_image, node_feat, n_images, names, name_off);
    for (uint32_t c = 0; c < C; ++c) {
      if (cgroup[c] >= G || !has_record[cgroup[c]]) continue;
      const std::array<uint64_t, 3> key{cgroup[c], dg[c].first, dg[c].second};
      if (!std::binary_search(earlier.begin(), earlier.end(), key)) {
        changed[c] = 1;
        ++nc;
      }
    }
  }
  join::join_decoded(d, N, node_image, node_feat, positions, held, nullptr);
  join::touch_components(N, p->comp, C, positions, held, n_held, n_touched, changed.data());
  if (n_changed) *n_changed = nc;
  return LFR_OK;
}

int64_t lfr_host_problem_record_groups(const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat,
                                       uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                                       const uint32_t* group_of_image, uint32_t n_groups, uint8_t* out, uint64_t cap,
                                       uint64_t* group_off) {
  namespace rec = lfr::record;
  if (!record_input_ok(p, node_image, node_feat, n_images, names, name_off) || !group_off) return LFR_EINVAL;
  const uint32_t C = p->n_components, G = n_groups;
  std::vector<uint32_t> cgroup;
  if (component_groups(p, node_image, n_images, group_of_image, G, cgroup) != LFR_OK) return LFR_EINVAL;
  std::vector<std::array<uint64_t, 3>> d(C);
  {
    const std::vector<Digest> dg = component_digests(p, node_image, node_feat, n_images, names, name_off);
    for (uint32_t c = 0; c < C; ++c) d[c] = {cgroup[c], dg[c].first, dg[c].second};
  }
  std::sort(d.begin(), d.end());
  // output g: its header, then its digests; group_off[g] = 16 g + 16 (the components of the groups before g)
  std::vector<uint64_t> count(G, 0);
  for (const auto& x : d) ++count[x[0]];
  group_off[0] = 0;
  for (uint32_t g = 0; g < G; ++g) group_off[g + 1] = group_off[g] + rec::record_bytes(count[g]);
  const uint64_t need = group_off[G];
  if (!out || cap < need) return (int64_t)need;
  for (uint32_t g = 0; g < G; ++g) {
    rec::store_u64(out + group_off[g], rec::kMagic);
    rec::store_u64(out + group_off[g] + 8, count[g]);
  }
  for (uint32_t c = 0; c < C; ++c) {
    uint8_t* at = out + rec::kHeaderBytes * (d[c][0] + 1) + 16 * (uint64_t)c;
    rec::store_u64(at, d[c][1]);
    rec::store_u64(at + 8, d[c][2]);
  }
  return (int64_t)need;
}

int64_t lfr_wire_encode_solution_carried(uint64_t n_images, const uint64_t* img_ptr, const uint8_t* names,
                                         const uint64_t* name_off, const float* fact, const uint32_t* feature_idx,
                                         const float* di, const float* dj, const uint8_t* file, uint64_t file_len,
                                         uint8_t* out, uint64_t cap, uint64_t* n_carried) {
  if (!img_ptr || !name_off || (n_images && !fact) || (!file && file_len) || n_images >= lfr::join::kNoImage)
    return LFR_EINVAL;
  for (uint64_t i = 0; i < n_images; ++i)
    if (img_ptr[i + 1] < img_ptr[i] || name_off[i + 1] < name_off[i]) return LFR_EINVAL;
  if ((name_off[n_images] && !names) || (img_ptr[n_images] && (!feature_idx || !di || !dj))) return LFR_EINVAL;
  const uint8_t no_name = 0;
  const uint8_t* nm = names ? names : &no_name;
  {
    std::unordered_set<std::string> seen;
    seen.reserve(n_images);
    for (uint64_t i = 0; i < n_images; ++i)
      if (!seen.emplace(reinterpret_cast<const char*>(nm) + name_off[i], name_off[i + 1] - name_off[i]).second)
        return LFR_EINVAL;  // a repeated scene image name
  }
  lfr::join::Decoded d;
  if (lfr::join::decode(file, file_len, (uint32_t)n_images, nm, name_off, d) != LFR_OK) return LFR_EINVAL;
  std::vector<uint64_t> msg_of(n_images, ~0ull);  // the winning message of each scene image
  for (uint64_t i = 0; i < d.n_images; ++i)
    if (d.image_id[i] != lfr::join::kNoImage) msg_of[d.image_id[i]] = i;
  // the output assembly: scene images with their displacements and then their carried entries, then the
  // winning messages of other names in file order; one lfr_wire_encode_solution() call writes it
  std::vector<uint64_t> o_ptr(1, 0), o_off(1, 0);
  std::vector<uint8_t> o_names;
  std::vector<float> o_fact, o_di, o_dj;
  std::vector<uint32_t> o_feat;
  std::vector<uint64_t> eff;
  std::vector<uint32_t> scene_feats;
  uint64_t carried = 0;
  auto put_name = [&](const uint8_t* p, uint64_t len, float f) {
    o_names.insert(o_names.end(), p, p + len);
    o_off.push_back(o_names.size());
    o_fact.push_back(f);
  };
  auto put_entry = [&](uint32_t f, float a, float b) {
    o_feat.push_back(f);
    o_di.push_back(a);
    o_dj.push_back(b);
  };
  for (uint64_t i = 0; i < n_images; ++i) {
    put_name(nm + name_off[i], name_off[i + 1] - name_off[i], fact[i]);
    for (uint64_t k = img_ptr[i]; k < img_ptr[i + 1]; ++k) put_entry(feature_idx[k], di[k], dj[k]);
    if (msg_of[i] != ~0ull) {
      scene_feats.assign(feature_idx + img_ptr[i], feature_idx + img_ptr[i + 1]);
      std::sort(scene_feats.begin(), scene_feats.end());
      lfr::join::effective_entries(d, msg_of[i], eff);
      for (uint64_t e : eff)
        if (!std::binary_search(scene_feats.begin(), scene_feats.end(), d.feature_idx[e])) {
          put_entry(d.feature_idx[e], d.di[e], d.dj[e]);
          ++carried;
        }
    }
    o_ptr.push_back(o_feat.size());
  }
  for (uint64_t i = 0; i < d.n_images; ++i) {
    if (!d.wins[i] || d.image_id[i] != lfr::join::kNoImage) continue;
    put_name(file + d.name_off[i], d.name_len[i], d.fact[i]);
    lfr::join::effective_entries(d, i, eff);
    for (uint64_t e : eff) put_entry(d.feature_idx[e], d.di[e], d.dj[e]);
    carried += eff.size();
    o_ptr.push_back(o_feat.size());
  }
  if (o_names.empty()) o_names.push_back(0);
  if (o_feat.empty()) put_entry(0, 0.f, 0.f);  // a valid pointer for every array; o_ptr does not reach it
  const uint64_t I = o_fact.size();
  const int64_t need = lfr_wire_encode_solution(I, o_ptr.data(), o_names.data(), o_off.data(), o_fact.data(), o_feat.data(),
                                                o_di.data(), o_dj.data(), nullptr, 0);
  if (out && cap >= (uint64_t)need)
    lfr_wire_encode_solution(I, o_ptr.data(), o_names.data(), o_off.data(), o_fact.data(), o_feat.data(), o_di.data(),
                             o_dj.data(), out, cap);
  if (n_carried) *n_carried = carried;
  return need;
}

}  // extern "C"
