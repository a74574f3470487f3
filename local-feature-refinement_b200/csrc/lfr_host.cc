// lfr_host.cc — native host graph stage (include/lfr_host.h): solve.cc:438-606
// from flat match arrays to the arrays of lfr_problem.  Mirrors
// local-feature-refinement_b200/graph.py statement for statement where order
// matters (tie-breaks, accumulation order, the deterministic 2-way cut), and is
// tested to produce identical arrays.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <condition_variable>
#include <map>
#include <thread>
#include <numeric>
#include <unordered_map>
#include <vector>

#include "../../include/lfr_host.h"
#include "lfr_cut.h"

// the 80-byte edge records: the bulk of the stage's output (cfg5: 877 MB), so never value-initialised
struct EdgeBuf {
  lfr_edge* p = nullptr;
  size_t n = 0;
  bool owned = true;
  ~EdgeBuf() {
    if (owned) std::free(p);
  }
  bool alloc(size_t m) {
    if (owned) std::free(p);
    owned = true;
    p = m ? static_cast<lfr_edge*>(std::malloc(m * sizeof(lfr_edge))) : nullptr;
    n = m;
    return m == 0 || p != nullptr;
  }
  void borrow(lfr_edge* q, size_t m) {  // caller-owned destination
    if (owned) std::free(p);
    owned = false;
    p = q;
    n = m;
  }
  lfr_edge& operator[](size_t i) { return p[i]; }
  const lfr_edge& operator[](size_t i) const { return p[i]; }
  const lfr_edge* data() const { return p; }
  size_t size() const { return n; }
};

struct lfr_host_stage {
  uint32_t N = 0, T = 0, C = 0;
  uint64_t E = 0;
  std::vector<uint32_t> row_ptr, track, comp, comp_ptr, comp_nodes, comp_order, node_image, node_feat;
  std::vector<uint8_t> is_root;
  EdgeBuf edges;
};

namespace {

using Clock = std::chrono::steady_clock;
double ms_since(Clock::time_point t0) { return std::chrono::duration<double, std::milli>(Clock::now() - t0).count(); }

// ---- open-addressing hash map uint64 -> uint32 (linear probing, power-of-two capacity) -------
// The reference interns nodes through std::map<pair<string, size_t>> (solve.cc:53-65) and meta
// edges through unordered_map (solve.cc:268-289); only the mapping matters, not the container.
struct FlatMap {
  std::vector<uint64_t> keys;
  std::vector<uint32_t> vals;
  uint64_t mask = 0;
  static constexpr uint64_t kEmpty = ~0ull;
  explicit FlatMap(size_t expected) {
    size_t cap = 16;
    while (cap < expected * 2 + 16) cap <<= 1;
    keys.assign(cap, kEmpty);
    vals.assign(cap, 0);
    mask = cap - 1;
  }
  static uint64_t mix(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    return x;
  }
  // returns the slot of `key`; *fresh = true when it was just inserted (caller sets vals[slot])
  size_t find_or_insert(uint64_t key, bool* fresh) {
    size_t i = (size_t)(mix(key) & mask);
    for (;;) {
      if (keys[i] == key) {
        *fresh = false;
        return i;
      }
      if (keys[i] == kEmpty) {
        keys[i] = key;
        *fresh = true;
        return i;
      }
      i = (i + 1) & mask;
    }
  }
};

// float -> uint32 whose unsigned order is the float order (finite values).  -0.0 maps to the key of
// +0.0: the reference sorts std::tuple<double, size_t, size_t> (solve.cc:489), where the two compare
// equal and the tie falls to (n1, n2).  Tested on the bits, so no flush-to-zero can merge a denormal in.
inline uint32_t sortable_bits(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Indices 0..M-1 sorted ASCENDING by (key[i], n1[i], n2[i]): LSD radix sort on the 32-bit key
// (three 11-bit passes), then the rare runs of equal keys are ordered by (n1, n2).
void sort_matches(const std::vector<uint32_t>& key, const std::vector<uint32_t>& n1, const std::vector<uint32_t>& n2,
                  std::vector<uint32_t>* order_out) {
  const size_t M = key.size();
  // (sorting (key, index) pairs instead, so that a pass streams its input, was measured slower: twice the
  // bytes through the scatter)
  std::vector<uint32_t> a(M), b(M);
  // all three histograms in one sequential sweep over the keys; the first pass reads them in place
  // (its input order is the identity), only the other two gather key[a[i]]
  std::vector<uint32_t> hist(3 * 2049, 0);
  for (size_t i = 0; i < M; ++i) {
    const uint32_t k = key[i];
    ++hist[(k & 2047u) + 1];
    ++hist[2049 + ((k >> 11) & 2047u) + 1];
    ++hist[2 * 2049 + ((k >> 22) & 2047u) + 1];
  }
  for (int pass = 0; pass < 3; ++pass) {
    uint32_t* h = &hist[pass * 2049];
    for (int d = 0; d < 2048; ++d) h[d + 1] += h[d];
  }
  for (size_t i = 0; i < M; ++i) a[hist[key[i] & 2047u]++] = (uint32_t)i;
  for (int pass = 1; pass < 3; ++pass) {
    const int shift = 11 * pass;
    uint32_t* h = &hist[pass * 2049];
    for (size_t i = 0; i < M; ++i) b[h[(key[a[i]] >> shift) & 2047u]++] = a[i];
    a.swap(b);
  }
  for (size_t i = 0; i < M;) {
    size_t j = i + 1;
    while (j < M && key[a[j]] == key[a[i]]) ++j;
    if (j - i > 1)
      std::sort(a.begin() + i, a.begin() + j, [&](uint32_t x, uint32_t y) {
        if (n1[x] != n1[y]) return n1[x] < n1[y];
        if (n2[x] != n2[y]) return n2[x] < n2[y];
        return x < y;
      });
    i = j;
  }
  order_out->swap(a);
}

// ---- connected components, labelled in order of the lowest member index (solve.cc:291-300)
std::vector<uint32_t> connected_components(uint32_t n, const std::vector<uint32_t>& a, const std::vector<uint32_t>& b,
                                           const std::vector<uint8_t>* keep, uint32_t* n_out) {
  std::vector<uint32_t> parent(n);
  std::iota(parent.begin(), parent.end(), 0u);
  auto find = [&](uint32_t x) {
    while (parent[x] != x) {
      parent[x] = parent[parent[x]];
      x = parent[x];
    }
    return x;
  };
  for (size_t i = 0; i < a.size(); ++i) {
    if (keep && !(*keep)[i]) continue;
    const uint32_t ra = find(a[i]), rb = find(b[i]);
    if (ra != rb) parent[std::max(ra, rb)] = std::min(ra, rb);
  }
  std::vector<uint32_t> label(n), of_root(n, UINT32_MAX);
  uint32_t next = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t r = find(i);
    if (of_root[r] == UINT32_MAX) of_root[r] = next++;
    label[i] = of_root[r];
  }
  *n_out = next;
  return label;
}


}  // namespace

extern "C" {

int lfr_host_stage_create(const lfr_host_input* in, lfr_host_stage** out, lfr_host_sizes* sz) {
  if (!in || !out) return LFR_EINVAL;
  *out = nullptr;
  lfr_host_stage* hs = new lfr_host_stage();
  lfr_host_sizes S;
  std::memset(&S, 0, sizeof S);
  const auto t_graph = Clock::now();
  // ---- H1: node interning + directed edges (solve.cc:438-481) -----------------------------
  std::vector<uint64_t> kept_matches;  // indices of matches of non-skipped pairs, in order
  std::vector<uint32_t> m_img1, m_img2;
  std::vector<uint8_t> seen_img(in->n_images, 0);
  {
    uint64_t n_kept = 0;
    for (uint64_t p = 0; p < in->n_pairs; ++p)
      if (!(in->pair_skip && in->pair_skip[p]) && in->pair_ptr[p + 1] >= in->pair_ptr[p]) n_kept += in->pair_ptr[p + 1] - in->pair_ptr[p];
    if (n_kept <= in->n_matches) {
      kept_matches.reserve(n_kept);
      m_img1.reserve(n_kept);
      m_img2.reserve(n_kept);
    }
  }
  for (uint64_t p = 0; p < in->n_pairs; ++p) {
    if (in->pair_skip && in->pair_skip[p]) continue;
    if (in->pair_img1[p] >= in->n_images || in->pair_img2[p] >= in->n_images) {
      delete hs;
      return LFR_EINVAL;
    }
    seen_img[in->pair_img1[p]] = 1;
    seen_img[in->pair_img2[p]] = 1;
    for (uint64_t m = in->pair_ptr[p]; m < in->pair_ptr[p + 1]; ++m) {
      if (!std::isfinite(in->sim[m])) {  // a NaN similarity has no place in the (sim, n1, n2) order of solve.cc:489
        delete hs;
        return LFR_EINVAL;
      }
      kept_matches.push_back(m);
      m_img1.push_back(in->pair_img1[p]);
      m_img2.push_back(in->pair_img2[p]);
    }
  }
  for (uint8_t v : seen_img) S.n_images_seen += v;
  const double t_g0 = ms_since(t_graph);
  const uint64_t M = kept_matches.size();
  std::vector<uint32_t> n1(M), n2(M);
  {
    // (image, feature_idx) -> node id in order of first appearance.  Feature indices are keypoint
    // numbers, so per image they are compact: a direct table per image (a few KB each, cache
    // resident while a pair is processed) replaces the hash map whenever the tables stay small.
    std::vector<uint32_t> max_feat(in->n_images, 0);
    std::vector<uint8_t> img_used(in->n_images, 0);
    for (uint64_t k = 0; k < M; ++k) {
      const uint64_t m = kept_matches[k];
      max_feat[m_img1[k]] = std::max(max_feat[m_img1[k]], in->feat1[m]);
      max_feat[m_img2[k]] = std::max(max_feat[m_img2[k]], in->feat2[m]);
      img_used[m_img1[k]] = img_used[m_img2[k]] = 1;
    }
    uint64_t table_size = 0;
    std::vector<uint64_t> table_off(in->n_images, 0);
    for (uint32_t i = 0; i < in->n_images; ++i) {
      table_off[i] = table_size;
      if (img_used[i]) table_size += (uint64_t)max_feat[i] + 1;
    }
    const bool dense = table_size <= 8 * (2 * M) + (1u << 20);
    std::vector<uint32_t> table(dense ? table_size : 0, 0);   // node id + 1, 0 = not seen yet
    FlatMap ids(dense ? 0 : (size_t)(2 * M));
    auto intern = [&](uint32_t img, uint32_t feat) {
      if (dense) {
        uint32_t& t = table[table_off[img] + feat];
        if (t) return t - 1;
        const uint32_t id = (uint32_t)hs->node_image.size();
        t = id + 1;
        hs->node_image.push_back(img);
        hs->node_feat.push_back(feat);
        return id;
      }
      const uint64_t key = ((uint64_t)img << 32) | feat;
      bool fresh;
      const size_t slot = ids.find_or_insert(key, &fresh);
      if (!fresh) return ids.vals[slot];
      const uint32_t id = (uint32_t)hs->node_image.size();
      ids.vals[slot] = id;
      hs->node_image.push_back(img);
      hs->node_feat.push_back(feat);
      return id;
    };
    for (uint64_t k = 0; k < M; ++k) {
      const uint64_t m = kept_matches[k];
      n1[k] = intern(m_img1[k], in->feat1[m]);   // find_or_create_node: side 1 then side 2
      n2[k] = intern(m_img2[k], in->feat2[m]);
    }
  }
  const double t_g1 = ms_since(t_graph);
  const uint32_t N = (uint32_t)hs->node_image.size();
  hs->N = N;
  hs->E = 2 * M;
  hs->row_ptr.assign((size_t)N + 1, 0);
  for (uint64_t k = 0; k < M; ++k) {
    ++hs->row_ptr[n1[k] + 1];
    ++hs->row_ptr[n2[k] + 1];
  }
  for (uint32_t v = 0; v < N; ++v) hs->row_ptr[v + 1] += hs->row_ptr[v];
  // destination and similarity of every directed edge once more, 8 bytes per edge: the root scores and
  // the track meta-graph below walk all edges three times and need nothing else of the 80-byte records
  std::vector<uint32_t> cdst;
  std::vector<float> csim;
  if (in->edges_out && in->edges_out_capacity >= 2 * M) {
    hs->edges.borrow(in->edges_out, 2 * M);
  } else if (!hs->edges.alloc(2 * M)) {
    delete hs;
    return LFR_ENOMEM;
  }
  {
    // out-edge slot of both directed edges of every match, in add_edge order (n1->n2 then n2->n1,
    // solve.cc:477-478): sequential; the 80-byte record copies then run on several threads
    std::vector<uint32_t> fill(hs->row_ptr.begin(), hs->row_ptr.end() - (N ? 1 : 0));
    std::vector<uint32_t> slot1(M), slot2(M);
    cdst.resize(2 * M);
    csim.resize(2 * M);
    for (uint64_t k = 0; k < M; ++k) {
      slot1[k] = fill[n1[k]]++;
      slot2[k] = fill[n2[k]]++;
    }
    auto copy_range = [&](uint64_t lo, uint64_t hi) {
      for (uint64_t k = lo; k < hi; ++k) {
        const uint64_t m = kept_matches[k];
        lfr_edge& e1 = hs->edges[slot1[k]];
        std::memcpy(e1.flow, in->disp2 + 18 * m, 18 * sizeof(float));   // n1 -> n2 carries disp2
        e1.sim = in->sim[m];
        e1.dst = n2[k];
        lfr_edge& e2 = hs->edges[slot2[k]];
        std::memcpy(e2.flow, in->disp1 + 18 * m, 18 * sizeof(float));   // n2 -> n1 carries disp1
        e2.sim = in->sim[m];
        e2.dst = n1[k];
        cdst[slot1[k]] = n2[k];
        csim[slot1[k]] = in->sim[m];
        cdst[slot2[k]] = n1[k];
        csim[slot2[k]] = in->sim[m];
      }
    };
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const unsigned nt = (M < (1u << 18)) ? 1u : std::min(8u, hw);
    if (nt == 1) {
      copy_range(0, M);
    } else {
      std::vector<std::thread> th;
      for (unsigned t = 0; t < nt; ++t) th.emplace_back(copy_range, M * t / nt, M * (t + 1) / nt);
      for (auto& x : th) x.join();
    }
  }
  if (N == 0) {
    hs->comp_ptr.assign(1, 0);
    *out = hs;
    if (sz) *sz = S;
    return LFR_OK;
  }
  S.graph_ms = ms_since(t_graph);
  if (std::getenv("LFR_HOST_TIMING"))
    std::fprintf(stderr, "graph: match list %.1f ms, node interning %.1f ms, CSR + edge records %.1f ms\n", t_g0, t_g1 - t_g0,
                 S.graph_ms - t_g1);
  const auto t_tracks = Clock::now();
  // ---- H2: constrained Kruskal (solve.cc:489-541) ------------------------------------------
  // std::sort + std::reverse on (sim, n1, n2) (solve.cc:489-490): ascending radix sort, walked backwards
  std::vector<uint32_t> order;
  {
    std::vector<uint32_t> key(M);
    for (uint64_t k = 0; k < M; ++k) key[k] = sortable_bits(in->sim[kept_matches[k]]);
    sort_matches(key, n1, n2, &order);
  }
  const double t_sorted = ms_since(t_tracks);
  // union-find node: parent link and, for roots, the image set (size; list / bitset slot) in one 12-byte record —
  // the root reached by find() is the line the set tests need next
  struct UfNode {
    int32_t parent;  // -1 = root
    uint32_t size;   // images in the set of this root (more than 64 images)
    int32_t slot;    // index into lists (size <= kListMax) or bitsets (above), -1 = singleton
  };
  std::vector<UfNode> uf(N, UfNode{-1, 1, -1});
  if (in->n_images > 65535) {
    delete hs;
    return LFR_EUNSUPPORTED;
  }
  const bool small_sets = in->n_images <= 64;  // image set of a union-find root as one 64-bit mask
  std::vector<uint64_t> mask(small_sets ? N : 0);
  // more than 64 images: a root's image set is {its own image} while it is a singleton (no storage),
  // a short sorted list up to kListMax entries, then a bitset of n_images bits from a pool
  const uint32_t W = (in->n_images + 63) / 64;
  constexpr uint32_t kListMax = 12;
  std::vector<uint16_t> lists;                               // kListMax entries per slot
  std::vector<uint64_t> bitsets;                             // W words per slot
  std::vector<int32_t> free_lists;
  if (small_sets)
    for (uint32_t v = 0; v < N; ++v) mask[v] = 1ull << hs->node_image[v];
  auto set_has = [&](uint32_t r, uint16_t img) -> bool {
    const uint32_t sz = uf[r].size;
    if (sz == 1) return (uint16_t)hs->node_image[r] == img;
    if (sz <= kListMax) {
      const uint16_t* l = &lists[(size_t)uf[r].slot * kListMax];
      for (uint32_t i = 0; i < sz; ++i)
        if (l[i] == img) return true;
      return false;
    }
    return (bitsets[(size_t)uf[r].slot * W + (img >> 6)] >> (img & 63)) & 1ull;
  };
  // visit the images of root r
  auto for_each_image = [&](uint32_t r, auto&& fn) {
    const uint32_t sz = uf[r].size;
    if (sz == 1) {
      fn((uint16_t)hs->node_image[r]);
    } else if (sz <= kListMax) {
      const uint16_t* l = &lists[(size_t)uf[r].slot * kListMax];
      for (uint32_t i = 0; i < sz; ++i) fn(l[i]);
    } else {
      const uint64_t* b = &bitsets[(size_t)uf[r].slot * W];
      for (uint32_t w = 0; w < W; ++w)
        for (uint64_t m = b[w]; m; m &= m - 1) fn((uint16_t)(64 * w + __builtin_ctzll(m)));
    }
  };
  auto sets_clash = [&](uint32_t a, uint32_t b) -> bool {  // a = the smaller set
    if (uf[a].size > kListMax && uf[b].size > kListMax) {
      const uint64_t* x = &bitsets[(size_t)uf[a].slot * W];
      const uint64_t* y = &bitsets[(size_t)uf[b].slot * W];
      for (uint32_t w = 0; w < W; ++w)
        if (x[w] & y[w]) return true;
      return false;
    }
    bool clash = false;
    for_each_image(a, [&](uint16_t img) { clash = clash || set_has(b, img); });
    return clash;
  };
  // dst <- dst U src (disjoint), src released
  auto absorb = [&](uint32_t dst, uint32_t src) {
    const uint32_t new_size = uf[dst].size + uf[src].size;
    if (new_size <= kListMax) {
      if (uf[dst].slot < 0) {  // singleton -> list
        int32_t sl;
        if (!free_lists.empty()) {
          sl = free_lists.back();
          free_lists.pop_back();
        } else {
          sl = (int32_t)(lists.size() / kListMax);
          lists.resize(lists.size() + kListMax);
        }
        lists[(size_t)sl * kListMax] = (uint16_t)hs->node_image[dst];
        uf[dst].slot = sl;
      }
      uint16_t* l = &lists[(size_t)uf[dst].slot * kListMax];
      uint32_t n = uf[dst].size;
      for_each_image(src, [&](uint16_t img) { l[n++] = img; });
    } else {
      if (uf[dst].size <= kListMax) {  // singleton / list -> bitset
        const int32_t sl = (int32_t)(bitsets.size() / W);
        bitsets.resize(bitsets.size() + W, 0);
        uint64_t* b = &bitsets[(size_t)sl * W];
        for_each_image(dst, [&](uint16_t img) { b[img >> 6] |= 1ull << (img & 63); });
        if (uf[dst].slot >= 0) free_lists.push_back(uf[dst].slot);
        uf[dst].slot = sl;
      }
      uint64_t* b = &bitsets[(size_t)uf[dst].slot * W];
      if (uf[src].size > kListMax) {
        const uint64_t* c = &bitsets[(size_t)uf[src].slot * W];
        for (uint32_t w = 0; w < W; ++w) b[w] |= c[w];
      } else {
        for_each_image(src, [&](uint16_t img) { b[img >> 6] |= 1ull << (img & 63); });
      }
    }
    if (uf[src].slot >= 0 && uf[src].size <= kListMax) free_lists.push_back(uf[src].slot);
    uf[dst].size = new_size;
    uf[src].size = 0;
    uf[src].slot = -1;
  };
  auto find = [&](uint32_t x) {
    uint32_t r = x;
    while (uf[r].parent != -1) r = (uint32_t)uf[r].parent;
    while (uf[x].parent != -1) {  // path compression (solve.cc:74-76)
      const uint32_t nx = (uint32_t)uf[x].parent;
      uf[x].parent = (int32_t)r;
      x = nx;
    }
    return r;
  };
  // the loop is a chain of dependent random reads (order -> n1/n2 -> parent -> set): the lines of the
  // edges to come are requested ahead, in two stages (node ids 16 edges ahead, their parents 8 ahead)
  constexpr uint64_t kAheadIds = 16, kAheadParents = 8;
  for (uint64_t oi = M; oi-- > 0;) {
    if (oi >= kAheadIds) {
      const uint32_t ka = order[oi - kAheadIds];
      __builtin_prefetch(&n1[ka]);
      __builtin_prefetch(&n2[ka]);
    }
    if (oi >= kAheadParents) {
      const uint32_t kb = order[oi - kAheadParents];
      __builtin_prefetch(&uf[n1[kb]].parent);
      __builtin_prefetch(&uf[n2[kb]].parent);
    }
    const uint32_t k = order[oi];
    const uint32_t r1 = find(n1[k]), r2 = find(n2[k]);
    if (r1 == r2) continue;
    if (small_sets) {
      if (mask[r1] & mask[r2]) continue;  // set_intersection non-empty (solve.cc:507-511)
      if (__builtin_popcountll(mask[r1]) < __builtin_popcountll(mask[r2])) {  // solve.cc:513-521
        uf[r1].parent = (int32_t)r2;
        mask[r2] |= mask[r1];
        mask[r1] = 0;
      } else {
        uf[r2].parent = (int32_t)r1;
        mask[r1] |= mask[r2];
        mask[r2] = 0;
      }
      continue;
    }
    // std::set_intersection non-empty (solve.cc:507-511); smaller set under larger, tie: root2 under root1 (:513-521)
    const bool r1_smaller = uf[r1].size < uf[r2].size;
    if (sets_clash(r1_smaller ? r1 : r2, r1_smaller ? r2 : r1)) continue;
    if (r1_smaller) {
      uf[r1].parent = (int32_t)r2;
      absorb(r2, r1);
    } else {
      uf[r2].parent = (int32_t)r1;
      absorb(r1, r2);
    }
  }
  const double t_union = ms_since(t_tracks);
  hs->track.assign(N, 0);
  uint32_t T = 0;
  for (uint32_t v = 0; v < N; ++v)
    if (uf[v].parent == -1) hs->track[v] = T++;
  for (uint32_t v = 0; v < N; ++v)
    if (uf[v].parent != -1) hs->track[v] = hs->track[find(v)];
  hs->T = T;
  std::vector<uint32_t> nodes_in_track(T, 0);
  for (uint32_t v = 0; v < N; ++v) ++nodes_in_track[hs->track[v]];
  S.max_track_size = *std::max_element(nodes_in_track.begin(), nodes_in_track.end());
  const double t_ids = ms_since(t_tracks);
  // track of every edge's destination, gathered once: the root scores and the two meta-graph sweeps
  // below then stream (cdst is not needed any more)
  for (size_t e = 0; e < cdst.size(); ++e) cdst[e] = hs->track[cdst[e]];
  const std::vector<uint32_t>& tdst = cdst;
  // ---- H3: roots (solve.cc:552-582) -----------------------------------------------------------
  hs->is_root.assign(N, 0);
  {
    std::vector<double> best_score(T, -1.0);
    std::vector<uint32_t> best_node(T, 0);
    std::vector<uint8_t> has(T, 0);
    for (uint32_t v = 0; v < N; ++v) {
      double score = 0.0;
      for (uint32_t e = hs->row_ptr[v]; e < hs->row_ptr[v + 1]; ++e)
        if (hs->track[v] == tdst[e]) score += (double)csim[e];
      const uint32_t t = hs->track[v];
      if (!has[t] || score > best_score[t] || (score == best_score[t] && v > best_node[t])) {
        has[t] = 1;
        best_score[t] = score;
        best_node[t] = v;
      }
    }
    for (uint32_t t = 0; t < T; ++t) hs->is_root[best_node[t]] = 1;
  }
  S.tracks_ms = ms_since(t_tracks);
  if (std::getenv("LFR_HOST_TIMING"))
    std::fprintf(stderr, "tracks: sort %.1f ms, union-find %.1f ms, track ids %.1f ms, roots %.1f ms\n", t_sorted, t_union - t_sorted,
                 t_ids - t_union, S.tracks_ms - t_ids);
  const auto t_cut = Clock::now();
  // ---- H4: meta-graph, connected components, size-capped cut (solve.cc:252-373) -------------
  std::vector<uint32_t> ma, mb;
  std::vector<double> wsum;
  {
    uint64_t n_inter = 0;
    for (uint32_t v = 0; v < N; ++v)
      for (uint32_t e = hs->row_ptr[v]; e < hs->row_ptr[v + 1]; ++e) n_inter += hs->track[v] != tdst[e];
    // the inter-track edges in traversal order, then a STABLE radix sort by (source track, destination
    // track): equal keys stay in traversal order, so each meta-edge weight is the same left-to-right
    // double sum a map keyed by the pair accumulates (solve.cc:262-283) — without a hash probe per edge
    std::vector<uint64_t> ikey(n_inter);
    std::vector<float> isim(n_inter);
    {
      size_t w = 0;
      for (uint32_t v = 0; v < N; ++v) {
        const uint32_t ts = hs->track[v];
        for (uint32_t e = hs->row_ptr[v]; e < hs->row_ptr[v + 1]; ++e) {
          const uint32_t tt = tdst[e];
          if (ts == tt) continue;
          ikey[w] = (uint64_t)ts * T + tt;
          isim[w] = csim[e];
          ++w;
        }
      }
    }
    std::vector<uint32_t> oa(n_inter), ob(n_inter);
    std::iota(oa.begin(), oa.end(), 0u);
    int key_bits = 1;
    while (key_bits < 64 && ((uint64_t)T * T >> key_bits)) ++key_bits;
    for (int shift = 0; shift < key_bits; shift += 11) {
      uint32_t hist[2049] = {0};
      for (size_t i = 0; i < n_inter; ++i) ++hist[((ikey[i] >> shift) & 2047u) + 1];
      for (int d = 0; d < 2048; ++d) hist[d + 1] += hist[d];
      for (size_t i = 0; i < n_inter; ++i) ob[hist[(ikey[oa[i]] >> shift) & 2047u]++] = oa[i];
      oa.swap(ob);
    }
    for (size_t i = 0; i < n_inter;) {
      const uint64_t key = ikey[oa[i]];
      double sum = (double)isim[oa[i]];
      size_t j = i + 1;
      for (; j < n_inter && ikey[oa[j]] == key; ++j) sum += (double)isim[oa[j]];
      ma.push_back((uint32_t)(key / T));
      mb.push_back((uint32_t)(key % T));
      wsum.push_back(sum);
      i = j;
    }
  }
  const double t_meta = ms_since(t_cut);
  uint32_t n_cc = 0;
  const std::vector<uint32_t> cc = connected_components(T, ma, mb, nullptr, &n_cc);
  S.n_meta_components = n_cc;
  std::vector<uint64_t> cc_nodes(n_cc, 0);
  for (uint32_t t = 0; t < T; ++t) cc_nodes[cc[t]] += nodes_in_track[t];
  std::vector<uint32_t> gc(cc);
  uint32_t next_label = n_cc;
  const uint32_t max_nodes = S.n_images_seen;
  std::vector<std::vector<lfr::CutEdge>> per_cc;
  std::vector<int32_t> big_slot(n_cc, -1);
  for (uint32_t c = 0; c < n_cc; ++c)
    if (cc_nodes[c] > max_nodes) {
      big_slot[c] = (int32_t)per_cc.size();
      per_cc.emplace_back();
    }
  S.n_oversized_meta_components = (uint32_t)per_cc.size();
  if (!per_cc.empty()) {
    for (size_t i = 0; i < ma.size(); ++i) {
      if (!(ma[i] < mb[i])) continue;  // undirected list, weight int(100 * sum sim) (solve.cc:327-330)
      const int32_t s = big_slot[cc[ma[i]]];
      if (s < 0) continue;
      per_cc[s].push_back(lfr::CutEdge{ma[i], mb[i], lfr::cut_weight(wsum[i])});  // static_cast<int>(100 * it.second), solve.cc:329
    }
    std::vector<std::vector<uint32_t>> groups;
    lfr::recursive_cut_all(std::move(per_cc), nodes_in_track, max_nodes, &groups);
    for (const auto& g : groups) {  // labels only say "same group": their order is irrelevant
      for (uint32_t t : g) gc[t] = next_label;
      ++next_label;
    }
    S.n_cut_groups += (uint32_t)groups.size();
  }
  const double t_rec = ms_since(t_cut);
  std::vector<uint8_t> keep(ma.size());
  for (size_t i = 0; i < ma.size(); ++i) keep[i] = gc[ma[i]] == gc[mb[i]];
  uint32_t n_final = 0;
  const std::vector<uint32_t> final_cc = connected_components(T, ma, mb, &keep, &n_final);
  hs->comp.resize(N);
  for (uint32_t v = 0; v < N; ++v) hs->comp[v] = final_cc[hs->track[v]];
  hs->C = n_final;
  S.graph_cut_ms = ms_since(t_cut);
  if (std::getenv("LFR_HOST_TIMING"))
    std::fprintf(stderr, "graph cut: meta-graph %.2f ms, cc + recursive cut %.2f ms (oversized %zu, groups %u), final cc %.2f ms; meta edges %zu\n",
                 t_meta, t_rec - t_meta, per_cc.size(), S.n_cut_groups, S.graph_cut_ms - t_rec, ma.size());
  const auto t_disp = Clock::now();
  // ---- H5: dispatch list (solve.cc:594-604) ----------------------------------------------------
  std::vector<uint32_t> sizes(n_final, 0);
  for (uint32_t v = 0; v < N; ++v) ++sizes[hs->comp[v]];
  hs->comp_order.resize(n_final);
  std::iota(hs->comp_order.begin(), hs->comp_order.end(), 0u);
  std::sort(hs->comp_order.begin(), hs->comp_order.end(), [&](uint32_t x, uint32_t y) {  // sort + reverse on (size, idx)
    if (sizes[x] != sizes[y]) return sizes[x] > sizes[y];
    return x > y;
  });
  std::vector<uint32_t> slot_of(n_final);
  for (uint32_t s = 0; s < n_final; ++s) slot_of[hs->comp_order[s]] = s;
  hs->comp_ptr.assign((size_t)n_final + 1, 0);
  for (uint32_t s = 0; s < n_final; ++s) hs->comp_ptr[s + 1] = hs->comp_ptr[s] + sizes[hs->comp_order[s]];
  hs->comp_nodes.resize(N);
  {
    std::vector<uint32_t> fill(hs->comp_ptr.begin(), hs->comp_ptr.end() - 1);
    for (uint32_t v = 0; v < N; ++v) hs->comp_nodes[fill[slot_of[hs->comp[v]]]++] = v;  // ascending node index
  }
  S.dispatch_ms = ms_since(t_disp);
  S.n_nodes = N;
  S.n_edges = hs->E;
  S.n_tracks = T;
  S.n_components = n_final;
  S.max_component_size = n_final ? sizes[hs->comp_order[0]] : 0;
  *out = hs;
  if (sz) *sz = S;
  return LFR_OK;
}

int lfr_host_stage_export(const lfr_host_stage* hs, uint32_t* row_ptr, lfr_edge* edges, uint32_t* track, uint32_t* comp,
                          uint8_t* is_root, uint32_t* comp_ptr, uint32_t* comp_nodes, uint32_t* comp_order,
                          uint32_t* node_image, uint32_t* node_feat) {
  if (!hs) return LFR_EINVAL;
  auto cp = [](void* dst, const void* src, size_t bytes) {
    if (dst && bytes) std::memcpy(dst, src, bytes);
  };
  cp(row_ptr, hs->row_ptr.data(), hs->row_ptr.size() * 4);
  if (edges != hs->edges.data()) cp(edges, hs->edges.data(), hs->edges.size() * sizeof(lfr_edge));
  cp(track, hs->track.data(), hs->track.size() * 4);
  cp(comp, hs->comp.data(), hs->comp.size() * 4);
  cp(is_root, hs->is_root.data(), hs->is_root.size());
  cp(comp_ptr, hs->comp_ptr.data(), hs->comp_ptr.size() * 4);
  cp(comp_nodes, hs->comp_nodes.data(), hs->comp_nodes.size() * 4);
  cp(comp_order, hs->comp_order.data(), hs->comp_order.size() * 4);
  cp(node_image, hs->node_image.data(), hs->node_image.size() * 4);
  cp(node_feat, hs->node_feat.data(), hs->node_feat.size() * 4);
  return LFR_OK;
}

void lfr_host_stage_destroy(lfr_host_stage* hs) { delete hs; }

}  // extern "C"
