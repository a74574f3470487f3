// lfr_cut.h — the deterministic 2-way cut that stands in for
// colmap::ComputeNormalizedMinGraphCut(edges, weights, 2) (solve.cc:192).
//
// The reference gets its cut from COLMAP's bundled Graclus, which is neither in the reference
// repository nor in this image, so results cannot be matched there; what can be matched is the
// INTERFACE: like the COLMAP call, the cut is a function of the undirected edge list and the
// integer edge weights only (no node weights).  Balance is on volume (weighted degree), the
// quantity a normalized cut normalises by.  One definition, used by the product host stage
// (lfr_host.cc), by its numpy twin (graph.py::two_way_cut, checked to agree) and by the COLMAP
// shim behind which the reference's own solve.cc is compiled as a checker
// (oracle/ref_shims/colmap/base/graph_cut.h).  The recursive cut built on it (cut_step,
// recursive_cut_all, at the end of this file) is shared by the host stage and the graph stage on the
// GPU (lfr_capi.cu), so both split oversized meta-components with the same code; lfr_cut.cuh is its
// level-parallel twin on the device, tested to give the same groups.
//
// Algorithm (all ties broken by ascending node id, so the result is unique):
//   1. adjacency with parallel edges merged, neighbours ascending; vol(x) = sum of incident weights
//   2. connected pieces by BFS from ascending start nodes
//   3. more than one piece: pieces sorted by (volume desc, first node asc) are dealt to the
//      lighter side (side 0 on ties)
//   4. one piece: BFS from the lowest node, restart from the node reached last (a pseudo-peripheral
//      node), grow side 0 along that BFS order until it holds half the volume (at least one node,
//      at most all but one), then one refinement sweep in the same order: a node moves across when
//      that lowers the cut and does not empty its side.
#pragma once
#include <algorithm>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>

#ifdef __CUDACC__
#define LFR_CUT_HD __host__ __device__
#else
#define LFR_CUT_HD
#endif

namespace lfr {

struct CutEdge {
  uint32_t a, b;
  int64_t w;
};

// The weight of an undirected meta-edge: static_cast<int>(100 * sum of similarities) (solve.cc:329).
// Out of int range that cast is undefined in C++; here it saturates at INT_MIN / INT_MAX (truncation
// toward zero inside), so the host stage and the graph stage on the GPU agree on every finite input.
LFR_CUT_HD inline int64_t cut_weight(double sim_sum) {
  const double x = 100.0 * sim_sum;
  if (x >= 2147483647.0) return 2147483647;
  if (x <= -2147483648.0) return -2147483647 - 1;
  return (int64_t)(int)x;
}

struct CutWorkspace {
  std::vector<int32_t> local;  // node id -> index in `nodes` (-1 outside a call); grown on demand
  std::vector<uint32_t> nodes;  // ascending node ids of the current call
  std::vector<uint8_t> side;    // per index in `nodes`
  // scratch
  std::vector<uint32_t> ptr, fill, nbr, order, queue, piece_of;
  std::vector<int64_t> wgt, vol;
  std::vector<uint8_t> mark;
  std::vector<std::pair<uint32_t, int64_t>> tmp;
};

// Fills W.nodes (ascending) and W.side; W.local maps node id -> index and must be released with
// cut_release() once the caller is done with it.
inline void two_way_cut(const CutEdge* edges, size_t m, CutWorkspace& W) {
  uint32_t max_id = 0;
  for (size_t i = 0; i < m; ++i) max_id = std::max(max_id, std::max(edges[i].a, edges[i].b));
  if (W.local.size() <= max_id) W.local.resize((size_t)max_id + 1, -1);
  W.nodes.clear();
  for (size_t i = 0; i < m; ++i) {
    if (W.local[edges[i].a] < 0) { W.local[edges[i].a] = 0; W.nodes.push_back(edges[i].a); }
    if (W.local[edges[i].b] < 0) { W.local[edges[i].b] = 0; W.nodes.push_back(edges[i].b); }
  }
  std::sort(W.nodes.begin(), W.nodes.end());
  const uint32_t n = (uint32_t)W.nodes.size();
  for (uint32_t i = 0; i < n; ++i) W.local[W.nodes[i]] = (int32_t)i;
  // 1. adjacency (CSR over local indices; local order = id order, so "ascending id" = ascending index)
  W.ptr.assign((size_t)n + 1, 0);
  for (size_t i = 0; i < m; ++i) {
    ++W.ptr[W.local[edges[i].a] + 1];
    ++W.ptr[W.local[edges[i].b] + 1];
  }
  for (uint32_t i = 0; i < n; ++i) W.ptr[i + 1] += W.ptr[i];
  W.fill.assign(W.ptr.begin(), W.ptr.end() - 1);
  W.nbr.resize(2 * m);
  W.wgt.resize(2 * m);
  for (size_t i = 0; i < m; ++i) {
    const uint32_t la = (uint32_t)W.local[edges[i].a], lb = (uint32_t)W.local[edges[i].b];
    W.nbr[W.fill[la]] = lb; W.wgt[W.fill[la]++] = edges[i].w;
    W.nbr[W.fill[lb]] = la; W.wgt[W.fill[lb]++] = edges[i].w;
  }
  W.vol.assign(n, 0);
  {  // sort each list by neighbour, merge parallel edges (compacting in place)
    uint32_t out = 0;
    for (uint32_t x = 0; x < n; ++x) {
      const uint32_t beg = W.ptr[x], end = W.ptr[x + 1];
      W.tmp.clear();
      for (uint32_t j = beg; j < end; ++j) W.tmp.emplace_back(W.nbr[j], W.wgt[j]);
      std::sort(W.tmp.begin(), W.tmp.end(), [](const std::pair<uint32_t, int64_t>& p, const std::pair<uint32_t, int64_t>& q) { return p.first < q.first; });
      W.ptr[x] = out;
      for (size_t j = 0; j < W.tmp.size(); ++j) {
        if (j > 0 && W.tmp[j].first == W.tmp[j - 1].first) {
          W.wgt[out - 1] += W.tmp[j].second;
        } else {
          W.nbr[out] = W.tmp[j].first;
          W.wgt[out] = W.tmp[j].second;
          ++out;
        }
        W.vol[x] += W.tmp[j].second;
      }
    }
    W.ptr[n] = out;
  }
  auto bfs = [&](uint32_t start, std::vector<uint32_t>& ord) {  // order of first visits; marks W.mark
    const size_t first = ord.size();
    ord.push_back(start);
    W.mark[start] = 1;
    for (size_t head = first; head < ord.size(); ++head) {
      const uint32_t u = ord[head];
      for (uint32_t j = W.ptr[u]; j < W.ptr[u + 1]; ++j) {
        const uint32_t v = W.nbr[j];
        if (!W.mark[v]) {
          W.mark[v] = 1;
          ord.push_back(v);
        }
      }
    }
  };
  W.side.assign(n, 0);
  // 2. connected pieces
  W.mark.assign(n, 0);
  W.order.clear();
  std::vector<uint32_t>& piece_start = W.queue;  // offsets into W.order
  piece_start.clear();
  for (uint32_t s = 0; s < n; ++s) {
    if (W.mark[s]) continue;
    piece_start.push_back((uint32_t)W.order.size());
    bfs(s, W.order);
  }
  const size_t n_pieces = piece_start.size();
  piece_start.push_back((uint32_t)W.order.size());
  if (n_pieces > 1) {
    // 3. deal whole pieces, heaviest first, to the lighter side
    std::vector<std::pair<int64_t, uint32_t>> key(n_pieces);  // (volume, piece); the first node of piece i is order[piece_start[i]], ascending in i
    for (size_t i = 0; i < n_pieces; ++i) {
      int64_t v = 0;
      for (uint32_t j = piece_start[i]; j < piece_start[i + 1]; ++j) v += W.vol[W.order[j]];
      key[i] = std::make_pair(v, (uint32_t)i);
    }
    std::stable_sort(key.begin(), key.end(), [](const std::pair<int64_t, uint32_t>& p, const std::pair<int64_t, uint32_t>& q) {
      if (p.first != q.first) return p.first > q.first;
      return p.second < q.second;  // pieces are numbered by ascending first node
    });
    int64_t w[2] = {0, 0};
    for (const auto& k : key) {
      const int s = (w[0] <= w[1]) ? 0 : 1;
      w[s] += k.first;
      for (uint32_t j = piece_start[k.second]; j < piece_start[k.second + 1]; ++j) W.side[W.order[j]] = (uint8_t)s;
    }
    return;
  }
  // 4. one piece: region growing from a pseudo-peripheral node
  const uint32_t start = W.order.back();  // last node reached by the BFS from node 0
  W.mark.assign(n, 0);
  W.order.clear();
  bfs(start, W.order);
  int64_t total = 0, acc = 0;
  for (uint32_t x = 0; x < n; ++x) total += W.vol[x];
  for (uint32_t x = 0; x < n; ++x) W.side[x] = 1;
  uint32_t cnt[2] = {0, n};
  for (size_t i = 0; i < W.order.size(); ++i) {
    if (i > 0 && (acc * 2 >= total || i == W.order.size() - 1)) break;
    W.side[W.order[i]] = 0;
    acc += W.vol[W.order[i]];
    ++cnt[0];
    --cnt[1];
  }
  for (uint32_t x : W.order) {  // one refinement sweep
    const int s = W.side[x];
    if (cnt[s] <= 1) continue;
    int64_t inside = 0, outside = 0;
    for (uint32_t j = W.ptr[x]; j < W.ptr[x + 1]; ++j) {
      if (W.side[W.nbr[j]] == s) inside += W.wgt[j]; else outside += W.wgt[j];
    }
    if (outside > inside) {
      W.side[x] = (uint8_t)(1 - s);
      --cnt[s];
      ++cnt[1 - s];
    }
  }
}

inline void cut_release(CutWorkspace& W) {
  for (uint32_t g : W.nodes) W.local[g] = -1;
}

// graph.py::recursive_cut (solve.cc:185-250 as a work list): split until every group weighs
// <= max_weight (node weight = nodes of the track, solve.cc:198) or has no internal edge (then its
// nodes become singleton groups, solve.cc:240-246).  The 2-way cut itself is lfr_cut.h.
// One step: cut `edges`, emit the finished groups, return the edge lists of the two sides that
// have to be cut again (empty when done).  A pure function of `edges` (in their order).
// `cap_of_node` (may be NULL): a per-node max_weight in place of `max_weight`; every node of one meta-component
// must have the same cap (the image count of its sub-scene, lfr_host_input::image_group).
inline void cut_step(const std::vector<CutEdge>& edges, const std::vector<uint32_t>& node_weight, uint32_t max_weight,
              CutWorkspace& W, std::vector<uint8_t>& covered, std::vector<std::vector<uint32_t>>* groups,
              std::vector<CutEdge> (&sub)[2], const uint32_t* cap_of_node = nullptr) {
  if (cap_of_node) max_weight = cap_of_node[edges[0].a];
  // a third of all sub-problems are two tracks joined by (parallel) edges: whatever their weights, each
  // side of the cut is one node with no edge inside — two singleton groups (solve.cc:205-211 / :240-246)
  {
    const uint32_t a = edges[0].a, b = edges[0].b;
    bool two_nodes = a != b;
    for (size_t i = 1; two_nodes && i < edges.size(); ++i)
      two_nodes = (edges[i].a == a && edges[i].b == b) || (edges[i].a == b && edges[i].b == a);
    if (two_nodes) {
      sub[0].clear();
      sub[1].clear();
      groups->push_back(std::vector<uint32_t>(1, a));
      groups->push_back(std::vector<uint32_t>(1, b));
      return;
    }
  }
  two_way_cut(edges.data(), edges.size(), W);
  const uint32_t n = (uint32_t)W.nodes.size();
  for (int s = 0; s < 2; ++s) {
    sub[s].clear();
    std::vector<uint32_t> members;
    int64_t w = 0;
    for (uint32_t i = 0; i < n; ++i)
      if (W.side[i] == s) {
        members.push_back(W.nodes[i]);  // ascending
        w += node_weight[W.nodes[i]];
      }
    if (members.empty()) continue;
    if (w <= (int64_t)max_weight) {
      groups->push_back(std::move(members));  // solve.cc:205-211
      continue;
    }
    covered.assign(n, 0);
    for (const CutEdge& e : edges) {
      const int32_t la = W.local[e.a], lb = W.local[e.b];
      if (W.side[la] == s && W.side[lb] == s) {
        sub[s].push_back(e);
        covered[la] = 1;
        covered[lb] = 1;
      }
    }
    for (uint32_t x : members)  // no edge left inside the subset: singleton groups
      if (!covered[W.local[x]]) groups->push_back(std::vector<uint32_t>(1, x));
  }
  cut_release(W);
}

// All oversized meta-components, cut down to groups.  The groups form a partition that does not
// depend on the order in which the sub-problems are processed (each cut is a function of its own edge
// list only), so the work list is shared by a few threads; only membership is used afterwards.
inline void recursive_cut_all(std::vector<std::vector<CutEdge>> roots, const std::vector<uint32_t>& node_weight,
                       uint32_t max_weight, std::vector<std::vector<uint32_t>>* groups,
                       const uint32_t* cap_of_node = nullptr) {
  uint64_t total_edges = 0;
  for (const auto& r : roots) total_edges += r.size();
  unsigned n_thr = 1;
  if (total_edges >= 2048) {
    const unsigned hw = std::thread::hardware_concurrency();
    n_thr = std::min(8u, hw ? hw : 1u);
  }
  if (const char* e = std::getenv("LFR_HOST_THREADS")) n_thr = (unsigned)std::max(1, std::min(64, std::atoi(e)));
  std::vector<std::vector<CutEdge>> work;
  for (auto it = roots.rbegin(); it != roots.rend(); ++it) work.push_back(std::move(*it));
  if (n_thr <= 1) {
    CutWorkspace W;
    std::vector<uint8_t> covered;
    std::vector<CutEdge> sub[2];
    while (!work.empty()) {
      const std::vector<CutEdge> edges = std::move(work.back());
      work.pop_back();
      cut_step(edges, node_weight, max_weight, W, covered, groups, sub, cap_of_node);
      if (!sub[1].empty()) work.push_back(std::move(sub[1]));
      if (!sub[0].empty()) work.push_back(std::move(sub[0]));
    }
    return;
  }
  // shared list: sub-problems of at least kShare edges (a handful per scene: the top of each recursion
  // tree); anything smaller is finished by the thread that produced it, on its own stack
  constexpr size_t kShare = 1024;
  std::mutex mu;
  std::condition_variable cv;
  unsigned active = 0;
  std::vector<std::vector<std::vector<uint32_t>>> found(n_thr);
  auto worker = [&](unsigned t) {
    CutWorkspace W;
    std::vector<uint8_t> covered;
    std::vector<CutEdge> sub[2];
    std::vector<std::vector<CutEdge>> mine;
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      cv.wait(lk, [&] { return !work.empty() || active == 0; });
      if (work.empty()) return;  // and nobody is producing more
      mine.push_back(std::move(work.back()));
      work.pop_back();
      ++active;
      lk.unlock();
      while (!mine.empty()) {
        const std::vector<CutEdge> edges = std::move(mine.back());
        mine.pop_back();
        cut_step(edges, node_weight, max_weight, W, covered, &found[t], sub, cap_of_node);
        for (int sd = 1; sd >= 0; --sd) {
          if (sub[sd].empty()) continue;
          if (sub[sd].size() >= kShare) {
            std::lock_guard<std::mutex> g(mu);
            work.push_back(std::move(sub[sd]));
            cv.notify_one();
          } else {
            mine.push_back(std::move(sub[sd]));
          }
        }
      }
      lk.lock();
      --active;
      cv.notify_all();
    }
  };
  std::vector<std::thread> helpers;
  for (unsigned t = 1; t < n_thr; ++t) helpers.emplace_back(worker, t);
  worker(0);
  for (std::thread& h : helpers) h.join();
  for (auto& f : found)
    for (auto& g : f) groups->push_back(std::move(g));
}

}  // namespace lfr
