// lfr_cut.cuh — the recursive 2-way cut of lfr_cut.h (cut_step / recursive_cut_all) on the device.
//
// The same groups as recursive_cut_all, bit for bit.  Three facts of lfr_cut.h make it parallel:
//   - a cut is a function of its own edge list, and the partition does not depend on the order in
//     which sub-problems are processed: all sub-problems of one recursion level are cut at once.  They
//     are node-disjoint (each is the inside of one side of its parent), so every per-node array is
//     indexed by the global node id and shared by the whole level;
//   - the adjacency with parallel edges merged and neighbours ascending is one radix sort of the level's
//     half-edges by (node, neighbour) and a reduce-by-key;
//   - the BFS order (queue order, neighbours ascending) is rebuilt level by level: every frontier node
//     claims its unvisited neighbours, the lowest frontier position wins, and each frontier node writes
//     the neighbours it won in ascending order at its scanned offset.
// One CTA cuts one sub-problem (cut_sub_kernel): the BFS from the lowest node finds the pieces, then
// either pieces are dealt (a bitonic sort on (volume desc, piece asc)) or the region grows from the
// pseudo-peripheral node to half the volume and one warp walks the refinement sweep, whose moves depend
// on the moves before them, with lane-parallel neighbour sums.  The host driver (lfr_capi.cu,
// recursive_cut_on_device) runs the levels: cut, label the finished groups, gather the edges of the
// sides still to be cut as the next level.
#pragma once
#include <cstdint>

#include <cub/cub.cuh>

#include "lfr_cut.h"

namespace lfr {
namespace cut {

constexpr int kThreads = 256;
constexpr uint32_t kNone = 0xffffffffu;

// The adjacency of one level: rows of global node ids, merged weights, per-node scratch.
struct Level {
  const uint32_t* nodes;     // the level's nodes, grouped by sub-problem, ascending inside one
  const uint32_t* node_ptr;  // [n_sub + 1] into nodes
  const uint32_t* beg;       // [n] row of node x: nbr / w [beg[x], end[x])
  const uint32_t* end;
  const uint32_t* nbr;
  const long long* w;
  const uint32_t* node_weight;
  long long* vol;            // [n]
  uint32_t* vis;             // [n] BFS stamps (0 = never visited)
  uint32_t* claim;           // [n] lowest claiming frontier position
  uint8_t* side;             // [n]
  uint32_t* order;           // [n_level_nodes]: BFS order, segment node_ptr[k] of sub-problem k
  uint32_t* piece_start;     // [n_level_nodes]
  long long* pvol;           // [n_level_nodes] piece volumes, then sorted keys
  uint32_t* pidx;            // [n_level_nodes]
  uint8_t* pside;            // [n_level_nodes]
  uint32_t stamp;            // two stamps per level: stamp (pieces), stamp + 1 (second BFS)
  uint64_t max_weight;
  const uint32_t* node_cap;  // may be NULL: max_weight per node, the same for a sub-problem's nodes (sub-scenes)
  long long* side_w;         // [2 n_sub] node weight of each side
  uint32_t* side_min;        // [2 n_sub] lowest node of each side
  uint8_t* cont;             // [2 n_sub] 1: the side is cut again (over max_weight, not two nodes)
  uint32_t* n_groups;        // groups finished as whole sides
};

using Scan = cub::BlockScan<uint32_t, kThreads>;
using ScanLL = cub::BlockScan<long long, kThreads>;
using ReduceLL = cub::BlockReduce<long long, kThreads>;

struct Shared {
  union {
    typename Scan::TempStorage scan;
    typename ScanLL::TempStorage scan_ll;
    typename ReduceLL::TempStorage reduce;
  };
  uint32_t u;
  long long ll;
  unsigned long long sw[2];
  uint32_t smin[2], scnt[2];
};

// Appends the BFS from `start` (order of first visits, neighbours ascending) to ord[tail..]; returns the
// new tail.  vis == stamp marks visited nodes; claim[] of every node it can reach must be kNone.
__device__ uint32_t block_bfs(const Level& L, uint32_t start, uint32_t* ord, uint32_t tail, uint32_t stamp, Shared& sh) {
  const uint32_t tid = threadIdx.x;
  if (tid == 0) {
    ord[tail] = start;
    L.vis[start] = stamp;
  }
  __syncthreads();
  uint32_t head = tail++;
  while (head < tail) {
    for (uint32_t p = head + tid; p < tail; p += kThreads) {
      const uint32_t u = ord[p];
      for (uint32_t j = L.beg[u]; j < L.end[u]; ++j) {
        const uint32_t v = L.nbr[j];
        if (L.vis[v] != stamp) atomicMin(&L.claim[v], p);
      }
    }
    __syncthreads();
    uint32_t out = tail;
    for (uint32_t c = head; c < tail; c += kThreads) {
      const uint32_t p = c + tid;
      uint32_t cnt = 0, off, total;
      if (p < tail) {
        const uint32_t u = ord[p];
        for (uint32_t j = L.beg[u]; j < L.end[u]; ++j) {
          const uint32_t v = L.nbr[j];
          cnt += (L.vis[v] != stamp && L.claim[v] == p) ? 1u : 0u;
        }
      }
      Scan(sh.scan).ExclusiveSum(cnt, off, total);
      if (cnt) {
        const uint32_t u = ord[p];
        uint32_t q = out + off;
        for (uint32_t j = L.beg[u]; j < L.end[u]; ++j) {
          const uint32_t v = L.nbr[j];
          if (L.vis[v] != stamp && L.claim[v] == p) ord[q++] = v;
        }
      }
      out += total;
      __syncthreads();
    }
    for (uint32_t q = tail + tid; q < out; q += kThreads) L.vis[ord[q]] = stamp;
    __syncthreads();
    head = tail;
    tail = out;
  }
  return tail;
}

__device__ __forceinline__ bool piece_less(long long va, uint32_t ia, long long vb, uint32_t ib) {
  return va != vb ? va > vb : ia < ib;
}

// lfr_cut.h two_way_cut + the side bookkeeping of cut_step, one CTA per sub-problem of the level
__global__ void __launch_bounds__(kThreads) cut_sub_kernel(Level L) {
  __shared__ Shared sh;
  const uint32_t k = blockIdx.x, tid = threadIdx.x;
  const uint32_t base = L.node_ptr[k], n = L.node_ptr[k + 1] - base;
  const uint32_t* nodes = L.nodes + base;
  uint32_t* ord = L.order + base;
  if (tid < 2) {
    sh.sw[tid] = 0;
    sh.smin[tid] = kNone;
    sh.scnt[tid] = 0;
  }
  if (n == 2) {  // cut_step's short-cut: two tracks joined by (parallel) edges are two singleton groups
    if (tid < 2) L.side[nodes[tid]] = (uint8_t)tid;
  } else {
    long long vsum = 0;
    for (uint32_t i = tid; i < n; i += kThreads) {
      const uint32_t x = nodes[i];
      long long v = 0;
      for (uint32_t j = L.beg[x]; j < L.end[x]; ++j) v += L.w[j];
      L.vol[x] = v;
      L.claim[x] = kNone;
      vsum += v;
    }
    const long long total = ReduceLL(sh.reduce).Sum(vsum);
    if (tid == 0) sh.ll = total;
    __syncthreads();
    const long long tot = sh.ll;
    // 2. connected pieces: BFS from the lowest node, then from every node still unvisited, ascending
    uint32_t tail = block_bfs(L, nodes[0], ord, 0, L.stamp, sh);
    if (tail < n) {
      uint32_t np = 1, cursor = 1;
      if (tid == 0) L.piece_start[base] = 0;
      for (;;) {
        if (tid == 0) sh.u = kNone;
        __syncthreads();
        uint32_t s = kNone;
        for (uint32_t c = cursor; c < n; c += kThreads) {
          const uint32_t i = c + tid;
          if (i < n && L.vis[nodes[i]] != L.stamp) atomicMin(&sh.u, i);
          __syncthreads();
          s = sh.u;
          __syncthreads();  // every thread has read sh.u before any thread's next atomicMin
          if (s != kNone) break;
        }
        if (s == kNone) break;
        if (tid == 0) L.piece_start[base + np] = tail;
        ++np;
        tail = block_bfs(L, nodes[s], ord, tail, L.stamp, sh);
        cursor = s + 1;
      }
      // piece volumes (pieces are numbered by ascending first node), padded to a power of two
      uint32_t P = 1;
      while (P < np) P <<= 1;
      long long* pv = L.pvol + base;
      uint32_t* pi = L.pidx + base;
      const uint32_t* ps = L.piece_start + base;
      for (uint32_t j = tid; j < P; j += kThreads) {
        pv[j] = j < np ? 0 : (long long)(-0x7fffffffffffffffLL - 1);
        pi[j] = j < np ? j : kNone;
      }
      __syncthreads();
      for (uint32_t q = tid; q < n; q += kThreads) {
        uint32_t lo = 0, hi = np;  // the last piece starting at or before q
        while (hi - lo > 1) {
          const uint32_t mid = (lo + hi) >> 1;
          if (ps[mid] <= q) lo = mid; else hi = mid;
        }
        atomicAdd(reinterpret_cast<unsigned long long*>(&pv[lo]), (unsigned long long)L.vol[ord[q]]);
      }
      __syncthreads();
      // 3. deal whole pieces by (volume desc, piece asc) to the lighter side (side 0 on ties)
      for (uint32_t kk = 2; kk <= P; kk <<= 1)
        for (uint32_t jj = kk >> 1; jj > 0; jj >>= 1) {
          for (uint32_t i = tid; i < P; i += kThreads) {
            const uint32_t l = i ^ jj;
            if (l > i) {
              const bool up = (i & kk) == 0;
              const long long vi = pv[i], vl = pv[l];
              const uint32_t ii = pi[i], il = pi[l];
              if (piece_less(vl, il, vi, ii) == up) {
                pv[i] = vl; pv[l] = vi;
                pi[i] = il; pi[l] = ii;
              }
            }
          }
          __syncthreads();
        }
      if (tid == 0) {
        long long w0 = 0, w1 = 0;
        for (uint32_t r = 0; r < np; ++r) {
          const int s = (w0 <= w1) ? 0 : 1;
          (s ? w1 : w0) += pv[r];
          L.pside[base + pi[r]] = (uint8_t)s;
        }
      }
      __syncthreads();
      for (uint32_t q = tid; q < n; q += kThreads) {
        uint32_t lo = 0, hi = np;
        while (hi - lo > 1) {
          const uint32_t mid = (lo + hi) >> 1;
          if (ps[mid] <= q) lo = mid; else hi = mid;
        }
        L.side[ord[q]] = L.pside[base + lo];
      }
    } else {
      // 4. one piece: BFS again from the node reached last, grow side 0 to half the volume
      const uint32_t start = ord[n - 1];
      for (uint32_t i = tid; i < n; i += kThreads) L.claim[nodes[i]] = kNone;
      __syncthreads();
      block_bfs(L, start, ord, 0, L.stamp + 1, sh);
      // side 0 = the first cut nodes of the order: the least i in [1, n-1] with 2 * vol(order[0..i)) >= total
      if (tid == 0) sh.u = n - 1;
      __syncthreads();
      long long carry = 0;
      uint32_t cut = n - 1;
      for (uint32_t c = 0; c + 1 < n; c += kThreads) {
        const uint32_t q = c + tid;
        const long long v = q + 1 < n ? L.vol[ord[q]] : 0;
        long long inc, agg;
        ScanLL(sh.scan_ll).InclusiveSum(v, inc, agg);
        if (q + 1 < n && (carry + inc) * 2 >= tot) atomicMin(&sh.u, q + 1);
        carry += agg;
        __syncthreads();
        cut = sh.u;
        __syncthreads();  // as above: read before the next chunk's atomicMin
        if (cut != n - 1) break;
      }
      for (uint32_t q = tid; q < n; q += kThreads) L.side[ord[q]] = q < cut ? 0 : 1;
      __syncthreads();
      // one refinement sweep in BFS order: a move depends on every move before it, so one warp walks
      // the order and sums each node's neighbours lane-parallel
      if (tid < 32) {
        volatile uint8_t* side = L.side;
        uint32_t cnt0 = cut, cnt1 = n - cut;
        for (uint32_t q = 0; q < n; ++q) {
          const uint32_t x = ord[q];
          const uint8_t s = side[x];
          if ((s ? cnt1 : cnt0) <= 1) continue;
          long long in = 0, out = 0;
          for (uint32_t j = L.beg[x] + tid; j < L.end[x]; j += 32) {
            if (side[L.nbr[j]] == s) in += L.w[j]; else out += L.w[j];
          }
          for (int o = 16; o > 0; o >>= 1) {
            in += __shfl_xor_sync(0xffffffffu, in, o);
            out += __shfl_xor_sync(0xffffffffu, out, o);
          }
          if (out > in) {
            if (tid == 0) side[x] = (uint8_t)(1 - s);
            if (s) { --cnt1; ++cnt0; } else { --cnt0; ++cnt1; }
          }
          __syncwarp();
        }
      }
    }
  }
  __syncthreads();
  // the sides: node weight, lowest member, size
  for (uint32_t i = tid; i < n; i += kThreads) {
    const uint32_t x = nodes[i];
    const int s = L.side[x];
    atomicAdd(&sh.sw[s], (unsigned long long)L.node_weight[x]);
    atomicMin(&sh.smin[s], x);
    atomicAdd(&sh.scnt[s], 1u);
  }
  __syncthreads();
  if (tid < 2) {
    const bool over = sh.sw[tid] > (L.node_cap ? (uint64_t)L.node_cap[nodes[0]] : L.max_weight);
    L.side_w[2 * k + tid] = (long long)sh.sw[tid];
    L.side_min[2 * k + tid] = sh.smin[tid];
    L.cont[2 * k + tid] = (sh.scnt[tid] && over && n != 2) ? 1 : 0;
    if (sh.scnt[tid] && !(over && n != 2)) atomicAdd(L.n_groups, 1u);
  }
}

// the level's half-edges: key (node, neighbour), weight; the sub-problem of every node
__global__ void half_edges_kernel(const uint32_t* ea, const uint32_t* eb, const long long* ew, const uint32_t* esub, uint32_t m,
                                  int bits, unsigned long long* key, long long* w, uint32_t* sub_of) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint32_t a = ea[i], b = eb[i];
  key[2 * i] = ((unsigned long long)a << bits) | b;
  key[2 * i + 1] = ((unsigned long long)b << bits) | a;
  w[2 * i] = ew[i];
  w[2 * i + 1] = ew[i];
  sub_of[a] = esub[i];
  sub_of[b] = esub[i];
}

// rows of the merged adjacency; the level's nodes (first entry of every row) with their sub-problem
__global__ void rows_kernel(const unsigned long long* ukey, const uint32_t* n_unique, uint32_t n_half, int bits, const uint32_t* sub_of,
                            uint32_t* nbr, uint32_t* beg, uint32_t* end, uint32_t* head, uint32_t* node, uint32_t* node_sub) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nu = *n_unique;
  if (i >= n_half) return;
  if (i >= nu) {  // the node selection reads all n_half flags
    head[i] = 0;
    return;
  }
  const unsigned long long mask = (1ull << bits) - 1;
  const uint32_t x = (uint32_t)(ukey[i] >> bits);
  nbr[i] = (uint32_t)(ukey[i] & mask);
  const bool first = i == 0 || (uint32_t)(ukey[i - 1] >> bits) != x;
  if (first) beg[x] = i;
  if (i + 1 == nu || (uint32_t)(ukey[i + 1] >> bits) != x) end[x] = i + 1;
  head[i] = first ? 1u : 0u;
  node[i] = x;
  node_sub[i] = sub_of[x];
}

__global__ void node_ptr_kernel(const uint32_t* sub, uint32_t n, uint32_t n_sub, uint32_t* node_ptr) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (i == 0 || sub[i] != sub[i - 1])) node_ptr[sub[i]] = i;
  if (i == 0) node_ptr[n_sub] = n;
}

// cut_step's sub-problems of the next level: the edges inside a side that is cut again, keyed by
// (sub-problem, side); their ends are covered
__global__ void keep_edges_kernel(const uint32_t* ea, const uint32_t* eb, const uint32_t* esub, uint32_t m, const uint8_t* side,
                                  const uint8_t* cont, uint32_t stamp, uint32_t* covered, uint32_t* keep, uint32_t* key) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint32_t a = ea[i], b = eb[i], s = side[a];
  const uint32_t k = 2 * esub[i] + s;
  const bool kept = side[b] == s && cont[k];
  keep[i] = kept ? 1u : 0u;
  key[i] = k;
  if (kept) {
    covered[a] = stamp;
    covered[b] = stamp;
  }
}

// the level's labels: a finished side is one group (its lowest node), a node of a side cut again with no
// edge left inside it is a singleton group (cut_step, solve.cc:240-246)
__global__ void label_nodes_kernel(const uint32_t* node, const uint32_t* node_sub, uint32_t n, const uint8_t* side,
                                   const uint8_t* cont, const uint32_t* side_min, const uint32_t* covered, uint32_t stamp,
                                   uint32_t label_base, uint32_t* label, uint32_t* n_groups) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t x = node[i], k = 2 * node_sub[i] + side[x];
  if (!cont[k]) {
    label[x] = label_base + side_min[k];
  } else if (covered[x] != stamp) {
    label[x] = label_base + x;
    atomicAdd(n_groups, 1u);
  }
}

// the roots: undirected meta-edges of the oversized components with their cut weight, keyed by component
__global__ void root_edges_kernel(const uint32_t* idx, uint32_t n, const uint32_t* ma, const uint32_t* mb, const double* wsum,
                                  const uint32_t* cc, uint32_t* ea, uint32_t* eb, long long* ew, uint32_t* key, uint32_t* iota) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e = idx[i];
  ea[i] = ma[e];
  eb[i] = mb[e];
  ew[i] = (long long)lfr::cut_weight(wsum[e]);
  key[i] = cc[ma[e]];
  iota[i] = i;
}

__global__ void heads_kernel(const uint32_t* key, uint32_t n, uint32_t* head) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) head[i] = (i == 0 || key[i] != key[i - 1]) ? 1u : 0u;
}

// edges of sub-problem id (inclusive head count - 1), gathered in key order
__global__ void gather_edges_kernel(const uint32_t* idx, const uint32_t* sid, uint32_t n, const uint32_t* ea, const uint32_t* eb,
                                    const long long* ew, uint32_t* oa, uint32_t* ob, long long* ow, uint32_t* osub) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e = idx[i];
  oa[i] = ea[e];
  ob[i] = eb[e];
  ow[i] = ew[e];
  osub[i] = sid[i] - 1;
}

}  // namespace cut
}  // namespace lfr
