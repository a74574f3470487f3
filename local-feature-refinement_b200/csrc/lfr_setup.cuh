// lfr_setup.cuh — a component's setup before the driver runs (solve.cc:98-143), written once for
// every solve tier: which out-edges become residual blocks, the start point, the warp-level node
// loader, the staging of edge records into shared memory by TMA bulk copies, and the setup of the
// staging tiers (warp2, tile) built from them.
#pragma once
#include "lfr_lm.cuh"

namespace lfr {

struct WarpBucket {
  const uint32_t* list;  // dispatch slots handled by this launch
  uint32_t n;
  int emax;    // max candidate out-edges of a component in this bucket
  int ncmax;   // max nodes
  int n2max;   // max unknowns (2 x free nodes)
  int smem_per_warp;
};

__host__ __device__ inline int align_up(int v, int a) { return (v + a - 1) / a * a; }

constexpr unsigned kFull = 0xffffffffu;
constexpr int kMaxWarpN2 = 96;      // unknowns a warp handles
constexpr int kMaxWarpNodes = 4095; // 12-bit local indices in `meta`

// node -> index inside its component's node list
__global__ void local_index_kernel(const uint32_t* comp_ptr, const uint32_t* comp_nodes,
                                   uint32_t n_components, uint32_t total, uint32_t* local_of) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  uint32_t lo = 0, hi = n_components - 1;  // largest c with comp_ptr[c] <= i
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (comp_ptr[mid] <= i) lo = mid; else hi = mid - 1;
  }
  local_of[comp_nodes[i]] = i - comp_ptr[lo];
}

struct EdgeClass {
  bool keep;
  uint32_t kind, dl;  // LFR_EDGE_*, local index of the destination (valid when kept)
};

// The out-edge v -> dst of the component whose node list is node[0, Nc): same track -> Cauchy
// (solve.cc:105), same component -> Tukey (solve.cc:114), otherwise no residual block (solve.cc:123);
// a block whose two ends are both roots is constant and dropped (Ceres removes it, A.1).  Malformed
// input raises *P.err_flag (reported by the host as LFR_EINVAL) and keeps nothing: a dst out of range,
// a self edge, or a node list that disagrees with `comp` (local_of[dst] is only filled for the nodes
// that comp_nodes lists, so it is checked against this node list before it is used as an index).
__device__ __forceinline__ EdgeClass classify_edge(const DevProblem& P, const uint32_t* node, uint32_t Nc, uint32_t v,
                                                   uint32_t dst) {
  EdgeClass r{false, 0u, 0u};
  if (dst >= P.n_nodes || dst == v) {
    *P.err_flag = 1;
    return r;
  }
  if (P.track[v] == P.track[dst]) r.kind = LFR_EDGE_CAUCHY;
  else if (P.comp[v] == P.comp[dst]) r.kind = LFR_EDGE_TUKEY;
  else return r;
  if (P.is_root[v] && P.is_root[dst]) return r;
  r.dl = P.local_of[dst];
  if (r.dl >= Nc || node[r.dl] != dst) {
    *P.err_flag = 1;
    return r;
  }
  r.keep = true;
  return r;
}

// IterationZero: x <- Plus(x, 0) projects the start point of a non-root node onto the box; a root is
// constant and keeps its value.
__device__ __forceinline__ void start_point(const DevProblem& P, const DevConsts& K, uint32_t v, double* x) {
  double p0 = P.positions[2 * (size_t)v], p1 = P.positions[2 * (size_t)v + 1];
  if (!P.is_root[v]) {
    p0 = fmin(fmax(p0, -K.bound), K.bound);
    p1 = fmin(fmax(p1, -K.bound), K.bound);
  }
  x[0] = p0;
  x[1] = p1;
}

// One warp loads component c's node list, the nodes' first out-edges and their start points into
// shared memory, and prefix-sums the out-degrees into candptr[0, Nc]: the candidate out-edges of
// node l are k in [candptr[l], candptr[l + 1]).  Returns their number.
template <class Ctx>
__device__ __forceinline__ int load_nodes(Ctx& C, uint32_t* rowstart, uint32_t* candptr, const DevProblem& P,
                                          const DevConsts& K, uint32_t c, int lane) {
  const uint32_t nbeg = P.comp_ptr[c];
  const int Nc = (int)(P.comp_ptr[c + 1] - nbeg);
  C.Nc = Nc;
  int run = 0;
  for (int l0 = 0; l0 < Nc; l0 += 32) {
    const int l = l0 + lane;
    int d = 0;
    if (l < Nc) {
      const uint32_t v = P.comp_nodes[nbeg + l];
      const uint32_t rs = P.row_ptr[v];
      d = (int)(P.row_ptr[v + 1] - rs);
      C.node[l] = v;
      rowstart[l] = rs;
      start_point(P, K, v, C.x + 2 * l);
    }
    const int inc = warp_incl_scan(d, lane);
    if (l < Nc) candptr[l] = run + inc - d;
    run += __shfl_sync(kFull, inc, 31);
  }
  if (lane == 0) candptr[Nc] = run;
  __syncwarp();
  return run;
}

// The node whose out-edges hold candidate k: the largest l with candptr[l] <= k.
__device__ __forceinline__ int cand_node(const uint32_t* candptr, int Nc, int k) {
  int lo = 0, hi = Nc - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((int)candptr[mid] <= k) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- TMA 1-D bulk copy global -> shared, completion on an mbarrier (sm_90a) -------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");  // make the init visible to the async proxy
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}

// Pull the candidate out-edge records of every node of the component into shared memory, once:
// a node's out-edges are contiguous in the CSR array, so each node is ONE 1-D bulk copy
// (cp.async.bulk, 80 * degree bytes, 16-byte aligned on both sides) completing on the warp's
// mbarrier; all copies are in flight together and no register is tied up.  `P.edges` may be device
// memory or the caller's pinned host buffer (zero-copy over PCIe: the records are read exactly
// once either way, every later evaluation runs from shared memory).
template <class Ctx>
__device__ __forceinline__ void stage_edges(Ctx& C, const uint32_t* rowstart, const uint32_t* candptr, int Nc,
                                            int Eup, const DevProblem& P, int lane) {
  if (Eup == 0) return;
  // Pacing of zero-copy pulls: every resident warp asking for its records at once makes the PCIe
  // link serve ~10 MB of requests round-robin, so the FIRST components (the largest, dispatched
  // first because they run longest) get their data last.  A ticket counter keeps at most
  // `pull_window` bytes outstanding: records arrive in dispatch order at the same link rate.
  const bool paced = P.pull_window != 0;
  if (paced) {
    if (lane == 0) {
      const unsigned long long ticket = atomicAdd(P.pull_ctr, 80ull * (unsigned)Eup);
      const volatile unsigned long long* arrived = P.pull_ctr + 1;
      while ((long long)(ticket - *arrived) >= (long long)P.pull_window) __nanosleep(64);
    }
    __syncwarp();
  }
  if (lane == 0) mbar_arrive_expect_tx(C.bar, 80u * (uint32_t)Eup);
  __syncwarp();
  for (int l = lane; l < Nc; l += 32) {
    const uint32_t d = candptr[l + 1] - candptr[l];
    if (d) bulk_copy_g2s(C.stage + 5 * candptr[l], P.edges + 5 * (size_t)rowstart[l], 80u * d, C.bar);
  }
  mbar_wait(C.bar, 0);
  if (paced && lane == 0) atomicAdd(P.pull_ctr + 1, 80ull * (unsigned)Eup);
  __syncwarp();
}

// Component setup of the staging tiers by ONE warp (the warp2 kernel's, and warp 0 of the tile
// kernel): nodes and start point, staged records, compaction of the kept out-edges with ballots,
// out-edge ranges, free-variable numbering, and the twin (reverse edge) of every kept edge.
template <class Ctx>
__device__ __forceinline__ void warp_setup(Ctx& C, uint32_t* rowstart, uint32_t* candptr, int* cnt, int ncmax,
                                           const DevProblem& P, const DevConsts& K, uint32_t c, int lane,
                                           int* Ec_out, int* nf_out, bool* irregular_out) {
  if (lane == 0) mbar_init(C.bar, 1);
  const int Eup = load_nodes(C, rowstart, candptr, P, K, c, lane);
  const int Nc = C.Nc;
  for (int l = lane; l < Nc; l += 32) {
    cnt[l] = 0;
    cnt[ncmax + l] = 0;
  }
  stage_edges(C, rowstart, candptr, Nc, Eup, P, lane);  // (its final __syncwarp orders the zeros before the counts)
  int kept = 0;
  for (int k0 = 0; k0 < Eup; k0 += 32) {
    const int k = k0 + lane;
    EdgeClass ec{false, 0u, 0u};
    int lo = 0;
    if (k < Eup) {
      lo = cand_node(candptr, Nc, k);
      ec = classify_edge(P, C.node, Nc, C.node[lo], __float_as_uint(C.stage[5 * k + 4].w));
      if (ec.keep) {
        atomicAdd(&cnt[lo], 1);              // kept out-degree (integer: order-independent)
        atomicAdd(&cnt[ncmax + ec.dl], 1);   // kept in-degree
      }
    }
    const unsigned m = __ballot_sync(kFull, ec.keep);
    if (ec.keep) {
      const int pos = kept + __popc(m & ((1u << lane) - 1u));
      C.eidx[pos] = (uint32_t)k;  // index of the record in the staged array
      C.meta[pos] = (uint32_t)lo | (ec.dl << 12) | (ec.kind << 24);
    }
    kept += __popc(m);
  }
  __syncwarp();
  const int Ec = kept;
  int orun = 0, frun = 0;
  for (int l0 = 0; l0 < Nc; l0 += 32) {
    const int l = l0 + lane;
    const int co = (l < Nc) ? cnt[l] : 0, ci = (l < Nc) ? cnt[ncmax + l] : 0;
    const int so = warp_incl_scan(co, lane);
    const bool is_free = (l < Nc) && (co + ci > 0) && !P.is_root[C.node[l < Nc ? l : 0]];
    const int sf = warp_incl_scan(is_free ? 1 : 0, lane);
    if (l < Nc) {
      C.outptr[l] = (uint16_t)(orun + so - co);
      C.freeof[l] = is_free ? (int16_t)(frun + sf - 1) : (int16_t)-1;
      if (is_free) C.lof[frun + sf - 1] = (uint16_t)l;
    }
    orun += __shfl_sync(kFull, so, 31);
    frun += __shfl_sync(kFull, sf, 31);
  }
  if (lane == 0) C.outptr[Nc] = (uint16_t)orun;
  __syncwarp();
  // twin of every kept edge: the unique kept edge dst -> src
  bool irregular = false;
  for (int e = lane; e < Ec; e += 32) {
    const uint32_t mt = C.meta[e];
    const int s = mt & 0xfff, d = (mt >> 12) & 0xfff;
    int found = 0, tw = e;
    for (int j = C.outptr[d]; j < C.outptr[d + 1]; ++j)
      if ((int)((C.meta[j] >> 12) & 0xfff) == s) {
        tw = j;
        ++found;
      }
    irregular = irregular || (found != 1);
    C.twin[e] = (uint16_t)tw;
  }
  *irregular_out = __any_sync(kFull, irregular);
  *Ec_out = Ec;
  *nf_out = frun;
}

}  // namespace lfr
