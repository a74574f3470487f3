// lfr_solve_warp2.cuh — the register tier: a component with <= 80 unknowns solved by T = 32, 64 or
// 128 threads with the rows of its normal matrix in registers.  Written once over T:
//
//   T = 32        one warp per component, n <= 32 unknowns (all of the exhaustive-pair configs: a
//                 component has at most #images nodes, solve.cc:586): solve_warp2_kernel and the
//                 persistent solve_warp2_queue_kernel, synchronised by __syncwarp()
//   T = 64, 128   one CTA per component, 32 < n <= 80 (e.g. the 17..41-node components of an
//                 ETH3D-courtyard-scale scene): solve_tile_kernel; warp 0 performs the setup, then the
//                 tile works in lock step with __syncthreads()
//
// A solve of a Fountain-scale graph is a few thousand independent, strictly
// sequential LM trajectories; its duration is the latency of the slowest one,
// not bandwidth.  Compared with lfr_solve_warp.cuh (the shared-memory Cholesky tier, kept for
// 80 < n <= 96 and for components whose staged records do not fit in shared memory) this tier
// shortens every dependent chain of one LM iteration:
//
//   * assembly is edge-parallel: each thread combines its directed edge with its
//     twin (the reverse edge, found once at setup) into the complete 2x2
//     off-diagonal block of the normal matrix and a 5-value contribution to its
//     source node's diagonal block / gradient; a node thread then adds its <= deg
//     contributions.  One owner per written word => no atomics, reproducible.
//   * the damped normal equations are solved in REGISTERS: thread i holds row i of
//     (S H S + D^2 | S g) and the group runs a Gauss-Jordan elimination, the pivot
//     rows broadcast through one shared-memory line (one reciprocal per pivot block, no
//     square roots, no back substitution).  For an SPD matrix the pivots
//     are the LDL^T pivots, so "pivot <= 0" is exactly the Cholesky failure test.
//   * warp reductions are batched (several values per butterfly).
//
// Inputs whose edges do not come in (src->dst, dst->src) pairs, or that repeat a
// pair, are still solved (a serial assembly path), just slower.
#pragma once
#include "lfr_setup.cuh"

namespace lfr {

// Doubles in one of the two pivot-row buffers of the elimination: 2 rows x (32 columns, rhs, spare)
// for a warp, 2 x (80 columns, rhs, spare) for a tile
__host__ __device__ constexpr int prow_buf(int threads) { return threads == 32 ? 72 : 168; }

// Shared memory of one component solved by `threads` threads; host and device must agree.  Every
// thread count above 32 has the same layout (sized for four warps and 80 columns).
struct RegLayout {
  int stage, bar;                                   // staged 80-byte edge records (float4 x 5 each), mbarrier
  int x, xc, g, S, dl, H, scr, tup, prow, red, hdr; // doubles (byte offsets); red, hdr: tiles only
  int eidx, meta, node, rowstart, candptr, cnt;     // u32 / i32
  int twin, outptr, freeof, lof;                    // u16 / i16
  int ldh, total;
  __host__ __device__ RegLayout(int emax, int ncmax, int n2max, int threads) {
    ldh = n2max | 1;  // odd row stride (in doubles): threads reading one column hit distinct banks
    int o = 0;
    stage = o; o += 80 * emax;  // 16-byte aligned: destination of the bulk copies
    bar = o; o += 16;
    x = o; o += 16 * ncmax;
    xc = o; o += 16 * ncmax;
    g = o; o += 8 * n2max;
    S = o; o += 8 * n2max;
    dl = o; o += 8 * n2max;
    H = o; o += 8 * n2max * ldh;
    scr = o; o += 8 * 7 * emax;  // the staged evaluation (7 doubles per candidate edge)
    tup = o; o += 8 * 5 * emax;  // the assembly tuples (5)
    o = align_up(o, 16);
    prow = o; o += 8 * 2 * prow_buf(threads);  // double-buffered pair of pivot rows
    red = hdr = o;
    if (threads > 32) {
      o += 8 * 3 * 4;           // block reductions (<= 4 warps)
      hdr = o; o += 16;         // Ec, nf, irregular broadcast by warp 0
    }
    eidx = o; o += 4 * emax;
    meta = o; o += 4 * emax;
    node = o; o += 4 * ncmax;
    rowstart = o; o += 4 * ncmax;
    candptr = o; o += 4 * (ncmax + 1);
    cnt = o; o += 4 * 2 * ncmax;
    twin = o; o += 2 * emax;
    outptr = o; o += 2 * (ncmax + 1);
    freeof = o; o += 2 * ncmax;
    lof = o; o += 2 * (n2max / 2 + 1);
    total = align_up(o, 16);
  }
};

template <int T>
struct RegCtx {
  int tid, Nc, Ec, nf, n, emax, ldh;  // tid: thread of the component's group (the lane, for a warp)
  bool irregular;
  double *x, *xc, *g, *S, *dl, *H, *scr, *tup, *prow;
  double* red;     // tiles only: the reductions' line
  uint32_t *eidx, *meta, *node;
  uint16_t *twin, *outptr, *lof;
  int16_t* freeof;
  float4* stage;   // this component's candidate out-edge records in shared memory, 5 x float4 each
  uint64_t* bar;   // mbarrier the bulk copies complete on
  uint32_t *rowstart, *candptr;  // the setup's: first out-edge of a node, its candidate range
  int* cnt;                      // the setup's: kept out- and in-degrees
  __device__ __forceinline__ RegCtx(unsigned char* base, const RegLayout& L, int emax_, int tid_)
      : tid(tid_), emax(emax_), ldh(L.ldh) {
    stage = (float4*)(base + L.stage);
    bar = (uint64_t*)(base + L.bar);
    x = (double*)(base + L.x);
    xc = (double*)(base + L.xc);
    g = (double*)(base + L.g);
    S = (double*)(base + L.S);
    dl = (double*)(base + L.dl);
    H = (double*)(base + L.H);
    scr = (double*)(base + L.scr);
    tup = (double*)(base + L.tup);
    prow = (double*)(base + L.prow);
    if constexpr (T > 32) red = (double*)(base + L.red);
    eidx = (uint32_t*)(base + L.eidx);
    meta = (uint32_t*)(base + L.meta);
    node = (uint32_t*)(base + L.node);
    rowstart = (uint32_t*)(base + L.rowstart);
    candptr = (uint32_t*)(base + L.candptr);
    cnt = (int*)(base + L.cnt);
    twin = (uint16_t*)(base + L.twin);
    outptr = (uint16_t*)(base + L.outptr);
    freeof = (int16_t*)(base + L.freeof);
    lof = (uint16_t*)(base + L.lof);
  }
};

template <int N>
__device__ __forceinline__ void warp_sum_n(double (&v)[N]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double t[N];
#pragma unroll
    for (int k = 0; k < N; ++k) t[k] = __shfl_xor_sync(kFull, v[k], o);
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] += t[k];
  }
}

__device__ __forceinline__ void warp_sum2_max1(double& s0, double& s1, double& m0) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double a = __shfl_xor_sync(kFull, s0, o), b = __shfl_xor_sync(kFull, s1, o),
                 c = __shfl_xor_sync(kFull, m0, o);
    s0 += a;
    s1 += b;
    m0 = fmax(m0, c);
  }
}

// What differs between a warp and a CTA of 2 or 4 warps working on one component: the barrier and the
// sum and max over the group ("every thread finite" is a warp vote, or one more of a CTA's sums: see
// reg_lm_step).  A CTA reduces by a butterfly in each warp, then adds the warps' partials from the `red`
// line in warp order; its reductions begin with a barrier (`red` is free, every thread's earlier
// shared-memory accesses are done) and contain a second one.
template <int T>
struct Group {
  static constexpr int NW = T / 32;
  static __device__ __forceinline__ void sync() {
    if constexpr (T == 32) __syncwarp(); else __syncthreads();
  }
  static __device__ __forceinline__ void cta_sum3(const RegCtx<T>& C, double& a, double& b, double& c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(kFull, a, o);
      b += __shfl_xor_sync(kFull, b, o);
      c += __shfl_xor_sync(kFull, c, o);
    }
    const int w = C.tid >> 5;
    __syncthreads();
    if ((C.tid & 31) == 0) {
      C.red[w] = a;
      C.red[NW + w] = b;
      C.red[2 * NW + w] = c;
    }
    __syncthreads();
    a = b = c = 0.0;
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      a += C.red[i];
      b += C.red[NW + i];
      c += C.red[2 * NW + i];
    }
  }
  static __device__ __forceinline__ double sum(const RegCtx<T>& C, double a) {
    if constexpr (T == 32) {
      return warp_sum(a);
    } else {
      double z1 = 0.0, z2 = 0.0;
      cta_sum3(C, a, z1, z2);
      return a;
    }
  }
  static __device__ __forceinline__ double max(const RegCtx<T>& C, double v) {
    if constexpr (T == 32) {
      return warp_max(v);
    } else {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(kFull, v, o));
      __syncthreads();
      if ((C.tid & 31) == 0) C.red[C.tid >> 5] = v;
      __syncthreads();
      v = C.red[0];
#pragma unroll
      for (int i = 1; i < NW; ++i) v = fmax(v, C.red[i]);
      return v;
    }
  }
};

// Evaluate every kept edge at positions `xe` ([2*Nc], component-local) from the records staged in
// shared memory (five conflict-free LDS.128 per edge: 80-byte stride = 20 banks, a quarter-warp of
// 16-byte accesses covers all 32 banks once); stage {a, r, M} (7 doubles, SoA) for the assembly.
// Adds this thread's edges to `cost` and, with DIRDERIV, to `dd`, the line search's
// phi'(alpha) = grad f(xe) . dl accumulated per edge from the same evaluation:
//   grad . dl = sum_e a_e r_e^T (dl_dst - M_e dl_src)      (J_src = -M, J_dst = I)
// so a line-search trial needs no separate gradient assembly pass.  The caller reduces (RegTier::eval).
template <bool DIRDERIV, int T>
__device__ __forceinline__ void reg_eval_edges(const RegCtx<T>& C, const double* xe, const DevConsts& K,
                                               double& cost, double& dd) {
  for (int j = C.tid; j < C.Ec; j += T) {
    const uint32_t mt = C.meta[j];
    const int s = mt & 0xfff, d = (mt >> 12) & 0xfff, kind = mt >> 24;
    const float4* qp = C.stage + 5 * C.eidx[j];
    float4 q[5];
#pragma unroll
    for (int t = 0; t < 5; ++t) q[t] = qp[t];
    const EdgeEval ev = eval_edge(q, kind, xe[2 * s], xe[2 * s + 1], xe[2 * d], xe[2 * d + 1], K);
    double* sc = C.scr + j;
    sc[0] = ev.a;
    sc[C.emax] = ev.r0;
    sc[2 * C.emax] = ev.r1;
    sc[3 * C.emax] = ev.m00;
    sc[4 * C.emax] = ev.m01;
    sc[5 * C.emax] = ev.m10;
    sc[6 * C.emax] = ev.m11;
    cost += ev.half_rho;
    if (DIRDERIV) {
      const int fs = C.freeof[s], fd = C.freeof[d];
      const double s0 = fs >= 0 ? C.dl[2 * fs] : 0.0, s1 = fs >= 0 ? C.dl[2 * fs + 1] : 0.0;
      const double d0 = fd >= 0 ? C.dl[2 * fd] : 0.0, d1 = fd >= 0 ? C.dl[2 * fd + 1] : 0.0;
      dd += ev.a * (ev.r0 * (d0 - (ev.m00 * s0 + ev.m01 * s1)) + ev.r1 * (d1 - (ev.m10 * s0 + ev.m11 * s1)));
    }
  }
}

// From the staged evaluation: GRAD_ONLY = false -> H (unscaled, full symmetric),
// g, on the first call the Jacobi scaling S; returns |x - P(x - g)|_inf.
// GRAD_ONLY = true -> returns grad . dl (phi'(alpha) of the line search).
template <bool GRAD_ONLY, int T>
__device__ __forceinline__ double reg_assemble(const RegCtx<T>& C, bool first, const DevConsts& K) {
  using G = Group<T>;
  const int E = C.emax, ldh = C.ldh;
  if (!GRAD_ONLY) {
    for (int i = C.tid; i < C.n * ldh; i += T) C.H[i] = 0.0;
    G::sync();
  }
  if (!C.irregular) {
    for (int e = C.tid; e < C.Ec; e += T) {
      const uint32_t mt = C.meta[e];
      const int fs = C.freeof[mt & 0xfff], fd = C.freeof[(mt >> 12) & 0xfff];
      const int t = C.twin[e];
      const double a = C.scr[e], r0 = C.scr[E + e], r1 = C.scr[2 * E + e];
      const double m00 = C.scr[3 * E + e], m01 = C.scr[4 * E + e], m10 = C.scr[5 * E + e],
                   m11 = C.scr[6 * E + e];
      const double at = C.scr[t], rt0 = C.scr[E + t], rt1 = C.scr[2 * E + t];
      // contribution of e (as out-edge of its source) and of its twin (as in-edge of the same node)
      C.tup[3 * E + e] = at * rt0 - a * (m00 * r0 + m10 * r1);
      C.tup[4 * E + e] = at * rt1 - a * (m01 * r0 + m11 * r1);
      if (!GRAD_ONLY) {
        C.tup[e] = a * (m00 * m00 + m10 * m10) + at;
        C.tup[E + e] = a * (m00 * m01 + m10 * m11);
        C.tup[2 * E + e] = a * (m01 * m01 + m11 * m11) + at;
        if (fs >= 0 && fd >= 0) {  // block (fs, fd) = -a M^T - a_t M_t
          const double t00 = C.scr[3 * E + t], t01 = C.scr[4 * E + t], t10 = C.scr[5 * E + t],
                       t11 = C.scr[6 * E + t];
          double* h0 = C.H + (2 * fs) * ldh + 2 * fd;
          h0[0] = -a * m00 - at * t00;
          h0[1] = -a * m10 - at * t01;
          h0[ldh] = -a * m01 - at * t10;
          h0[ldh + 1] = -a * m11 - at * t11;
        }
      }
    }
    G::sync();
  }
  double acc = 0.0, gmax = 0.0;
  if (!C.irregular) {
    for (int f = C.tid; f < C.nf; f += T) {
      const int l = C.lof[f];
      double d00 = 0., d01 = 0., d11 = 0., g0 = 0., g1 = 0.;
      for (int j = C.outptr[l]; j < C.outptr[l + 1]; ++j) {
        g0 += C.tup[3 * E + j];
        g1 += C.tup[4 * E + j];
        if (!GRAD_ONLY) {
          d00 += C.tup[j];
          d01 += C.tup[E + j];
          d11 += C.tup[2 * E + j];
        }
      }
      if (GRAD_ONLY) {
        acc += g0 * C.dl[2 * f] + g1 * C.dl[2 * f + 1];
      } else {
        double* hd = C.H + (2 * f) * ldh + 2 * f;
        hd[0] = d00;
        hd[1] = d01;
        hd[ldh] = d01;
        hd[ldh + 1] = d11;
        C.g[2 * f] = g0;
        C.g[2 * f + 1] = g1;
        if (first) {
          C.S[2 * f] = 1.0 / (1.0 + sqrt(d00));
          C.S[2 * f + 1] = 1.0 / (1.0 + sqrt(d11));
        }
        const double x0 = C.x[2 * l], x1 = C.x[2 * l + 1];
        const double p0 = fmin(fmax(x0 - g0, -K.bound), K.bound), p1 = fmin(fmax(x1 - g1, -K.bound), K.bound);
        gmax = fmax(gmax, fmax(fabs(x0 - p0), fabs(x1 - p1)));
      }
    }
  } else {
    // serial path for inputs without clean edge twins: one thread accumulates every edge in order.
    // GRAD_ONLY sums into the pivot-row buffer (free outside lm_step), not g: g stays the gradient at x,
    // which the next lm_step reads when the line search's step is rejected
    double* const gs = GRAD_ONLY ? C.prow : C.g;
    if (C.tid == 0) {
      for (int i = 0; i < C.n; ++i) gs[i] = 0.0;
      for (int e = 0; e < C.Ec; ++e) {
        const uint32_t mt = C.meta[e];
        const int fs = C.freeof[mt & 0xfff], fd = C.freeof[(mt >> 12) & 0xfff];
        const double a = C.scr[e], r0 = C.scr[E + e], r1 = C.scr[2 * E + e];
        const double m00 = C.scr[3 * E + e], m01 = C.scr[4 * E + e], m10 = C.scr[5 * E + e],
                     m11 = C.scr[6 * E + e];
        if (fs >= 0) {
          gs[2 * fs] -= a * (m00 * r0 + m10 * r1);
          gs[2 * fs + 1] -= a * (m01 * r0 + m11 * r1);
          if (!GRAD_ONLY) {
            double* hd = C.H + (2 * fs) * ldh + 2 * fs;
            hd[0] += a * (m00 * m00 + m10 * m10);
            hd[1] += a * (m00 * m01 + m10 * m11);
            hd[ldh] += a * (m00 * m01 + m10 * m11);
            hd[ldh + 1] += a * (m01 * m01 + m11 * m11);
          }
        }
        if (fd >= 0) {
          gs[2 * fd] += a * r0;
          gs[2 * fd + 1] += a * r1;
          if (!GRAD_ONLY) {
            C.H[(2 * fd) * ldh + 2 * fd] += a;
            C.H[(2 * fd + 1) * ldh + 2 * fd + 1] += a;
          }
        }
        if (!GRAD_ONLY && fs >= 0 && fd >= 0) {
          double* h0 = C.H + (2 * fs) * ldh + 2 * fd;
          double* h1 = C.H + (2 * fd) * ldh + 2 * fs;
          h0[0] -= a * m00; h0[1] -= a * m10; h0[ldh] -= a * m01; h0[ldh + 1] -= a * m11;
          h1[0] -= a * m00; h1[1] -= a * m01; h1[ldh] -= a * m10; h1[ldh + 1] -= a * m11;
        }
      }
    }
    G::sync();
    for (int i = C.tid; i < C.n; i += T) {
      if (GRAD_ONLY) {
        acc += gs[i] * C.dl[i];
      } else {
        if (first) C.S[i] = 1.0 / (1.0 + sqrt(C.H[i * ldh + i]));
        const int l = C.lof[i >> 1];
        const double xi = C.x[2 * l + (i & 1)];
        const double p = fmin(fmax(xi - C.g[i], -K.bound), K.bound);
        gmax = fmax(gmax, fabs(xi - p));
      }
    }
  }
  if constexpr (T == 32) __syncwarp();  // (a CTA's reductions begin with their own barrier)
  if (GRAD_ONLY) return G::sum(C, acc);
  return G::max(C, gmax);
}

// (S H S + D^2) y = S g by Gauss-Jordan elimination with the rows in registers
// (thread i <-> row i, n <= NREG <= T).  Writes dl = -S y; returns validity and
// {model_cost_change, g . dl, |dl|_inf}.
template <int NREG, int T>
__device__ __forceinline__ bool reg_lm_step(const RegCtx<T>& C, double radius, const DevConsts& K,
                                            double* model_change, double* gd, double* dmax) {
  const int n = C.n, i = C.tid;
  const bool act = i < n;
  const double si = act ? C.S[i] : 0.0;
  const double gi = act ? C.g[i] : 0.0;
  const double* Hi = C.H + (act ? i : 0) * C.ldh;
  const double hii = act ? Hi[i] * si * si : 1.0;
  const double d2 = act ? fmin(fmax(hii, K.min_diag), K.max_diag) / radius : 0.0;
  double a[NREG];
#pragma unroll
  for (int k = 0; k < NREG; ++k) {
    double v = 0.0;
    if (k < n && act) v = Hi[k] * si * C.S[k];
    if (k == i) v = act ? v + d2 : 1.0;  // idle threads carry identity rows
    a[k] = v;
  }
  const double b0 = si * gi;
  double b = b0;
  bool ok = true;
  // Gauss-Jordan: the pivot threads publish their raw rows through a double-buffered
  // shared-memory line (one broadcast LDS.128 per two elements instead of
  // shuffles); every other thread eliminates the pivot columns from its own row.
  // The register row is shifted left after every step, so the leading slots
  // always hold the current pivot columns and ONE compact loop body serves every
  // step (a fully unrolled elimination is ~100 KB of straight-line code and stalls
  // on instruction fetch).
  // No per-element guards: all NREG slots are processed every step (slots past
  // the live columns hold zeros), so the step is a straight run of 128-bit
  // shared-memory accesses and DFMAs that the scheduler can overlap freely.
  // 2x2 block pivots (n = 2 x free nodes is even; the diagonal blocks of an SPD
  // matrix are SPD): half as many publish / synchronise / reciprocal rounds on
  // the dependent chain as scalar pivots for the same number of DFMAs.  Threads j, j+1
  // publish their raw rows; every thread inverts the 2x2 pivot block B itself.
  constexpr int R = NREG + 2;  // second published row (16-byte aligned: NREG is even)
  // 128-bit words of each pivot row loaded per group of DFMAs: a scheduling choice with the same
  // arithmetic per element; each width keeps the grouping its generated code was measured with
  constexpr int W = T == 32 ? 1 : 2;
  double inv0 = 0.0, inv1 = 0.0;  // this thread's row of B^-1 (pivot threads)
  for (int j = 0; j < n; j += 2) {
    double* buf = C.prow + ((j >> 1) & 1) * prow_buf(T);
    if (i == j || i == j + 1) {
      double* row = buf + (i - j) * R;
      double2* row2 = reinterpret_cast<double2*>(row);
#pragma unroll
      for (int k = 0; k < NREG; k += 2) row2[k / 2] = make_double2(a[k], a[k + 1]);
      row[NREG] = b;
    }
    Group<T>::sync();
    const double2* r0 = reinterpret_cast<const double2*>(buf);
    const double2* r1 = reinterpret_cast<const double2*>(buf + R);
    const double2 p0 = r0[0], p1 = r1[0];  // B = [p0.x p0.y; p1.x p1.y]
    const double bj0 = buf[NREG], bj1 = buf[R + NREG];
    const double det = p0.x * p1.y - p0.y * p1.x;
    ok = ok && (p0.x > 0.0) && (det > 0.0) && isfinite(det);
    const double rdet = 1.0 / det;
    const bool piv = (i == j) || (i == j + 1);
    if (i == j) { inv0 = p1.y * rdet; inv1 = -p0.y * rdet; }
    if (i == j + 1) { inv0 = -p1.x * rdet; inv1 = p0.x * rdet; }
    // [f0 f1] B = [a0 a1]; the pivot rows themselves are kept (raw)
    const double f0 = piv ? 0.0 : (a[0] * p1.y - a[1] * p1.x) * rdet;
    const double f1 = piv ? 0.0 : (a[1] * p0.x - a[0] * p0.y) * rdet;
#pragma unroll
    for (int k0 = 2; k0 < NREG; k0 += 2 * W) {
      double2 u[W], v[W];
#pragma unroll
      for (int q = 0; q < W; ++q) {
        if (k0 + 2 * q < NREG) { u[q] = r0[k0 / 2 + q]; v[q] = r1[k0 / 2 + q]; }
      }
#pragma unroll
      for (int q = 0; q < W; ++q) {
        const int k = k0 + 2 * q;
        if (k < NREG) {
          a[k - 2] = a[k] - f0 * u[q].x - f1 * v[q].x;
          a[k - 1] = a[k + 1] - f0 * u[q].y - f1 * v[q].y;
        }
      }
    }
    a[NREG - 2] = 0.0;
    a[NREG - 1] = 0.0;
    b -= f0 * bj0 + f1 * bj1;
  }
  // rows j, j+1 now read  B [y_j y_j+1]^T = [b_j b_j+1]^T
  const double bp = __shfl_xor_sync(kFull, b, 1);
  const double y = (i & 1) ? inv0 * bp + inv1 * b : inv0 * b + inv1 * bp;
  double mc = 0.0, dot = 0.0, mx = 0.0;
  bool finite = true;
  if (act) {
    const double d = -si * y;
    C.dl[i] = d;
    mc = y * (b0 + d2 * y);
    dot = gi * d;
    mx = fabs(d);
    finite = isfinite(y);
  }
  if constexpr (T == 32) {
    warp_sum2_max1(mc, dot, mx);
  } else {
    double bad = finite ? 0.0 : 1.0;  // "every thread finite" rides in the sums
    Group<T>::cta_sum3(C, mc, dot, bad);
    mx = Group<T>::max(C, mx);
    finite = bad == 0.0;
  }
  *model_change = 0.5 * mc;
  *gd = dot;
  *dmax = mx;
  if constexpr (T == 32) {  // a warp votes, behind the stores (ahead of them the warp kernels' generated code changes)
    finite = __all_sync(kFull, finite);
    __syncwarp();
  }
  return ok && finite;
}

// Thread partials of |x - xc|^2 and |xc|^2 over the free coordinates, produced by a warp where the
// candidate is formed and summed in the evaluation pass's butterfly: the parameter-tolerance
// test and the accepted point's norm cost no reduction of their own.
struct CandNorms {
  double dn2, xn2;
};

// xc = P(x + alpha dl) for free nodes, x for constants.
template <int T>
__device__ __forceinline__ CandNorms reg_candidate(const RegCtx<T>& C, double alpha, const DevConsts& K) {
  CandNorms nr{0.0, 0.0};
  for (int i = C.tid; i < 2 * C.Nc; i += T) {
    const int f = C.freeof[i >> 1];
    const double xv = C.x[i];
    double v = xv;
    if (f >= 0) {
      v = fmin(fmax(xv + alpha * C.dl[2 * f + (i & 1)], -K.bound), K.bound);
      if constexpr (T == 32) {
        const double dv = xv - v;
        nr.dn2 += dv * dv;
        nr.xn2 += v * v;
      }
    }
    C.xc[i] = v;
  }
  Group<T>::sync();
  return nr;
}

// The register size class of a component of (at most) n2max unknowns: 8, 16, 24 or 32 for a warp
__host__ __device__ constexpr int reg_class(int n2max) { return (n2max + 7) & ~7; }

// The register tier's primitives as the driver's operations (see lfr_lm.cuh).  What the widths keep
// apart is how they reduce: a warp sums cost, phi' and the CandNorms of the parameter test in one
// butterfly of the candidate's evaluation; a tile reduces cost and phi' through `red` and takes each
// norm by a sum of its own.
// NREG is the register rows' size class, fixed at compile time (the per-bucket and tile kernels), or 0:
// the class is the warp-uniform run-time `nreg` (the queue kernel).  Only the elimination needs a
// compile-time row size, so with NREG = 0 lm_step branches over the four inlined reg_lm_step<8..32>
// and one copy of everything else (setup, evaluation, assembly, line search, write-back) serves every
// class: about a third of the instructions of four whole solves, which an SM's warps would otherwise
// fetch from up to four places at once.
template <int T, int NREG>
struct RegTier {
  static_assert(NREG > 0 || T == 32, "a run-time register class is a warp's");
  using G = Group<T>;
  static constexpr int kStride = T;
  static constexpr unsigned kTier = T == 32 ? LmProfile::kWarp2 : LmProfile::kTile;
  static constexpr int kPolyWord = LmProfile::kTierWord;
  RegCtx<T>& C;
  const DevConsts& K;
  CandNorms nr;  // of the last candidate (warp)
  int nreg;      // NREG == 0: reg_class() of the component
  // The queue kernel keeps the last trial()'s cost and norms: a failed line search takes them back
  // instead of evaluating the full step again, and restages its evaluation only if the step is accepted.
  // The tiles (which sum the norms from xc) and the per-bucket warp kernels evaluate the full step again:
  // at 168 registers for 12 warps per SM the kept values spill, which measured slower on cfg3, whose
  // searches do not fail.
  static constexpr bool kKeepFullStep = T == 32 && NREG == 0;
  static constexpr bool kSkipFailingContraction = kKeepFullStep;  // see lm_solve
  double cost_full = 0.0;
  CandNorms nr_full{0.0, 0.0};
  bool restored = false;  // xc and the staged evaluation are a trial_slope()'s, not the restored step's
  __device__ int tid() const { return C.tid; }
  __device__ int lane() const { return C.tid & 31; }
  __device__ bool lead() const { return C.tid == 0; }
  // CAND: xe is the candidate whose norms `nr` holds
  template <bool DIRDERIV, bool CAND>
  __device__ __forceinline__ double eval(const double* xe, double* dphi = nullptr) {
    double cost = 0.0, dd = 0.0;
    reg_eval_edges<DIRDERIV>(C, xe, K, cost, dd);
    if constexpr (T > 32) {
      double z = 0.0;
      G::cta_sum3(C, cost, dd, z);  // (its barriers also publish the staged values)
    } else {
      if constexpr (DIRDERIV) {
        double v[4] = {cost, dd, nr.dn2, nr.xn2};
        warp_sum_n<4>(v);
        cost = v[0];
        dd = v[1];
        nr.dn2 = v[2];
        nr.xn2 = v[3];
      } else if constexpr (CAND) {
        double v[3] = {cost, nr.dn2, nr.xn2};
        warp_sum_n<3>(v);
        cost = v[0];
        nr.dn2 = v[1];
        nr.xn2 = v[2];
      } else {
        cost = warp_sum(cost);
      }
    }
    if constexpr (DIRDERIV) *dphi = dd;
    if constexpr (T == 32) __syncwarp();  // publishes the staged values
    return cost;
  }
  __device__ double eval_x() { return eval<false, false>(C.x); }
  __device__ double assemble(bool first) { return reg_assemble<false>(C, first, K); }
  __device__ bool lm_step(double radius, double* model_change, double* gd, double* dmax) {
    if constexpr (NREG > 0) {
      return reg_lm_step<NREG>(C, radius, K, model_change, gd, dmax);
    } else {
      switch (nreg) {
        case 8: return reg_lm_step<8>(C, radius, K, model_change, gd, dmax);
        case 16: return reg_lm_step<16>(C, radius, K, model_change, gd, dmax);
        case 24: return reg_lm_step<24>(C, radius, K, model_change, gd, dmax);
        default: return reg_lm_step<32>(C, radius, K, model_change, gd, dmax);
      }
    }
  }
  __device__ double trial(double alpha) {
    nr = reg_candidate(C, alpha, K);
    const double cost = eval<false, true>(C.xc);
    if constexpr (kKeepFullStep) {
      cost_full = cost;
      nr_full = nr;
      restored = false;
    }
    return cost;
  }
  __device__ double trial_slope(double alpha, double* dphi) {
    nr = reg_candidate(C, alpha, K);
    return eval<true, true>(C.xc, dphi);
  }
  __device__ double slope() { return reg_assemble<true>(C, false, K); }
  __device__ double restore_full_step() {
    if constexpr (kKeepFullStep) {
      nr = nr_full;
      restored = true;
      return cost_full;
    } else {
      return trial(1.0);
    }
  }
  __device__ void scale_step(double s) {
    for (int i = C.tid; i < C.n; i += T) C.dl[i] *= s;
    G::sync();
  }
  __device__ double x_norm() {
    double a = 0.0;
    for (int i = C.tid; i < C.n; i += T) {
      const int l = C.lof[i >> 1];
      const double xv = C.x[2 * l + (i & 1)];
      a += xv * xv;
    }
    return sqrt(G::sum(C, a));
  }
  __device__ double step_norm() {
    if constexpr (T == 32) {
      return sqrt(nr.dn2);
    } else {
      double dn2 = 0.0;
      for (int i = C.tid; i < C.n; i += T) {
        const int l = C.lof[i >> 1];
        const double dv = C.x[2 * l + (i & 1)] - C.xc[2 * l + (i & 1)];
        dn2 += dv * dv;
      }
      return sqrt(G::sum(C, dn2));
    }
  }
  __device__ double accept() {
    if constexpr (T == 32) {
      if (kKeepFullStep && restored) {  // the same candidate and staged evaluation as the restored trial(1.0) made
        reg_candidate(C, 1.0, K);
        eval<false, false>(C.xc);
        restored = false;
      }
      for (int i = C.tid; i < 2 * C.Nc; i += T) C.x[i] = C.xc[i];
      __syncwarp();
      return sqrt(nr.xn2);
    } else {
      double a2 = 0.0;
      for (int i = C.tid; i < 2 * C.Nc; i += T) {
        const double v = C.xc[i];
        C.x[i] = v;
        if (C.freeof[i >> 1] >= 0) a2 += v * v;
      }
      return sqrt(G::sum(C, a2));
    }
  }
  __device__ void reject() {}  // lm_step reads H and g, which only assemble() writes
  __device__ unsigned long long counter() const { return 0; }
};

// One component on T threads, in the shared memory at `base` laid out for (emax, ncmax, n2max): the
// per-bucket kernels and the queue kernel below run exactly this (the queue kernel with NREG = 0, the
// register class then taken from n2max).  The setup is one warp's work (solve.cc:98-143); a tile's
// warp 0 broadcasts its three results through `hdr`.
template <int T, int NREG>
__device__ __forceinline__ void reg_solve(const DevProblem& P, const DevConsts& K, uint32_t c, unsigned char* base,
                                          int emax, int ncmax, int n2max, int tid) {
  const RegLayout L(emax, ncmax, n2max, T);
  RegCtx<T> C(base, L, emax, tid);
  if constexpr (T > 32) C.Nc = (int)(P.comp_ptr[c + 1] - P.comp_ptr[c]);  // (warp 0's load_nodes sets only its own)
  LmProfile prof(P, c, tid == 0);
  int Ec = 0, nf = 0;
  bool irregular = false;
  if (T == 32 || tid < 32) warp_setup(C, C.rowstart, C.candptr, C.cnt, ncmax, P, K, c, tid, &Ec, &nf, &irregular);
  if constexpr (T > 32) {
    int* hdr = (int*)(base + L.hdr);
    if (tid == 0) {
      hdr[0] = Ec;
      hdr[1] = nf;
      hdr[2] = irregular ? 1 : 0;
    }
    __syncthreads();
    Ec = hdr[0];
    nf = hdr[1];
    irregular = hdr[2] != 0;
  }
  C.Ec = Ec;
  C.irregular = irregular;
  C.nf = nf;
  C.n = 2 * nf;
  if constexpr (T == 32) __syncwarp();
  RegTier<T, NREG> Tr{C, K, {0.0, 0.0}, reg_class(n2max)};
  lm_solve(Tr, P, K, c, prof);
}

// One bucket per launch, WARPS components per CTA: the four-warp buckets of queues without a member
// above 16 unknowns, and the single-warp launches of the components whose slot does not fit four to a
// CTA (12 resident warps per SM = 168 registers for NREG <= 16; 8 (255 registers) above)
template <int WARPS, int NREG>
__global__ void __launch_bounds__(WARPS * 32, (NREG > 16 ? 8 : 12) / WARPS)
solve_warp2_kernel(const DevProblem P, const DevConsts K, const WarpBucket B) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t item = blockIdx.x * WARPS + wib;
  if (item >= B.n) return;  // warps are independent: no block-level barrier anywhere
  reg_solve<32, NREG>(P, K, B.list[item], smem_raw + (size_t)wib * B.smem_per_warp, B.emax, B.ncmax, B.n2max, lane);
}

// One bucket per launch, one component per CTA of T threads
template <int T, int NREG>
__global__ void __launch_bounds__(T)
solve_tile_kernel(const DevProblem P, const DevConsts K, const WarpBucket B) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  reg_solve<T, NREG>(P, K, B.list[blockIdx.x], smem_raw, B.emax, B.ncmax, B.n2max, threadIdx.x);
}

// ---- the warp width as one persistent launch ---------------------------------------------------
// One CTA of W warps per SM.  Every warp takes the next component from one device queue — the
// tier's dispatch slots in dispatch order, largest first — solves it in its own shared-memory slot
// (sized for the queue's largest member, laid out from the component's own sizes) and takes the
// next: the longest components start first, on SMs that are not yet crowded, and a warp that
// finishes early picks up work instead of leaving its SM share idle until a launch drains.
struct Warp2Queue {
  const uint32_t* list;  // 2 words per entry: dispatch slot, warp2_queue_dims()
  uint32_t n;
  int slot_bytes;
  uint32_t* ctr;         // [0] next ticket, [1] warps done; the last warp to finish puts both back to 0
};

// A queue entry's layout sizes in one word: candidate out-edges (<= 65535), nodes (<= 4095), and
// unknowns (2..32, even) as n2 / 2 - 1.
__host__ __device__ inline uint32_t warp2_queue_dims(int emax, int ncmax, int n2max) {
  return (uint32_t)emax | (uint32_t)ncmax << 16 | (uint32_t)(n2max / 2 - 1) << 28;
}

// At most kWarp2QueueMaxWarps warps per CTA: 255 registers cover all four register classes, whose
// eliminations are inlined into the one copy of the rest of the solve (RegTier<32, 0>: four whole
// solves, one per class, made the kernel 55 k instructions; the classes as separately allocated
// __noinline__ functions, reading P and K through their addresses, ran cfg2 about 6 % slower)
constexpr int kWarp2QueueMaxWarps = 8;
__global__ void __launch_bounds__(kWarp2QueueMaxWarps * 32, 1)
solve_warp2_queue_kernel(const DevProblem P, const DevConsts K, const Warp2Queue Q) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  unsigned char* base = smem_raw + (size_t)(threadIdx.x >> 5) * Q.slot_bytes;
  for (;;) {
    uint32_t t = 0;
    if (lane == 0) t = atomicAdd(Q.ctr, 1u);
    t = __shfl_sync(kFull, t, 0);
    if (t >= Q.n) break;
    const uint32_t c = Q.list[2 * t], dims = Q.list[2 * t + 1];
    const int emax = dims & 0xffff, ncmax = (dims >> 16) & 0xfff, n2max = 2 * ((int)(dims >> 28) + 1);
    // the slot's previous component wrote it through the generic proxy; this one's records arrive by bulk copies
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    reg_solve<32, 0>(P, K, c, base, emax, ncmax, n2max, lane);  // register class reg_class(n2max)
    // the mbarrier's word is ordinary shared memory in the next component's layout
    __syncwarp();
    if (lane == 0) mbar_inval((uint64_t*)(base + RegLayout(emax, ncmax, n2max, 32).bar));
    __syncwarp();
  }
  if (lane == 0) {
    __threadfence();
    if (atomicAdd(Q.ctr + 1, 1u) == gridDim.x * (blockDim.x >> 5) - 1) {
      __threadfence();  // every other warp's last ticket and its count are in before the reset
      atomicExch(Q.ctr, 0u);
      atomicExch(Q.ctr + 1, 0u);
    }
  }
}

}  // namespace lfr
