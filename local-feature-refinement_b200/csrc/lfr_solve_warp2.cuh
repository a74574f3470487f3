// lfr_solve_warp2.cuh — latency-optimised warp-per-component solve for
// components with <= 32 unknowns (all of the exhaustive-pair configs: a
// component has at most #images nodes, solve.cc:586).
//
// A solve of a Fountain-scale graph is a few thousand independent, strictly
// sequential LM trajectories; its duration is the latency of the slowest one,
// not bandwidth.  Compared with lfr_solve_warp.cuh (the shared-memory Cholesky tier, kept for
// 80 < n <= 96 and for components whose staged records do not fit in shared memory) this kernel
// shortens every dependent chain of one LM iteration:
//
//   * assembly is edge-parallel: each lane combines its directed edge with its
//     twin (the reverse edge, found once at setup) into the complete 2x2
//     off-diagonal block of the normal matrix and a 5-value contribution to its
//     source node's diagonal block / gradient; a node lane then adds its <= deg
//     contributions.  One owner per written word => no atomics, reproducible.
//   * the damped normal equations are solved in REGISTERS: lane i holds row i of
//     (S H S + D^2 | S g) and the warp runs a Gauss-Jordan elimination, the pivot
//     row broadcast through one shared-memory line (one reciprocal per pivot, no
//     square roots, no back substitution).  For an SPD matrix the pivots
//     are the LDL^T pivots, so "pivot <= 0" is exactly the Cholesky failure test.
//   * warp reductions are batched (several values per butterfly).
//
// Inputs whose edges do not come in (src->dst, dst->src) pairs, or that repeat a
// pair, are still solved (a serial assembly path), just slower.
#pragma once
#include "lfr_setup.cuh"

namespace lfr {

struct Warp2Layout {
  int stage, bar;                                   // staged 80-byte edge records (float4 x 5 each), mbarrier
  int x, xc, g, S, dl, H, scr, tup, prow;           // doubles (byte offsets)
  int eidx, meta, node, rowstart, candptr, cnt;     // u32 / i32
  int twin, outptr, freeof, lof;                    // u16 / i16
  int ldh, total;
  __host__ __device__ Warp2Layout(int emax, int ncmax, int n2max) {
    ldh = n2max | 1;  // odd row stride (in doubles): lanes reading one column hit distinct banks
    int o = 0;
    stage = o; o += 80 * emax;  // 16-byte aligned: destination of the bulk copies
    bar = o; o += 16;
    x = o; o += 16 * ncmax;
    xc = o; o += 16 * ncmax;
    g = o; o += 8 * n2max;
    S = o; o += 8 * n2max;
    dl = o; o += 8 * n2max;
    H = o; o += 8 * n2max * ldh;
    scr = o; o += 8 * 7 * emax;
    tup = o; o += 8 * 5 * emax;
    o = align_up(o, 16);
    prow = o; o += 8 * 2 * 72;  // double-buffered pivot rows of the elimination: 2 rows x (32 columns, rhs, spare)
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

struct Warp2Ctx {
  int lane, Nc, Ec, nf, n, emax, ldh;
  bool irregular;
  double *x, *xc, *g, *S, *dl, *H, *scr, *tup, *prow;
  int prow_stride;
  uint32_t *eidx, *meta, *node;
  uint16_t *twin, *outptr, *lof;
  int16_t* freeof;
  float4* stage;   // this component's candidate out-edge records in shared memory, 5 x float4 each
  uint64_t* bar;   // mbarrier the bulk copies complete on
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
__device__ __forceinline__ void warp_sum2(double& s0, double& s1) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double a = __shfl_xor_sync(kFull, s0, o), b = __shfl_xor_sync(kFull, s1, o);
    s0 += a;
    s1 += b;
  }
}

// Lane partials of |x - xc|^2 and |xc|^2 over the free coordinates, produced where the candidate
// is formed (make_candidate2) and summed in the evaluation pass's butterfly: the parameter-tolerance
// test and the accepted point's norm cost no reduction of their own.
struct CandNorms {
  double dn2, xn2;
};

// Evaluate every kept edge at positions `xe` ([2*Nc], component-local) from the records staged in
// shared memory (five conflict-free LDS.128 per edge: 80-byte stride = 20 banks, a quarter-warp of
// 16-byte accesses covers all 32 banks once); stage {a, r, M} (7 doubles, SoA) for the assembly.
// DIRDERIV = true additionally returns phi'(alpha) = grad f(xe) . dl of the line
// search, accumulated per edge from the same evaluation:
//   grad . dl = sum_e a_e r_e^T (dl_dst - M_e dl_src)      (J_src = -M, J_dst = I)
// so a line-search trial needs no separate gradient assembly pass.
template <bool DIRDERIV, bool NORMS>
__device__ __forceinline__ double eval_pass2(const Warp2Ctx& C, const double* xe, const DevConsts& K,
                                             double* dphi = nullptr, CandNorms* nrm = nullptr) {
  double cost = 0.0, dd = 0.0;
  for (int j = C.lane; j < C.Ec; j += 32) {
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
  if (DIRDERIV && NORMS) {
    double v[4] = {cost, dd, nrm->dn2, nrm->xn2};
    warp_sum_n<4>(v);
    cost = v[0];
    *dphi = v[1];
    nrm->dn2 = v[2];
    nrm->xn2 = v[3];
  } else if (NORMS) {
    double v[3] = {cost, nrm->dn2, nrm->xn2};
    warp_sum_n<3>(v);
    cost = v[0];
    nrm->dn2 = v[1];
    nrm->xn2 = v[2];
  } else if (DIRDERIV) {
    warp_sum2(cost, dd);
    *dphi = dd;
  } else {
    cost = warp_sum(cost);
  }
  __syncwarp();
  return cost;
}

// From the staged evaluation: GRAD_ONLY = false -> H (unscaled, full symmetric),
// g, on the first call the Jacobi scaling S; returns |x - P(x - g)|_inf.
// GRAD_ONLY = true -> returns grad . dl (phi'(alpha) of the line search).
template <bool GRAD_ONLY>
__device__ __forceinline__ double assemble2(const Warp2Ctx& C, bool first, const DevConsts& K) {
  const int E = C.emax, ldh = C.ldh;
  if (!GRAD_ONLY) {
    for (int i = C.lane; i < C.n * ldh; i += 32) C.H[i] = 0.0;
    __syncwarp();
  }
  if (!C.irregular) {
    for (int e = C.lane; e < C.Ec; e += 32) {
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
    __syncwarp();
  }
  double acc = 0.0, gmax = 0.0;
  if (!C.irregular) {
    for (int f = C.lane; f < C.nf; f += 32) {
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
    // serial path for inputs without clean edge twins: one lane accumulates every edge in order
    if (C.lane == 0) {
      for (int i = 0; i < C.n; ++i) C.g[i] = 0.0;
      for (int e = 0; e < C.Ec; ++e) {
        const uint32_t mt = C.meta[e];
        const int fs = C.freeof[mt & 0xfff], fd = C.freeof[(mt >> 12) & 0xfff];
        const double a = C.scr[e], r0 = C.scr[E + e], r1 = C.scr[2 * E + e];
        const double m00 = C.scr[3 * E + e], m01 = C.scr[4 * E + e], m10 = C.scr[5 * E + e],
                     m11 = C.scr[6 * E + e];
        if (fs >= 0) {
          C.g[2 * fs] -= a * (m00 * r0 + m10 * r1);
          C.g[2 * fs + 1] -= a * (m01 * r0 + m11 * r1);
          if (!GRAD_ONLY) {
            double* hd = C.H + (2 * fs) * ldh + 2 * fs;
            hd[0] += a * (m00 * m00 + m10 * m10);
            hd[1] += a * (m00 * m01 + m10 * m11);
            hd[ldh] += a * (m00 * m01 + m10 * m11);
            hd[ldh + 1] += a * (m01 * m01 + m11 * m11);
          }
        }
        if (fd >= 0) {
          C.g[2 * fd] += a * r0;
          C.g[2 * fd + 1] += a * r1;
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
    __syncwarp();
    for (int i = C.lane; i < C.n; i += 32) {
      if (GRAD_ONLY) {
        acc += C.g[i] * C.dl[i];
      } else {
        if (first) C.S[i] = 1.0 / (1.0 + sqrt(C.H[i * ldh + i]));
        const int l = C.lof[i >> 1];
        const double xi = C.x[2 * l + (i & 1)];
        const double p = fmin(fmax(xi - C.g[i], -K.bound), K.bound);
        gmax = fmax(gmax, fabs(xi - p));
      }
    }
  }
  __syncwarp();
  if (GRAD_ONLY) return warp_sum(acc);
  return warp_max(gmax);
}

// (S H S + D^2) y = S g by Gauss-Jordan elimination with the rows in registers
// (lane i <-> row i, n <= NREG <= 32).  Writes dl = -S y; returns validity and
// {model_cost_change, g . dl, |dl|_inf}.
// NREG up to which lm_step2 eliminates with 2x2 block pivots (above: scalar pivots,
// kept for comparison; -DLFR_BLOCK_PIVOT_MAX_NREG=0 restores them everywhere)
#ifndef LFR_BLOCK_PIVOT_MAX_NREG
#define LFR_BLOCK_PIVOT_MAX_NREG 32
#endif
constexpr int kBlockPivotMaxNreg = LFR_BLOCK_PIVOT_MAX_NREG;

template <int NREG>
__device__ __forceinline__ bool lm_step2(const Warp2Ctx& C, double radius, const DevConsts& K,
                                         double* model_change, double* gd, double* dmax) {
  const int n = C.n, i = C.lane;
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
    if (k == i) v = act ? v + d2 : 1.0;  // idle lanes carry identity rows
    a[k] = v;
  }
  const double b0 = si * gi;
  double b = b0;
  bool ok = true;
  // Gauss-Jordan: the pivot lanes publish their raw rows through a double-buffered
  // shared-memory line (one broadcast LDS.128 per two elements instead of
  // shuffles); every other lane eliminates the pivot columns from its own row.
  // The register row is shifted left after every step, so the leading slots
  // always hold the current pivot columns and ONE compact loop body serves every
  // step (a fully unrolled elimination is ~100 KB of straight-line code and stalls
  // on instruction fetch).
  // No per-element guards: all NREG slots are processed every step (slots past
  // the live columns hold zeros), so the step is a straight run of 128-bit
  // shared-memory accesses and DFMAs that the scheduler can overlap freely.
  double y;
  if constexpr (NREG <= kBlockPivotMaxNreg) {
    // 2x2 block pivots (n = 2 x free nodes is even; the diagonal blocks of an SPD
    // matrix are SPD): half as many publish / synchronise / reciprocal rounds on
    // the dependent chain for the same number of DFMAs.  Lanes j, j+1 publish
    // their raw rows; every lane inverts the 2x2 pivot block B itself.
    constexpr int R = NREG + 2;  // second published row (16-byte aligned: NREG is even)
    double inv0 = 0.0, inv1 = 0.0;  // this lane's row of B^-1 (pivot lanes)
    for (int j = 0; j < n; j += 2) {
      double* buf = C.prow + ((j >> 1) & 1) * C.prow_stride;
      if (i == j || i == j + 1) {
        double* row = buf + (i - j) * R;
        double2* row2 = reinterpret_cast<double2*>(row);
#pragma unroll
        for (int k = 0; k < NREG; k += 2) row2[k / 2] = make_double2(a[k], a[k + 1]);
        row[NREG] = b;
      }
      __syncwarp();
      const double2* r0 = reinterpret_cast<const double2*>(buf);
      const double2* r1 = reinterpret_cast<const double2*>(buf + R);
      const double2 p0 = r0[0], p1 = r1[0];  // B = [p0.x p0.y; p1.x p1.y]
      const double bj0 = buf[NREG], bj1 = buf[R + NREG];
      const double det = p0.x * p1.y - p0.y * p1.x;
      ok = ok && (p0.x > 0.0) && (det > 0.0) && isfinite(det);
      const double rdet = 1.0 / det;
      const bool piv_lane = (i == j) || (i == j + 1);
      if (i == j) { inv0 = p1.y * rdet; inv1 = -p0.y * rdet; }
      if (i == j + 1) { inv0 = -p1.x * rdet; inv1 = p0.x * rdet; }
      // [f0 f1] B = [a0 a1]; the pivot rows themselves are kept (raw)
      const double f0 = piv_lane ? 0.0 : (a[0] * p1.y - a[1] * p1.x) * rdet;
      const double f1 = piv_lane ? 0.0 : (a[1] * p0.x - a[0] * p0.y) * rdet;
#pragma unroll
      for (int k = 2; k < NREG; k += 2) {
        const double2 u = r0[k / 2], v = r1[k / 2];
        a[k - 2] = a[k] - f0 * u.x - f1 * v.x;
        a[k - 1] = a[k + 1] - f0 * u.y - f1 * v.y;
      }
      a[NREG - 2] = 0.0;
      a[NREG - 1] = 0.0;
      b -= f0 * bj0 + f1 * bj1;
    }
    // rows j, j+1 now read  B [y_j y_j+1]^T = [b_j b_j+1]^T
    const double bp = __shfl_xor_sync(kFull, b, 1);
    y = (i & 1) ? inv0 * bp + inv1 * b : inv0 * b + inv1 * bp;
  } else {  // scalar pivots (kept for comparison: -DLFR_BLOCK_PIVOT_MAX_NREG=0)
  double myrp = 1.0;
  for (int j = 0; j < n; ++j) {
    double* buf = C.prow + (j & 1) * C.prow_stride;
    double2* buf2 = reinterpret_cast<double2*>(buf);
    if (i == j) {  // the pivot lane only publishes its registers (slot 0 = the pivot)
#pragma unroll
      for (int k = 0; k < NREG; k += 2) buf2[k / 2] = make_double2(a[k], a[k + 1]);
      buf[NREG] = b;
    }
    __syncwarp();
    double2 t[NREG / 2];
#pragma unroll
    for (int k = 0; k < NREG; k += 2) t[k / 2] = buf2[k / 2];
    const double bj = buf[NREG];
    const double piv = t[0].x;
    ok = ok && (piv > 0.0) && isfinite(piv);
    const double rp = 1.0 / piv;  // every lane: no serial work in the pivot lane
    if (i == j) myrp = rp;
    const double f = (i == j) ? 0.0 : a[0] * rp;  // the pivot row itself is kept (un-normalised)
#pragma unroll
    for (int k = 1; k < NREG; ++k) a[k - 1] = a[k] - f * ((k & 1) ? t[k / 2].y : t[k / 2].x);
    a[NREG - 1] = 0.0;
    b -= f * bj;
  }
  y = b * myrp;  // row i now reads  piv_i * y_i = b_i
  }
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
  warp_sum2_max1(mc, dot, mx);
  *model_change = 0.5 * mc;
  *gd = dot;
  *dmax = mx;
  finite = __all_sync(kFull, finite);
  __syncwarp();
  return ok && finite;
}

__device__ __forceinline__ CandNorms make_candidate2(const Warp2Ctx& C, double alpha, const DevConsts& K) {
  CandNorms nr{0.0, 0.0};
  for (int i = C.lane; i < 2 * C.Nc; i += 32) {
    const int f = C.freeof[i >> 1];
    const double xv = C.x[i];
    double v = xv;
    if (f >= 0) {
      v = fmin(fmax(xv + alpha * C.dl[2 * f + (i & 1)], -K.bound), K.bound);
      const double dv = xv - v;
      nr.dn2 += dv * dv;
      nr.xn2 += v * v;
    }
    C.xc[i] = v;
  }
  __syncwarp();
  return nr;
}

// The warp2 tier's primitives as the driver's operations (see lfr_lm.cuh).  Both norms of the
// parameter test come from the CandNorms fused into the candidate's evaluation.
template <int NREG>
struct Warp2Tier {
  static constexpr int kStride = 32;
  static constexpr unsigned kTier = LmProfile::kWarp2;
  static constexpr int kPolyWord = LmProfile::kTierWord;
  Warp2Ctx& C;
  const DevConsts& K;
  CandNorms nr;  // of the last candidate
  __device__ int tid() const { return C.lane; }
  __device__ int lane() const { return C.lane; }
  __device__ bool lead() const { return C.lane == 0; }
  __device__ double eval_x() { return eval_pass2<false, false>(C, C.x, K); }
  __device__ double assemble(bool first) { return assemble2<false>(C, first, K); }
  __device__ bool lm_step(double radius, double* model_change, double* gd, double* dmax) {
    return lm_step2<NREG>(C, radius, K, model_change, gd, dmax);
  }
  __device__ double trial(double alpha) {
    nr = make_candidate2(C, alpha, K);
    return eval_pass2<false, true>(C, C.xc, K, nullptr, &nr);
  }
  __device__ double trial_slope(double alpha, double* dphi) {
    nr = make_candidate2(C, alpha, K);
    return eval_pass2<true, true>(C, C.xc, K, dphi, &nr);
  }
  __device__ double slope() { return assemble2<true>(C, false, K); }
  __device__ void scale_step(double s) {
    for (int i = C.lane; i < C.n; i += 32) C.dl[i] *= s;
    __syncwarp();
  }
  __device__ double x_norm() {
    double a = 0.0;
    for (int i = C.lane; i < C.n; i += 32) {
      const int l = C.lof[i >> 1];
      const double xv = C.x[2 * l + (i & 1)];
      a += xv * xv;
    }
    return sqrt(warp_sum(a));
  }
  __device__ double step_norm() { return sqrt(nr.dn2); }
  __device__ double accept() {
    for (int i = C.lane; i < 2 * C.Nc; i += 32) C.x[i] = C.xc[i];
    __syncwarp();
    return sqrt(nr.xn2);
  }
  __device__ unsigned long long counter() const { return 0; }
};

// (12 resident warps per SM = 168 registers for NREG <= 16; 8 (255 registers) and 16 (128 registers)
// are the alternatives)
template <int WARPS, int NREG>
__global__ void __launch_bounds__(WARPS * 32, (NREG > 16 ? 8 : 12) / WARPS)
solve_warp2_kernel(const DevProblem P, const DevConsts K, const WarpBucket B) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t item = blockIdx.x * WARPS + wib;
  if (item >= B.n) return;  // warps are independent: no block-level barrier anywhere
  const uint32_t c = B.list[item];
  unsigned char* base = smem_raw + (size_t)wib * B.smem_per_warp;
  const Warp2Layout L(B.emax, B.ncmax, B.n2max);
  Warp2Ctx C;
  C.lane = lane;
  C.emax = B.emax;
  C.ldh = L.ldh;
  C.stage = (float4*)(base + L.stage);
  C.bar = (uint64_t*)(base + L.bar);
  C.x = (double*)(base + L.x);
  C.xc = (double*)(base + L.xc);
  C.g = (double*)(base + L.g);
  C.S = (double*)(base + L.S);
  C.dl = (double*)(base + L.dl);
  C.H = (double*)(base + L.H);
  C.scr = (double*)(base + L.scr);
  C.tup = (double*)(base + L.tup);
  C.prow = (double*)(base + L.prow);
  C.prow_stride = 72;
  C.eidx = (uint32_t*)(base + L.eidx);
  C.meta = (uint32_t*)(base + L.meta);
  C.node = (uint32_t*)(base + L.node);
  uint32_t* rowstart = (uint32_t*)(base + L.rowstart);
  uint32_t* candptr = (uint32_t*)(base + L.candptr);
  int* cnt = (int*)(base + L.cnt);
  C.twin = (uint16_t*)(base + L.twin);
  C.outptr = (uint16_t*)(base + L.outptr);
  C.freeof = (int16_t*)(base + L.freeof);
  C.lof = (uint16_t*)(base + L.lof);

  LmProfile prof(P, c, lane == 0);
  // ---- component setup (solve.cc:98-143) --------------------------------------
  int Ec = 0, nf = 0;
  bool irregular = false;
  warp_setup(C, rowstart, candptr, cnt, B.ncmax, P, K, c, lane, &Ec, &nf, &irregular);
  C.Ec = Ec;
  C.irregular = irregular;
  C.nf = nf;
  C.n = 2 * nf;
  __syncwarp();
  Warp2Tier<NREG> T{C, K, {0.0, 0.0}};
  lm_solve(T, P, K, c, prof);
}

}  // namespace lfr
