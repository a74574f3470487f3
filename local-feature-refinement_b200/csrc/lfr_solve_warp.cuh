// lfr_solve_warp.cuh — one warp solves one component (one ceres::Problem of
// solve.cc:79-160) start to finish: residual/Jacobian evaluation, J^T J block
// assembly, exact linear solve, LM damping / projected Armijo line search /
// termination (the driver of lfr_lm.cuh, SURVEY Appendix A.6), with no host round trip inside the loop.
//
// Mapping (SURVEY 7 "device-mapping notes"):
//   * lanes <-> directed edges for the evaluation: each lane reads its 80-byte
//     edge record as five 128-bit loads, evaluates cost.cc's interpolator and
//     the robust loss in fp64 registers and stages {a, r, M} (7 doubles) in
//     shared memory;
//   * lanes <-> free nodes for the assembly: each lane gathers its node's
//     out-edges (contiguous, CSR by source) and in-edges (index list built once)
//     from shared memory into the node's 2x2 diagonal block, its gradient pair
//     and its block row of the packed lower-triangular normal matrix — row
//     ownership makes the sums atomics-free and bit-reproducible;
//   * the warp factorises the (<= 96 x 96) damped normal matrix in shared
//     memory (Cholesky with the right-hand side carried as an extra row), and
//     all trust-region scalars live in registers, identical in every lane.
#pragma once
#include "lfr_setup.cuh"

namespace lfr {

__host__ __device__ inline int tri(int n) { return n * (n + 1) / 2; }

// Per-warp shared-memory carve-up; host and device must agree.
struct WarpLayout {
  int x, xc, g, S, dl, dinv, H, A, scr;             // doubles (byte offsets)
  int eidx, meta, node, rowstart, candptr;          // u32
  int inlist, outptr, inptr, freeof, lof;           // u16 / i16
  int total;
  __host__ __device__ WarpLayout(int emax, int ncmax, int n2max) {
    int o = 0;
    x = o; o += 16 * ncmax;
    xc = o; o += 16 * ncmax;
    g = o; o += 8 * n2max;
    S = o; o += 8 * n2max;
    dl = o; o += 8 * n2max;
    dinv = o; o += 8 * n2max;
    H = o; o += 8 * tri(n2max);
    A = o; o += 8 * tri(n2max + 1);
    scr = o; o += 8 * 7 * emax;
    eidx = o; o += 4 * emax;
    meta = o; o += 4 * emax;
    node = o; o += 4 * ncmax;
    rowstart = o; o += 4 * ncmax;
    candptr = o; o += 4 * (ncmax + 1);
    inlist = o; o += 2 * emax;
    outptr = o; o += 2 * (ncmax + 1);
    inptr = o; o += 2 * (ncmax + 1);
    freeof = o; o += 2 * ncmax;
    lof = o; o += 2 * (n2max / 2 + 1);
    total = align_up(o, 16);
  }
};

struct WarpCtx {
  int lane, Nc, Ec, nf, n, emax;
  double *x, *xc, *g, *S, *dl, *dinv, *H, *A, *scr;
  uint32_t *eidx, *meta, *node;
  uint16_t *inlist, *outptr, *inptr, *lof;
  int16_t* freeof;
  const float4* edges;
};

// Evaluate every kept edge at positions `xe` ([2*Nc], component-local); stage
// {a, r0, r1, m00, m01, m10, m11} in shared memory; return the cost (A.1).
__device__ __forceinline__ double eval_pass(const WarpCtx& C, const double* xe, const DevConsts& K) {
  double cost = 0.0;
  for (int j = C.lane; j < C.Ec; j += 32) {
    const uint32_t mt = C.meta[j];
    const int s = mt & 0xfff, d = (mt >> 12) & 0xfff, kind = mt >> 24;
    const float4* qp = C.edges + 5 * (size_t)C.eidx[j];
    float4 q[5];
#pragma unroll
    for (int t = 0; t < 5; ++t) q[t] = __ldg(qp + t);
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
  }
  cost = warp_sum(cost);
  __syncwarp();
  return cost;
}

// Gradient of the cost at the staged evaluation, dotted with dl (phi'(alpha)
// of the line search).
__device__ __forceinline__ double staged_grad_dot(const WarpCtx& C) {
  double acc = 0.0;
  const int E = C.emax;
  for (int f = C.lane; f < C.nf; f += 32) {
    const int l = C.lof[f];
    double g0 = 0., g1 = 0.;
    for (int j = C.outptr[l]; j < C.outptr[l + 1]; ++j) {
      const double a = C.scr[j], r0 = C.scr[E + j], r1 = C.scr[2 * E + j];
      g0 -= a * (C.scr[3 * E + j] * r0 + C.scr[5 * E + j] * r1);
      g1 -= a * (C.scr[4 * E + j] * r0 + C.scr[6 * E + j] * r1);
    }
    for (int t = C.inptr[l]; t < C.inptr[l + 1]; ++t) {
      const int j = C.inlist[t];
      const double a = C.scr[j];
      g0 += a * C.scr[E + j];
      g1 += a * C.scr[2 * E + j];
    }
    acc += g0 * C.dl[2 * f] + g1 * C.dl[2 * f + 1];
  }
  return warp_sum(acc);
}

// J^T J and J^T r from the staged evaluation.  On the first call also fixes the
// Jacobi column scaling S = 1/(1 + sqrt(diag)) (A.6 iter 0).  Leaves H = S H S
// (packed lower triangle), g = raw gradient.  Returns the projected-gradient
// max norm  |x - P(x - g)|_inf.
__device__ __forceinline__ double assemble(const WarpCtx& C, bool first, const DevConsts& K) {
  const int E = C.emax;
  for (int i = C.lane; i < tri(C.n); i += 32) C.H[i] = 0.0;
  __syncwarp();
  for (int f = C.lane; f < C.nf; f += 32) {
    const int l = C.lof[f];
    double d00 = 0., d01 = 0., d11 = 0., g0 = 0., g1 = 0.;
    double* H0 = C.H + tri(2 * f);
    double* H1 = C.H + tri(2 * f + 1);
    for (int j = C.outptr[l]; j < C.outptr[l + 1]; ++j) {
      const double a = C.scr[j], r0 = C.scr[E + j], r1 = C.scr[2 * E + j];
      const double m00 = C.scr[3 * E + j], m01 = C.scr[4 * E + j], m10 = C.scr[5 * E + j],
                   m11 = C.scr[6 * E + j];
      d00 += a * (m00 * m00 + m10 * m10);
      d01 += a * (m00 * m01 + m10 * m11);
      d11 += a * (m01 * m01 + m11 * m11);
      g0 -= a * (m00 * r0 + m10 * r1);
      g1 -= a * (m01 * r0 + m11 * r1);
      const int fd = C.freeof[(C.meta[j] >> 12) & 0xfff];
      if (fd >= 0 && fd < f) {  // block (f, fd) = a J_s^T J_d = -a M^T
        H0[2 * fd] -= a * m00;
        H0[2 * fd + 1] -= a * m10;
        H1[2 * fd] -= a * m01;
        H1[2 * fd + 1] -= a * m11;
      }
    }
    for (int t = C.inptr[l]; t < C.inptr[l + 1]; ++t) {
      const int j = C.inlist[t];
      const double a = C.scr[j];
      d00 += a;
      d11 += a;
      g0 += a * C.scr[E + j];
      g1 += a * C.scr[2 * E + j];
      const int fs = C.freeof[C.meta[j] & 0xfff];
      if (fs >= 0 && fs < f) {  // block (f, fs) = a J_d^T J_s = -a M
        H0[2 * fs] -= a * C.scr[3 * E + j];
        H0[2 * fs + 1] -= a * C.scr[4 * E + j];
        H1[2 * fs] -= a * C.scr[5 * E + j];
        H1[2 * fs + 1] -= a * C.scr[6 * E + j];
      }
    }
    H0[2 * f] = d00;
    H1[2 * f] = d01;
    H1[2 * f + 1] = d11;
    C.g[2 * f] = g0;
    C.g[2 * f + 1] = g1;
    if (first) {
      C.S[2 * f] = 1.0 / (1.0 + sqrt(d00));
      C.S[2 * f + 1] = 1.0 / (1.0 + sqrt(d11));
    }
  }
  __syncwarp();
  double gmax = 0.0;
  for (int i = C.lane; i < C.n; i += 32) {  // scale row i, projected gradient
    double* Hi = C.H + tri(i);
    const double si = C.S[i];
    for (int j = 0; j <= i; ++j) Hi[j] *= si * C.S[j];
    const int l = C.lof[i >> 1];
    const double xi = C.x[2 * l + (i & 1)];
    const double p = fmin(fmax(xi - C.g[i], -K.bound), K.bound);
    gmax = fmax(gmax, fabs(xi - p));
  }
  gmax = warp_max(gmax);
  __syncwarp();
  return gmax;
}

// Solve (S H S + D^2) y = S g exactly (dense Cholesky, rhs as extra row),
// write dl = -S y.  Returns false on a non-positive pivot / non-finite step.
// model_cost_change = y'Sg - y'(SHS)y/2 = (y'Sg + y'D^2 y)/2.
__device__ __forceinline__ bool lm_step(const WarpCtx& C, double radius, const DevConsts& K,
                                        double* model_change) {
  const int n = C.n;
  for (int i = C.lane; i < tri(n); i += 32) C.A[i] = C.H[i];
  __syncwarp();
  double* An = C.A + tri(n);
  for (int i = C.lane; i < n; i += 32) {
    const double hii = C.H[tri(i) + i];
    const double d2 = fmin(fmax(hii, K.min_diag), K.max_diag) / radius;
    C.A[tri(i) + i] = hii + d2;
    An[i] = C.S[i] * C.g[i];
  }
  __syncwarp();
  bool ok = true;
  for (int j = 0; j < n; ++j) {
    const double* Aj = C.A + tri(j);
    // rows j + lane + 32 p of this column, all passes in ONE k-loop: four
    // independent accumulators share the broadcast load of A[j][k]
    double s[4];
    const double* Ar[4];
    const int npass = (n - j) / 32 + 1;  // passes that have at least one live row (warp-uniform)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int i = j + C.lane + 32 * p;
      const bool live = i <= n;
      Ar[p] = C.A + tri(live ? i : j);  // dead lanes shadow row j (harmless, never stored)
      s[p] = Ar[p][j];
    }
    if (npass == 1) {
      for (int k = 0; k < j; ++k) s[0] -= Ar[0][k] * Aj[k];
    } else if (npass == 2) {
      for (int k = 0; k < j; ++k) {
        const double ajk = Aj[k];
        s[0] -= Ar[0][k] * ajk;
        s[1] -= Ar[1][k] * ajk;
      }
    } else {
      for (int k = 0; k < j; ++k) {
        const double ajk = Aj[k];
#pragma unroll
        for (int p = 0; p < 4; ++p) s[p] -= Ar[p][k] * ajk;
      }
    }
    const double sjj = __shfl_sync(kFull, s[0], 0);
    if (!(sjj > 0.0) || !isfinite(sjj)) {
      ok = false;
      break;
    }
    const double rs = rsqrt(sjj);
    __syncwarp();  // every lane's reads of column j / row j are done before the column is overwritten
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int i = j + C.lane + 32 * p;
      if (i <= n) C.A[tri(i) + j] = s[p] * rs;
    }
    if (C.lane == 0) C.dinv[j] = rs;
    __syncwarp();
  }
  if (!ok) return false;
  // back substitution L^T y = z, z = row n of A; lane holds y[lane + 32 p]
  double z[3];
#pragma unroll
  for (int p = 0; p < 3; ++p) z[p] = (C.lane + 32 * p < n) ? An[C.lane + 32 * p] : 0.0;
  for (int i = n - 1; i >= 0; --i) {
    const double* Li = C.A + tri(i);
    const int slot = i >> 5;
    double yi = (slot == 0 ? z[0] : (slot == 1 ? z[1] : z[2])) * C.dinv[i];
    yi = __shfl_sync(kFull, yi, i & 31);
#pragma unroll
    for (int p = 0; p < 3; ++p)
      if (C.lane + 32 * p < i) z[p] -= Li[C.lane + 32 * p] * yi;
    if (C.lane == (i & 31)) {
      if (slot == 0) z[0] = yi; else if (slot == 1) z[1] = yi; else z[2] = yi;
    }
  }
  double mc = 0.0;
  bool finite = true;
#pragma unroll
  for (int p = 0; p < 3; ++p) {
    const int i = C.lane + 32 * p;
    if (i < n) {
      const double y = z[p];
      const double hii = C.H[tri(i) + i];
      const double d2 = fmin(fmax(hii, K.min_diag), K.max_diag) / radius;
      const double si = C.S[i];
      mc += y * (si * C.g[i] + d2 * y);
      C.dl[i] = -si * y;
      finite = finite && isfinite(y);
    }
  }
  *model_change = 0.5 * warp_sum(mc);
  finite = __all_sync(kFull, finite);
  __syncwarp();
  return finite;
}

// xc = P(x + alpha dl) for free nodes, x for constants.
__device__ __forceinline__ void make_candidate(const WarpCtx& C, double alpha, const DevConsts& K) {
  for (int i = C.lane; i < 2 * C.Nc; i += 32) {
    const int f = C.freeof[i >> 1];
    double v = C.x[i];
    if (f >= 0) v = fmin(fmax(v + alpha * C.dl[2 * f + (i & 1)], -K.bound), K.bound);
    C.xc[i] = v;
  }
  __syncwarp();
}

// The warp tier's primitives as the driver's operations (see lfr_lm.cuh).
struct WarpTier {
  static constexpr int kStride = 32;
  static constexpr unsigned kTier = LmProfile::kWarp;
  static constexpr int kPolyWord = LmProfile::kTierWord;
  static constexpr bool kSkipFailingContraction = false;  // see lm_solve
  WarpCtx& C;
  const DevConsts& K;
  __device__ int tid() const { return C.lane; }
  __device__ int lane() const { return C.lane; }
  __device__ bool lead() const { return C.lane == 0; }
  __device__ double eval_x() { return eval_pass(C, C.x, K); }
  __device__ double assemble(bool first) { return lfr::assemble(C, first, K); }
  __device__ bool lm_step(double radius, double* model_change, double* gd, double* dmax) {
    if (!lfr::lm_step(C, radius, K, model_change) || !(*model_change > 0.0)) return false;
    double dot = 0.0, mx = 0.0;
    for (int i = C.lane; i < C.n; i += 32) {
      dot += C.g[i] * C.dl[i];
      mx = fmax(mx, fabs(C.dl[i]));
    }
    *gd = warp_sum(dot);
    *dmax = warp_max(mx);
    return true;
  }
  __device__ double trial(double alpha) {
    make_candidate(C, alpha, K);
    return eval_pass(C, C.xc, K);
  }
  __device__ double trial_slope(double alpha, double* dphi) {
    const double cost = trial(alpha);
    if (isfinite(cost)) *dphi = staged_grad_dot(C);
    return cost;
  }
  __device__ double slope() { return staged_grad_dot(C); }
  __device__ double restore_full_step() { return trial(1.0); }
  __device__ void scale_step(double s) {
    for (int i = C.lane; i < C.n; i += 32) C.dl[i] *= s;
    __syncwarp();
  }
  __device__ double free_norm(const double* a, const double* b) {  // |a - b|_2 over free coordinates (b may be null)
    double acc = 0.0;
    for (int i = C.lane; i < C.n; i += 32) {
      const int l = C.lof[i >> 1];
      const double v = a[2 * l + (i & 1)] - (b ? b[2 * l + (i & 1)] : 0.0);
      acc += v * v;
    }
    const double r = sqrt(warp_sum(acc));
    __syncwarp();  // reads above are ordered before later writes of x (shuffles are not a memory barrier)
    return r;
  }
  __device__ double x_norm() { return free_norm(C.x, nullptr); }
  __device__ double step_norm() { return free_norm(C.x, C.xc); }
  __device__ double accept() {
    for (int i = C.lane; i < 2 * C.Nc; i += 32) C.x[i] = C.xc[i];
    __syncwarp();
    return free_norm(C.x, nullptr);
  }
  __device__ void reject() {}  // lm_step reads H and g, which only assemble() writes
  __device__ unsigned long long counter() const { return 0; }
};

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 16 / WARPS)
solve_warp_kernel(const DevProblem P, const DevConsts K, const WarpBucket B) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t item = blockIdx.x * WARPS + wib;
  if (item >= B.n) return;  // warps are independent: no block-level barrier anywhere
  const uint32_t c = B.list[item];
  unsigned char* base = smem_raw + (size_t)wib * B.smem_per_warp;
  const WarpLayout L(B.emax, B.ncmax, B.n2max);
  WarpCtx C;
  C.lane = lane;
  C.emax = B.emax;
  C.x = (double*)(base + L.x);
  C.xc = (double*)(base + L.xc);
  C.g = (double*)(base + L.g);
  C.S = (double*)(base + L.S);
  C.dl = (double*)(base + L.dl);
  C.dinv = (double*)(base + L.dinv);
  C.H = (double*)(base + L.H);
  C.A = (double*)(base + L.A);
  C.scr = (double*)(base + L.scr);
  C.eidx = (uint32_t*)(base + L.eidx);
  C.meta = (uint32_t*)(base + L.meta);
  C.node = (uint32_t*)(base + L.node);
  uint32_t* rowstart = (uint32_t*)(base + L.rowstart);
  uint32_t* candptr = (uint32_t*)(base + L.candptr);
  C.inlist = (uint16_t*)(base + L.inlist);
  C.outptr = (uint16_t*)(base + L.outptr);
  C.inptr = (uint16_t*)(base + L.inptr);
  C.freeof = (int16_t*)(base + L.freeof);
  C.lof = (uint16_t*)(base + L.lof);
  C.edges = P.edges;

  LmProfile prof(P, c, lane == 0);
  // ---- component setup (solve.cc:98-143) --------------------------------------
  const int Eup = load_nodes(C, rowstart, candptr, P, K, c, lane);
  const int Nc = C.Nc;
  // kept out-edges; this tier reads their records from global memory by index
  int kept = 0;
  for (int k0 = 0; k0 < Eup; k0 += 32) {
    const int k = k0 + lane;
    EdgeClass ec{false, 0u, 0u};
    uint32_t e = 0;
    int lo = 0;
    if (k < Eup) {
      lo = cand_node(candptr, Nc, k);
      e = rowstart[lo] + (uint32_t)(k - (int)candptr[lo]);
      ec = classify_edge(P, C.node, Nc, C.node[lo], __float_as_uint(__ldg(&P.edges[5 * (size_t)e + 4].w)));
    }
    const unsigned m = __ballot_sync(kFull, ec.keep);
    if (ec.keep) {
      const int pos = kept + __popc(m & ((1u << lane) - 1u));
      C.eidx[pos] = e;
      C.meta[pos] = (uint32_t)lo | (ec.dl << 12) | (ec.kind << 24);
    }
    kept += __popc(m);
  }
  __syncwarp();
  const int Ec = kept;
  C.Ec = Ec;
  // out/in edge ranges per node, free-variable numbering
  int orun = 0, irun = 0, frun = 0;
  for (int l0 = 0; l0 < Nc; l0 += 32) {
    const int l = l0 + lane;
    int co = 0, ci = 0;
    for (int j = 0; j < Ec; ++j) {
      const uint32_t mt = C.meta[j];
      co += ((int)(mt & 0xfff) == l);
      ci += ((int)((mt >> 12) & 0xfff) == l);
    }
    if (l >= Nc) co = ci = 0;
    const int so = warp_incl_scan(co, lane), si = warp_incl_scan(ci, lane);
    const bool is_free = (l < Nc) && (co + ci > 0) && !P.is_root[C.node[l < Nc ? l : 0]];
    const int sf = warp_incl_scan(is_free ? 1 : 0, lane);
    if (l < Nc) {
      C.outptr[l] = (uint16_t)(orun + so - co);
      C.inptr[l] = (uint16_t)(irun + si - ci);
      C.freeof[l] = is_free ? (int16_t)(frun + sf - 1) : (int16_t)-1;
      if (is_free) C.lof[frun + sf - 1] = (uint16_t)l;
    }
    orun += __shfl_sync(kFull, so, 31);
    irun += __shfl_sync(kFull, si, 31);
    frun += __shfl_sync(kFull, sf, 31);
  }
  if (lane == 0) {
    C.outptr[Nc] = (uint16_t)orun;
    C.inptr[Nc] = (uint16_t)irun;
  }
  __syncwarp();
  for (int l0 = 0; l0 < Nc; l0 += 32) {
    const int l = l0 + lane;
    int w = (l < Nc) ? C.inptr[l] : 0;
    for (int j = 0; j < Ec; ++j)
      if (l < Nc && (int)((C.meta[j] >> 12) & 0xfff) == l) C.inlist[w++] = (uint16_t)j;
  }
  C.nf = frun;
  C.n = 2 * frun;
  __syncwarp();
  WarpTier T{C, K};
  lm_solve(T, P, K, c, prof);
}

// Test hook: the line search's step-size selection (hermite_minimizer) on caller-supplied
// samples, one warp per case (lfr_debug_ls_minimizer).  in[c] = {f0, g0, x1, f1, g1, three,
// x2, f2, g2, lo, hi}.
__global__ void ls_minimizer_kernel(const double* __restrict__ in, int n, double* __restrict__ out) {
  const int wid = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (wid >= n) return;  // whole warps leave together
  const double* s = in + 11 * (size_t)wid;
  const double x = hermite_minimizer(s[0], s[1], s[2], s[3], s[4], s[5] != 0.0, s[6], s[7], s[8], s[9], s[10], lane);
  if (lane == 0) out[wid] = x;
}

// Test hook: the line search's quartic root finders on caller-supplied polynomials,
// one warp per polynomial (lfr_debug_quartic_roots).
__global__ void quartic_roots_kernel(const double* __restrict__ coef, const double* __restrict__ lohi, int n,
                                     int use_grid, double* __restrict__ roots, int* __restrict__ counts) {
  const int wid = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (wid >= n) return;  // whole warps leave together
  const double q[5] = {coef[5 * wid], coef[5 * wid + 1], coef[5 * wid + 2], coef[5 * wid + 3], coef[5 * wid + 4]};
  double out[4] = {0.0, 0.0, 0.0, 0.0};
  long long pp = 0;
  const int c = use_grid ? quartic_roots_grid(q, lohi[2 * wid], lohi[2 * wid + 1], out, lane, pp)
                         : quartic_roots_in(q, lohi[2 * wid], lohi[2 * wid + 1], out, lane, pp);
  if (lane == 0) {
    counts[wid] = c;
    for (int k = 0; k < 4; ++k) roots[4 * wid + k] = out[k];
  }
}

// K1 test hook: one thread per edge.
__global__ void edge_eval_kernel(const float4* edges, const uint8_t* kind, uint64_t n, const double* xs,
                                 const double* xd, const DevConsts K, double* r, double* jac, double* rho) {
  const uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  float4 q[5];
#pragma unroll
  for (int t = 0; t < 5; ++t) q[t] = __ldg(edges + 5 * e + t);
  const EdgeEval ev = eval_edge(q, kind[e], xs[2 * e], xs[2 * e + 1], xd[2 * e], xd[2 * e + 1], K);
  r[2 * e] = ev.r0;
  r[2 * e + 1] = ev.r1;
  jac[4 * e] = -ev.m00;
  jac[4 * e + 1] = -ev.m01;
  jac[4 * e + 2] = -ev.m10;
  jac[4 * e + 3] = -ev.m11;
  rho[3 * e] = 2.0 * ev.half_rho;
  rho[3 * e + 1] = ev.a;
  rho[3 * e + 2] = 0.0;  // rho'' is not used by the solve (always <= 0, A.3)
}

}  // namespace lfr
