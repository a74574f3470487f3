// lfr_oracle.cc — CPU ORACLE for the multi-view refinement solve.
//
// TEST INFRASTRUCTURE ONLY.  Nothing in the product path (the package
// local-feature-refinement_b200/, the solve launcher, the `value`/`e2e` legs of
// bench.py) may import, link or execute this file; only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
// do, and only as the checker or the timed CPU baseline.
//
// PARITY: PINNED AT THE REFERENCE'S OWN SOURCES, UNPINNED INSIDE CERES.  The
// arithmetic of the reference's hot path lives in Ceres Solver (un-vendored,
// version unpinned by the reference; CMakeLists.txt:9 `find_package(Ceres
// REQUIRED)`, `-std=c++11` => Ceres 1.13/1.14 era); neither Ceres, Eigen,
// COLMAP, Boost nor protoc exist in this image and the reference ships no tests
// or golden vectors.  What IS pinned: interpolate() / the residual and its
// Jacobian are bitwise equal to the reference's cost.cc compiled unmodified
// against shim headers (oracle/_ref/libref_cost.so, tests/test_ref_cost.py), and
// the whole pipeline is compared with the reference's solve.cc compiled the same
// way (oracle/_ref/solve, tests/test_ref_solve.py).  What is NOT: the internals
// of Ceres itself (no Ceres binary to run).  This file restates
//   * multi-view-refinement/cost.cc:13-48   (BiquadraticInterpolator::Evaluate)
//   * multi-view-refinement/cost.cc:78-90   (InterpolatedCostFunctor)
//   * multi-view-refinement/solve.cc:79-160 (create_and_solve_problem)
//   * multi-view-refinement/solve.cc:614-635 (thread-pool dispatch)
// and the published algorithm of Ceres Solver 1.14's bounds-constrained
// Levenberg-Marquardt trust-region minimizer (trust_region_minimizer.cc,
// levenberg_marquardt_strategy.cc, trust_region_step_evaluator.cc,
// line_search.cc, polynomial.cc, loss_function.cc, corrector.cc,
// residual_block.cc, parameter_block.h; SURVEY.md Appendix A).  What pins it
// instead: the analytic known-answer tests in tests/test_oracle_kat.py and an
// independent scipy minimum check (tests/test_oracle_scipy.py).
//
// Exports the same C ABI as the product library (include/lfr.h), plus a few
// lfr_ref_* hooks that expose the inner functions to the tests.
//
// Build: oracle/build.py  (g++ -O2 -ffp-contract=off: no FMA contraction, so the
// interpolator rounds exactly like the reference's -O0 build).

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <complex>
#include <cstring>
#include <limits>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../include/lfr.h"
#include "ceres/ceres.h"  // oracle/ref_shims: the literal polynomial.cc restatement (ceres::shim)

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

// ---------------------------------------------------------------------------
// cost.cc:13-48 — biquadratic (3x3 Lagrange) interpolation of a 2-channel grid
// sampled at {-0.5, 0, +0.5}^2, with clamping.  D[2*(3*i+j)+k].
// ---------------------------------------------------------------------------
void interpolate(const double* D, double row, double col, double* f,
                 double* dfdrow, double* dfdcol) {
  const double row_in = row, col_in = col;
  row = std::max(std::min(row, .5), -.5);  // cost.cc:17
  col = std::max(std::min(col, .5), -.5);  // cost.cc:18
  // Lagrange bases and their derivatives, expression order of cost.cc:20-23.
  const double Lr[3] = {2. * row * (row - .5), (-4.) * (row - .5) * (row + .5),
                        2. * row * (row + .5)};
  const double dLr[3] = {2. * row + 2. * (row - .5),
                         (-4.) * (row - .5) + (-4.) * (row + .5),
                         2. * row + 2. * (row + .5)};
  const double Lc[3] = {2. * col * (col - .5), (-4.) * (col - .5) * (col + .5),
                        2. * col * (col + .5)};
  const double dLc[3] = {2. * col + 2. * (col - .5),
                         (-4.) * (col - .5) + (-4.) * (col + .5),
                         2. * col + 2. * (col + .5)};
  const bool row_free = (row_in == row);  // cost.cc:38
  const bool col_free = (col_in == col);  // cost.cc:41
  for (int k = 0; k < 2; ++k) {
    double v = 0., vr = 0., vc = 0.;
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) {
        const double d = D[2 * (3 * i + j) + k];
        v += Lr[i] * Lc[j] * d;                    // cost.cc:35
        if (row_free) vr += dLr[i] * Lc[j] * d;    // cost.cc:39
        if (col_free) vc += Lr[i] * dLc[j] * d;    // cost.cc:42
      }
    }
    f[k] = v;
    if (dfdrow) {
      dfdrow[k] = vr;
      dfdcol[k] = vc;
    }
  }
}

// ---------------------------------------------------------------------------
// Loss functions (Ceres loss_function.cc), wrapped in ScaledLoss(., sim).
// ---------------------------------------------------------------------------
void loss_eval(int kind, double sim, double s, const lfr_options& o,
               double rho[3]) {
  if (kind == LFR_EDGE_CAUCHY) {
    const double b = o.cauchy_a * o.cauchy_a, c = 1.0 / b;
    const double sum = 1.0 + s * c;
    const double inv = 1.0 / sum;
    rho[0] = b * std::log(sum);
    rho[1] = std::max(std::numeric_limits<double>::min(), inv);
    rho[2] = -c * (inv * inv);
  } else {
    const double a2 = o.tukey_a * o.tukey_a;
    if (s <= a2) {
      const double value = 1.0 - s / a2;
      const double value_sq = value * value;
      if (o.tukey_variant == 2) {  // Ceres 2.x
        rho[0] = a2 / 3.0 * (1.0 - value_sq * value);
        rho[1] = value_sq;
        rho[2] = -2.0 / a2 * value;
      } else {  // Ceres 1.x
        rho[0] = a2 / 6.0 * (1.0 - value_sq * value);
        rho[1] = 0.5 * value_sq;
        rho[2] = -1.0 / a2 * value;
      }
    } else {
      rho[0] = (o.tukey_variant == 2) ? a2 / 3.0 : a2 / 6.0;
      rho[1] = 0.0;
      rho[2] = 0.0;
    }
  }
  rho[0] *= sim;  // ScaledLoss::Evaluate
  rho[1] *= sim;
  rho[2] *= sim;
}

// ---------------------------------------------------------------------------
// polynomial.cc — the interpolating polynomial of the Armijo line search and
// its bounded minimisation.
//
// Ceres (FindInterpolatingPolynomial + MinimizePolynomial) fits the polynomial
// through {value, gradient} at step 0, at the current trial step and, from the
// second contraction on, at the previous one, by a 4x4 / 6x6 Vandermonde solve
// (Eigen fullPivLu), and takes the minimiser over [x_min, x_max] among: interval
// middle, both ends, the real parts of all roots of p' (closed forms up to
// degree 2, eigenvalues of the balanced companion matrix above), and the sample
// abscissae.  The restatement builds the SAME polynomial in the normalised
// variable t = x / h (h = largest sample step): the two constraints at 0 fix
// the two lowest coefficients, the others come from a 2x2 solve (closed form) or
// from the divided differences of the reduced cubic; of the companion-matrix eigenvalues only the real
// ones inside the interval can win the minimisation, and those are bracketed
// exactly (real_roots_in).  csrc/lfr_math.cuh mirrors this operation for operation
// (and additionally has a lane-parallel route to the same quartic roots, checked
// against this one by the GPU tests).
// ---------------------------------------------------------------------------
struct Sample {
  double x = 0, value = 0, gradient = 0;
  bool value_valid = false, gradient_valid = false;
};

double poly_eval(const double* p, int n, double x) {
  double v = 0.0;
  for (int i = 0; i < n; ++i) v = v * x + p[i];
  return v;
}

// Line-search interpolation mode.
//   0 (default) LITERAL: Ceres' polynomial.cc as written — Vandermonde system in the raw step
//     sizes solved by full-pivot LU, critical points = real parts of ALL eigenvalues of the
//     balanced companion matrix (ceres::shim::MinimizeInterpolatingPolynomial in
//     oracle/ref_shims/mini_ceres.cc).  This is what the GPU is compared with.
//   1 FAST: the normalised-variable / bracketed-real-roots formulation below, which the CUDA
//     path mirrors operation for operation (lfr_math.cuh).  Kept so that the two can be compared
//     state by state (tests/test_linesearch_modes.py).
std::atomic<int> g_ls_mode(0);
// Optional recording of every line-search interpolation state {f0, g0, x1, f1, g1, three, x2, f2,
// g2, lo, hi} (the input format of lfr_debug_ls_minimizer) for the mode-comparison tests.
std::atomic<bool> g_harvest(false);
std::mutex g_harvest_mutex;
std::vector<double> g_harvested;

// ---- real roots of a polynomial inside an interval ---------------------------
// MinimizePolynomial looks at the real parts of ALL roots of p', but a candidate
// only wins if its value is strictly below the best of {middle, ends}; on an
// interval the minimum of p is attained at an end or at a REAL critical point
// inside it, so complex roots and roots outside [lo, hi] can never be selected.
// The real roots inside the interval are found exactly and cheaply by
// recursion on the derivative: between two consecutive critical points a
// polynomial is monotone, so every sign change brackets exactly one root, which
// a safeguarded Newton iteration (Numerical Recipes' rtsafe) then polishes.
void horner2(const double* q, int nq, double x, double* f, double* df) {
  double v = q[0], d = 0.0;
  for (int i = 1; i < nq; ++i) {
    d = d * x + v;
    v = v * x + q[i];
  }
  *f = v;
  *df = d;
}

// f / df for the Newton step.  The step only has to be accurate enough to keep
// the quadratic convergence, so the quotient uses the correctly rounded SINGLE
// precision reciprocal of df (relative error 2^-24; bit-identical on CPU and in
// CUDA's __frcp_rn) instead of a double division, which is the longest
// dependent chain of the iteration on the GPU.  Outside the safe single
// precision range it is the plain division.
double newton_quotient(double f, double df) {
  const double adf = std::fabs(df);
  if (!(adf > 1e-30 && adf < 1e30)) return f / df;
  const float r = 1.0f / static_cast<float>(df);
  return f * static_cast<double>(r);
}

// One real root of q inside the bracket [a, b] (opposite signs at the ends, q monotone there):
// Newton from the regula-falsi point, bisection whenever a step would leave the shrinking bracket;
// stops after a Newton step of relative size <= 1e-8 (quadratic convergence: error ~1e-16 afterwards; the
// 6e-8 relative error of newton_quotient only adds 6e-8 * 1e-8).  Same operations as
// csrc/lfr_math.cuh::bracket_root.
double bracket_root(const double* q, int nq, double a, double b, double fa, double fb) {
  if (fa == 0.0) return a;
  if (fb == 0.0) return b;
  double xl = fa < 0.0 ? a : b, xh = fa < 0.0 ? b : a;
  double x = a - fa * newton_quotient(b - a, fb - fa);
  if (!(x > std::fmin(a, b) && x < std::fmax(a, b))) x = 0.5 * (a + b);
  for (int it = 0; it < 100; ++it) {
    double f, df;
    horner2(q, nq, x, &f, &df);
    if (f == 0.0) return x;
    if (f < 0.0) xl = x; else xh = x;
    double dx = newton_quotient(f, df);
    double xn = x - dx;
    if (xn == x) return x;  // converged to the last bit (checked before the bracket test: x itself is one end of the bracket)
    if (!(xn >= std::fmin(xl, xh) && xn <= std::fmax(xl, xh))) {
      xn = 0.5 * (xl + xh);
      dx = std::numeric_limits<double>::quiet_NaN();  // no stop after a bisection step
    }
    if (xn == x) return x;
    x = xn;
    if (std::fabs(dx) <= 1e-8 * std::fabs(x)) return x;
  }
  return x;
}

// Roots of q in the segments cut out of [lo, hi] by its sorted critical points
// brk[0..nbrk): q is monotone on each segment, so a sign change brackets exactly
// one root.  (The CUDA path runs the segments on separate lanes.)
int segment_roots(const double* q, int nq, const double* brk, int nbrk, double lo, double hi, double* out) {
  int cnt = 0;
  for (int s = 0; s <= nbrk; ++s) {
    const double xa = (s == 0) ? lo : brk[s - 1];
    const double xb = (s < nbrk) ? brk[s] : hi;
    double fa, fb, tmp;
    horner2(q, nq, xa, &fa, &tmp);
    horner2(q, nq, xb, &fb, &tmp);
    const bool has = ((fa <= 0.0 && fb >= 0.0) || (fa >= 0.0 && fb <= 0.0)) && !(fa == 0.0 && fb == 0.0);
    if (!has) continue;
    const double r = bracket_root(q, nq, xa, xb, fa, fb);
    if (cnt == 0 || r != out[cnt - 1]) out[cnt++] = r;
  }
  return cnt;
}

// Real roots inside [lo, hi] of a polynomial of degree <= 3, ascending.
// Degree <= 2: the closed forms of Ceres' polynomial.cc.
int roots_upto3(const double* c, int n, double lo, double hi, double* out) {
  int lead = 0;
  while (lead + 1 < n && c[lead] == 0.0) ++lead;  // RemoveLeadingZeros
  const double* p = c + lead;
  const int degree = n - lead - 1;
  if (degree <= 0) return 0;
  int cnt = 0;
  if (degree == 1) {
    const double r = -p[1] / p[0];
    if (r >= lo && r <= hi) out[cnt++] = r;
    return cnt;
  }
  if (degree == 2) {  // FindQuadraticPolynomialRoots, real case
    const double a = p[0], b = p[1], cc = p[2];
    const double D = b * b - 4 * a * cc;
    if (D < 0) return 0;
    const double sq = std::sqrt(D);
    double r0, r1;
    if (b >= 0) {
      r0 = (-b - sq) / (2.0 * a);
      r1 = (2.0 * cc) / (-b - sq);
    } else {
      r0 = (2.0 * cc) / (-b + sq);
      r1 = (-b + sq) / (2.0 * a);
    }
    if (r1 < r0) std::swap(r0, r1);
    if (r0 >= lo && r0 <= hi) out[cnt++] = r0;
    if (r1 >= lo && r1 <= hi && r1 != r0) out[cnt++] = r1;
    return cnt;
  }
  const double d[3] = {3.0 * p[0], 2.0 * p[1], p[2]};  // critical points of the cubic
  double crit[2] = {0.0, 0.0};
  const int ncrit = roots_upto3(d, 3, lo, hi, crit);
  return segment_roots(p, 4, crit, ncrit, lo, hi, out);
}

// Real roots of c[0..n-1] (highest degree first, degree <= 4) inside [lo, hi], ascending.
int real_roots_in(const double* c, int n, double lo, double hi, double* out) {
  int lead = 0;
  while (lead + 1 < n && c[lead] == 0.0) ++lead;
  if (n - lead - 1 <= 3) return roots_upto3(c + lead, n - lead, lo, hi, out);
  const double* p = c + lead;  // quartic
  const double d[4] = {4.0 * p[0], 3.0 * p[1], 2.0 * p[2], p[3]};
  double crit[3] = {0.0, 0.0, 0.0};
  const int ncrit = roots_upto3(d, 4, lo, hi, crit);
  return segment_roots(p, 5, crit, ncrit, lo, hi, out);
}

// MinimizeInterpolatingPolynomial for the samples (0, f0, g0), (x1, f1, g1)
// [, (x2, f2, g2)] over [lo, hi]; returns the minimiser, *value = p(minimiser).
double hermite_minimizer(double f0, double g0, double x1, double f1, double g1, bool three, double x2,
                         double f2, double g2, double lo, double hi, double* value) {
  const double h = three ? std::max(x1, x2) : x1;
  const double ih = 1.0 / h;  // the only division by h: t = x * ih
  const double g0h = g0 * h;
  double c[6];
  int nc;
  if (!three) {
    const double u = f1 - f0 - g0h, v = (g1 - g0) * h;
    c[0] = v - 2.0 * u;
    c[1] = 3.0 * u - v;
    c[2] = g0h;
    c[3] = f0;
    nc = 4;
  } else {
    // p(t) = f0 + g0h t + t^2 s(t): s is the cubic Hermite interpolant of
    // S = (p - f0 - g0h t) / t^2 and its derivative D at ta and tb, written in
    // Newton's divided differences and expanded to monomials.  Three independent
    // reciprocals instead of the four dependent pivots of a 4x4 elimination.
    const double ta = x1 * ih, tb = x2 * ih;
    const double ita = 1.0 / ta, itb = 1.0 / tb, iw = 1.0 / (tb - ta);
    const double ita2 = ita * ita, itb2 = itb * itb;
    const double Sa = (f1 - f0 - g0h * ta) * ita2;
    const double Sb = (f2 - f0 - g0h * tb) * itb2;
    const double Da = ((g1 - g0) * h - 2.0 * ta * Sa) * ita2;
    const double Db = ((g2 - g0) * h - 2.0 * tb * Sb) * itb2;
    const double m = (Sb - Sa) * iw;
    const double e2 = (m - Da) * iw;
    const double e3 = ((Db - m) - (m - Da)) * iw * iw;
    c[0] = e3;
    c[1] = e2 - e3 * (2.0 * ta + tb);
    c[2] = Da + ta * (e3 * (ta + 2.0 * tb) - 2.0 * e2);
    c[3] = Sa + ta * (ta * (e2 - e3 * tb) - Da);
    c[4] = g0h;
    c[5] = f0;
    nc = 6;
  }
  const double tlo = lo * ih, thi = hi * ih;
  double ox = (lo + hi) / 2.0;  // MinimizePolynomial starts from the middle
  double ov = poly_eval(c, nc, ox * ih);
  double v = poly_eval(c, nc, tlo);
  if (v < ov) { ov = v; ox = lo; }
  v = poly_eval(c, nc, thi);
  if (v < ov) { ov = v; ox = hi; }
  double der[5], roots[4];
  const int degree = nc - 1;
  for (int i = 0; i < degree; ++i) der[i] = (degree - i) * c[i];
  const int nr = real_roots_in(der, degree, tlo, thi, roots);
  for (int i = 0; i < nr; ++i) {
    if (roots[i] < tlo || roots[i] > thi) continue;
    v = poly_eval(c, nc, roots[i]);
    if (v < ov) { ov = v; ox = roots[i] * h; }
  }
  const double sx[3] = {0.0, x1, x2};
  for (int i = 0; i < (three ? 3 : 2); ++i) {
    if (sx[i] < lo || sx[i] > hi) continue;
    v = poly_eval(c, nc, sx[i] * ih);
    if (v < ov) { ov = v; ox = sx[i]; }
  }
  if (value) *value = ov;
  return ox;
}

// ---------------------------------------------------------------------------
// One component = one ceres::Problem (solve.cc:79-160).
// ---------------------------------------------------------------------------
struct Block {            // one kept residual block with >= 1 free end
  int src_local, dst_local;
  int src_free, dst_free;  // index of the free parameter block, or -1 (constant)
  int kind;
  double sim;
  double D[18];            // flow grid widened to double (solve.cc:460-472)
};

struct Component {
  std::vector<uint32_t> nodes;   // local -> global node index
  std::vector<double> pos;       // [2*nlocal] user state (in/out)
  std::vector<int> free_of;      // local -> free block index or -1
  std::vector<int> local_of_free;
  std::vector<Block> blocks;
  int n_free = 0;
};

struct EvalOut {
  double cost = 0;
  std::vector<double> r;    // [2*nb] corrected residuals
  std::vector<double> Js;   // [4*nb] corrected d r/d x_src (row-major 2x2)
  std::vector<double> Jd;   // [4*nb] corrected d r/d x_dst
  std::vector<double> grad; // [2*n_free]
};

// Position of local node l given the reduced state vector x.
inline const double* node_pos(const Component& C, const std::vector<double>& x, int l) {
  const int f = C.free_of[l];
  return f >= 0 ? &x[2 * f] : &C.pos[2 * l];
}

// ProgramEvaluator::Evaluate + ResidualBlock::Evaluate + Corrector.
// Cost is summed in residual-block order (num_threads = 1, solve.cc:148,632).
void evaluate(const Component& C, const lfr_options& o, const std::vector<double>& x,
              bool want_residuals, bool want_jacobian, bool want_gradient,
              EvalOut* out) {
  const size_t nb = C.blocks.size();
  const bool need_jac = want_jacobian || want_gradient;
  out->cost = 0.0;
  if (want_residuals) out->r.assign(2 * nb, 0.0);
  if (want_jacobian) {
    out->Js.assign(4 * nb, 0.0);
    out->Jd.assign(4 * nb, 0.0);
  }
  if (want_gradient) out->grad.assign(2 * C.n_free, 0.0);
  for (size_t b = 0; b < nb; ++b) {
    const Block& B = C.blocks[b];
    const double* x1 = node_pos(C, x, B.src_local);
    const double* x2 = node_pos(C, x, B.dst_local);
    double f[2], dr[2], dc[2];
    interpolate(B.D, x1[0], x1[1], f, need_jac ? dr : nullptr, need_jac ? dc : nullptr);
    // cost.cc:87  residuals = x2 - x1 - disp
    double r[2] = {x2[0] - x1[0] - f[0], x2[1] - x1[1] - f[1]};
    const double sq = r[0] * r[0] + r[1] * r[1];
    double rho[3];
    loss_eval(B.kind, B.sim, sq, o, rho);
    out->cost += 0.5 * rho[0];
    if (!want_residuals && !need_jac) continue;
    // Corrector: rho'' <= 0 for both losses => residual and Jacobian scaled by
    // sqrt(rho') (corrector.cc "common case").  Jacobian first, then residual.
    const double s1 = std::sqrt(rho[1]);
    double js[4], jd[4];
    if (need_jac) {
      // AutoDiff of (x2 - x1 - disp): d/dx1 = (0 - 1) - dfd., d/dx2 = 1.
      js[0] = (0.0 - 1.0) - dr[0];
      js[1] = (0.0 - 0.0) - dc[0];
      js[2] = (0.0 - 0.0) - dr[1];
      js[3] = (0.0 - 1.0) - dc[1];
      jd[0] = 1.0; jd[1] = 0.0; jd[2] = 0.0; jd[3] = 1.0;
      for (int t = 0; t < 4; ++t) {
        js[t] *= s1;
        jd[t] *= s1;
      }
    }
    r[0] *= s1;
    r[1] *= s1;
    if (want_residuals) {
      out->r[2 * b] = r[0];
      out->r[2 * b + 1] = r[1];
    }
    if (want_jacobian) {
      if (B.src_free >= 0) std::memcpy(&out->Js[4 * b], js, sizeof js);
      if (B.dst_free >= 0) std::memcpy(&out->Jd[4 * b], jd, sizeof jd);
    }
    if (want_gradient) {
      if (B.src_free >= 0) {
        out->grad[2 * B.src_free] += js[0] * r[0] + js[2] * r[1];
        out->grad[2 * B.src_free + 1] += js[1] * r[0] + js[3] * r[1];
      }
      if (B.dst_free >= 0) {
        out->grad[2 * B.dst_free] += jd[0] * r[0] + jd[2] * r[1];
        out->grad[2 * B.dst_free + 1] += jd[1] * r[0] + jd[3] * r[1];
      }
    }
  }
}

// Program::Plus with ParameterBlock::Plus: x + delta, projected on the box.
void plus(const std::vector<double>& x, const std::vector<double>& delta, double bound,
          std::vector<double>* out) {
  out->resize(x.size());
  for (size_t i = 0; i < x.size(); ++i) {
    double v = x[i] + delta[i];
    v = std::max(v, -bound);
    v = std::min(v, bound);
    (*out)[i] = v;
  }
}

double norm2(const std::vector<double>& v) {
  double s = 0;
  for (double a : v) s += a * a;
  return std::sqrt(s);
}

// Dense Cholesky solve of the SPD system A y = b (A is n x n, row-major, lower
// part used).  Stands in for SPARSE_NORMAL_CHOLESKY (solve.cc:147): an exact
// solve; ordering/sparsity only change round-off.
// Row i's entries left of its first nonzero `first[i]` (its profile) stay +0 in
// the factor, so the products with them are skipped.  In the factorisation and the
// forward substitution they are the leading terms of each sum, which starts from an
// entry of A or b (never -0): skipping them changes no bit.  In the back
// substitution they are signed zeros among the terms, which can at most flip the
// sign of an exact zero.  Long tracks and grids in natural order have a narrow
// profile, which keeps components of thousands of nodes within reach.
bool cholesky_solve(std::vector<double>& A, int n, const std::vector<double>& b,
                    std::vector<double>* y) {
  std::vector<int> first(n);
  for (int i = 0; i < n; ++i) {
    int k = 0;
    while (k < i && A[(size_t)i * n + k] == 0.0) ++k;
    first[i] = k;
  }
  for (int j = 0; j < n; ++j) {
    const double* Aj = &A[(size_t)j * n];
    double d = Aj[j];
    for (int k = first[j]; k < j; ++k) d -= Aj[k] * Aj[k];
    if (!(d > 0.0) || !std::isfinite(d)) return false;
    const double l = std::sqrt(d);
    A[(size_t)j * n + j] = l;
    for (int i = j + 1; i < n; ++i) {
      if (first[i] > j) continue;  // L(i, j) = +0
      double* Ai = &A[(size_t)i * n];
      double s = Ai[j];
      for (int k = std::max(first[i], first[j]); k < j; ++k) s -= Ai[k] * Aj[k];
      Ai[j] = s / l;
    }
  }
  y->assign(n, 0.0);
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int k = first[i]; k < i; ++k) s -= A[(size_t)i * n + k] * (*y)[k];
    (*y)[i] = s / A[(size_t)i * n + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = (*y)[i];
    for (int k = i + 1; k < n; ++k)
      if (first[k] <= i) s -= A[(size_t)k * n + i] * (*y)[k];
    (*y)[i] = s / A[(size_t)i * n + i];
  }
  for (int i = 0; i < n; ++i)
    if (!std::isfinite((*y)[i])) return false;
  return true;
}

struct SolveResult {
  int iterations = 0;
  int termination = LFR_TERM_EMPTY;
  double initial_cost = 0, final_cost = 0;
  int line_search_steps = 0;
};

// LineSearchFunction::Evaluate + ArmijoLineSearch::DoSearch (line_search.cc),
// as called by TrustRegionMinimizer::DoLineSearch.
void do_line_search(const Component& C, const lfr_options& o,
                    const std::vector<double>& x, const std::vector<double>& gradient,
                    double cost, std::vector<double>* delta, int* num_ls_iterations) {
  const int n = (int)x.size();
  double initial_gradient = 0.0;
  for (int i = 0; i < n; ++i) initial_gradient += gradient[i] * (*delta)[i];
  Sample initial;
  initial.x = 0.0;
  initial.value = cost;
  initial.gradient = initial_gradient;
  initial.value_valid = initial.gradient_valid = true;
  double dir_max = 0.0;
  for (double d : *delta) dir_max = std::max(dir_max, std::fabs(d));
  Sample previous;  // invalid
  Sample current;
  EvalOut ev;
  std::vector<double> scaled(n), px;
  auto evaluate_at = [&](double step, Sample* s) {
    *s = Sample();
    s->x = step;
    for (int i = 0; i < n; ++i) scaled[i] = step * (*delta)[i];
    plus(x, scaled, o.bound, &px);
    evaluate(C, o, px, false, false, true, &ev);  // CUBIC => gradient too
    if (!std::isfinite(ev.cost)) return;
    s->value = ev.cost;
    s->value_valid = true;
    double g = 0.0;
    for (int i = 0; i < n; ++i) g += (*delta)[i] * ev.grad[i];
    if (!std::isfinite(g)) return;
    s->gradient = g;
    s->gradient_valid = true;
  };
  evaluate_at(1.0, &current);
  int iters = 0;
  while (!current.value_valid ||
         current.value > cost + o.line_search_sufficient_function_decrease *
                                    initial_gradient * current.x) {
    ++iters;
    ++*num_ls_iterations;
    if (iters >= o.max_num_line_search_step_size_iterations) return;  // failed
    const double min_step = o.max_line_search_step_contraction * current.x;
    const double max_step = o.min_line_search_step_contraction * current.x;
    double step_size;
    if (g_harvest.load() && current.value_valid && current.gradient_valid &&
        !(previous.value_valid && !previous.gradient_valid)) {
      const double st[11] = {initial.value, initial.gradient, current.x, current.value, current.gradient,
                             previous.value_valid ? 1.0 : 0.0, previous.x, previous.value, previous.gradient,
                             min_step, max_step};
      std::lock_guard<std::mutex> lock(g_harvest_mutex);
      g_harvested.insert(g_harvested.end(), st, st + 11);
    }
    if (g_ls_mode.load() == 0) {
      // LineSearch::InterpolatingPolynomialMinimizingStepSize, CUBIC: bisection only for an invalid
      // value; otherwise interpolate {lower bound, current [, previous]} with whatever is valid
      if (!current.value_valid) {
        step_size = std::min(std::max(current.x * 0.5, min_step), max_step);
      } else {
        double smp[15];
        int ns = 0;
        auto push = [&](const Sample& q) {
          smp[5 * ns] = q.x;
          smp[5 * ns + 1] = q.value;
          smp[5 * ns + 2] = q.gradient;
          smp[5 * ns + 3] = q.value_valid ? 1.0 : 0.0;
          smp[5 * ns + 4] = q.gradient_valid ? 1.0 : 0.0;
          ++ns;
        };
        push(initial);
        push(current);
        if (previous.value_valid) push(previous);
        double unused = 0.0;
        ceres::shim::MinimizeInterpolatingPolynomial(smp, ns, min_step, max_step, &step_size, &unused);
      }
    } else if (!current.value_valid || !current.gradient_valid ||
               (previous.value_valid && !previous.gradient_valid)) {
      // invalid sample (a non-finite gradient with a finite value needs overflow): bisection rule
      step_size = std::min(std::max(current.x * 0.5, min_step), max_step);
    } else {
      step_size = hermite_minimizer(initial.value, initial.gradient, current.x, current.value,
                                    current.gradient, previous.value_valid, previous.x, previous.value,
                                    previous.gradient, min_step, max_step, nullptr);
    }
    if (step_size * dir_max < o.min_line_search_step_size) return;  // failed
    previous = current;
    evaluate_at(step_size, &current);
  }
  for (double& d : *delta) d *= current.x;  // success
}

// TrustRegionMinimizer::Minimize (Ceres 1.14) with LevenbergMarquardtStrategy.
SolveResult minimize(Component& C, const lfr_options& o) {
  SolveResult R;
  const int n = 2 * C.n_free;
  if (n == 0) return R;  // "No non-constant parameter blocks found."
  const size_t nb = C.blocks.size();
  const double kMax = std::numeric_limits<double>::max();

  std::vector<double> x(n), best(n);
  for (int f = 0; f < C.n_free; ++f) {
    x[2 * f] = C.pos[2 * C.local_of_free[f]];
    x[2 * f + 1] = C.pos[2 * C.local_of_free[f] + 1];
  }
  // IterationZero: project the start point (is_constrained).
  {
    std::vector<double> zero(n, 0.0), px;
    plus(x, zero, o.bound, &px);
    x = px;
  }
  double x_norm = norm2(x);
  std::vector<double> scale(n, 1.0);  // jacobian_scaling_
  EvalOut J;                          // current linearisation (scaled columns)
  double x_cost = kMax, gradient_max_norm = 0.0;

  auto evaluate_gradient_and_jacobian = [&](bool first) {
    evaluate(C, o, x, true, true, true, &J);
    x_cost = J.cost;
    if (first) {  // jacobi_scaling: 1 / (1 + sqrt(squared column norm)), once
      std::vector<double> col(n, 0.0);
      for (size_t b = 0; b < nb; ++b) {
        const Block& B = C.blocks[b];
        if (B.src_free >= 0)
          for (int c = 0; c < 2; ++c)
            col[2 * B.src_free + c] += J.Js[4 * b + c] * J.Js[4 * b + c] +
                                       J.Js[4 * b + 2 + c] * J.Js[4 * b + 2 + c];
        if (B.dst_free >= 0)
          for (int c = 0; c < 2; ++c)
            col[2 * B.dst_free + c] += J.Jd[4 * b + c] * J.Jd[4 * b + c] +
                                       J.Jd[4 * b + 2 + c] * J.Jd[4 * b + 2 + c];
      }
      for (int i = 0; i < n; ++i) scale[i] = 1.0 / (1.0 + std::sqrt(col[i]));
    }
    for (size_t b = 0; b < nb; ++b) {  // ScaleColumns
      const Block& B = C.blocks[b];
      if (B.src_free >= 0)
        for (int rr = 0; rr < 2; ++rr)
          for (int c = 0; c < 2; ++c) J.Js[4 * b + 2 * rr + c] *= scale[2 * B.src_free + c];
      if (B.dst_free >= 0)
        for (int rr = 0; rr < 2; ++rr)
          for (int c = 0; c < 2; ++c) J.Jd[4 * b + 2 * rr + c] *= scale[2 * B.dst_free + c];
    }
    // |x - Plus(x, -gradient)|_inf
    std::vector<double> neg(n), proj;
    for (int i = 0; i < n; ++i) neg[i] = -J.grad[i];
    plus(x, neg, o.bound, &proj);
    gradient_max_norm = 0.0;
    for (int i = 0; i < n; ++i)
      gradient_max_norm = std::max(gradient_max_norm, std::fabs(x[i] - proj[i]));
  };

  evaluate_gradient_and_jacobian(true);
  R.initial_cost = x_cost;
  double minimum_cost = kMax;
  best = x;
  bool step_is_successful = true;  // iteration 0
  int iteration = 0;
  double radius = o.initial_trust_region_radius, decrease_factor = 2.0;
  bool reuse_diagonal = false;
  std::vector<double> diagonal(n), lm_diag(n);
  int num_consecutive_invalid = 0;
  // TrustRegionStepEvaluator with max_consecutive_nonmonotonic_steps = 0.
  double reference_cost = x_cost, current_cost = x_cost, candidate_ref_cost = x_cost,
         se_minimum_cost = x_cost;
  double acc_reference_mcc = 0.0, acc_candidate_mcc = 0.0;
  int num_nonmonotonic = 0;

  std::vector<double> step(n), delta(n), candidate_x(n), model_res(2 * nb), lhs, rhs(n), y;
  EvalOut cand;

  for (;;) {
    // FinalizeIterationAndCheckIfMinimizerCanContinue
    if (step_is_successful && x_cost < minimum_cost) {
      minimum_cost = x_cost;
      best = x;
    }
    if (iteration >= o.max_num_iterations) {
      R.termination = LFR_TERM_NO_CONVERGENCE;
      break;
    }
    if (step_is_successful && gradient_max_norm <= o.gradient_tolerance) {
      R.termination = LFR_TERM_GRADIENT_TOL;
      break;
    }
    if (radius <= o.min_trust_region_radius) {
      R.termination = LFR_TERM_MIN_RADIUS;
      break;
    }
    ++iteration;
    step_is_successful = false;

    // ComputeTrustRegionStep -> LevenbergMarquardtStrategy::ComputeStep
    if (!reuse_diagonal) {
      std::fill(diagonal.begin(), diagonal.end(), 0.0);
      for (size_t b = 0; b < nb; ++b) {
        const Block& B = C.blocks[b];
        if (B.src_free >= 0)
          for (int c = 0; c < 2; ++c)
            diagonal[2 * B.src_free + c] += J.Js[4 * b + c] * J.Js[4 * b + c] +
                                            J.Js[4 * b + 2 + c] * J.Js[4 * b + 2 + c];
        if (B.dst_free >= 0)
          for (int c = 0; c < 2; ++c)
            diagonal[2 * B.dst_free + c] += J.Jd[4 * b + c] * J.Jd[4 * b + c] +
                                            J.Jd[4 * b + 2 + c] * J.Jd[4 * b + 2 + c];
      }
      for (int i = 0; i < n; ++i)
        diagonal[i] = std::min(std::max(diagonal[i], o.min_lm_diagonal), o.max_lm_diagonal);
    }
    for (int i = 0; i < n; ++i) lm_diag[i] = std::sqrt(diagonal[i] / radius);
    // Normal equations (J'J + D'D) y = J'r  (SparseNormalCholeskySolver).
    lhs.assign((size_t)n * n, 0.0);
    std::fill(rhs.begin(), rhs.end(), 0.0);
    for (size_t b = 0; b < nb; ++b) {
      const Block& B = C.blocks[b];
      const double* js = &J.Js[4 * b];
      const double* jd = &J.Jd[4 * b];
      const double* r = &J.r[2 * b];
      const int s = B.src_free, d = B.dst_free;
      if (s >= 0) {
        for (int a = 0; a < 2; ++a) {
          rhs[2 * s + a] += js[a] * r[0] + js[2 + a] * r[1];
          for (int c = 0; c < 2; ++c)
            lhs[(size_t)(2 * s + a) * n + 2 * s + c] += js[a] * js[c] + js[2 + a] * js[2 + c];
        }
      }
      if (d >= 0) {
        for (int a = 0; a < 2; ++a) {
          rhs[2 * d + a] += jd[a] * r[0] + jd[2 + a] * r[1];
          for (int c = 0; c < 2; ++c)
            lhs[(size_t)(2 * d + a) * n + 2 * d + c] += jd[a] * jd[c] + jd[2 + a] * jd[2 + c];
        }
      }
      if (s >= 0 && d >= 0) {
        for (int a = 0; a < 2; ++a)
          for (int c = 0; c < 2; ++c) {
            const double v = js[a] * jd[c] + js[2 + a] * jd[2 + c];
            lhs[(size_t)(2 * s + a) * n + 2 * d + c] += v;
            lhs[(size_t)(2 * d + c) * n + 2 * s + a] += v;
          }
      }
    }
    for (int i = 0; i < n; ++i) lhs[(size_t)i * n + i] += lm_diag[i] * lm_diag[i];
    bool solved = cholesky_solve(lhs, n, rhs, &y);
    reuse_diagonal = true;
    bool step_is_valid = false;
    double model_cost_change = 0.0;
    if (solved) {
      for (int i = 0; i < n; ++i) step[i] = -y[i];
      // model_cost_change = -(J step)'(r + J step / 2)
      for (size_t b = 0; b < nb; ++b) {
        const Block& B = C.blocks[b];
        double m0 = 0.0, m1 = 0.0;
        if (B.src_free >= 0) {
          const double* js = &J.Js[4 * b];
          m0 += js[0] * step[2 * B.src_free] + js[1] * step[2 * B.src_free + 1];
          m1 += js[2] * step[2 * B.src_free] + js[3] * step[2 * B.src_free + 1];
        }
        if (B.dst_free >= 0) {
          const double* jd = &J.Jd[4 * b];
          m0 += jd[0] * step[2 * B.dst_free] + jd[1] * step[2 * B.dst_free + 1];
          m1 += jd[2] * step[2 * B.dst_free] + jd[3] * step[2 * B.dst_free + 1];
        }
        model_res[2 * b] = m0;
        model_res[2 * b + 1] = m1;
      }
      double dot = 0.0;
      for (size_t i = 0; i < 2 * nb; ++i) dot += model_res[i] * (J.r[i] + model_res[i] / 2.0);
      model_cost_change = -dot;
      step_is_valid = model_cost_change > 0.0;
    }
    if (!step_is_valid) {  // HandleInvalidStep
      ++num_consecutive_invalid;
      if (num_consecutive_invalid >= o.max_num_consecutive_invalid_steps) {
        R.termination = LFR_TERM_FAILURE;
        break;
      }
      radius = radius / decrease_factor;  // StepIsInvalid -> StepRejected(0)
      decrease_factor *= 2.0;
      reuse_diagonal = true;
      continue;
    }
    num_consecutive_invalid = 0;
    for (int i = 0; i < n; ++i) delta[i] = step[i] * scale[i];

    // is_constrained => projected Armijo line search along delta.
    do_line_search(C, o, x, J.grad, x_cost, &delta, &R.line_search_steps);

    // ComputeCandidatePointAndEvaluateCost
    plus(x, delta, o.bound, &candidate_x);
    evaluate(C, o, candidate_x, false, false, false, &cand);
    double candidate_cost = std::isfinite(cand.cost) ? cand.cost : kMax;

    // ParameterToleranceReached
    double step_norm = 0.0;
    for (int i = 0; i < n; ++i) step_norm += (x[i] - candidate_x[i]) * (x[i] - candidate_x[i]);
    step_norm = std::sqrt(step_norm);
    if (step_norm <= o.parameter_tolerance * (x_norm + o.parameter_tolerance)) {
      R.termination = LFR_TERM_PARAMETER_TOL;
      break;
    }
    // FunctionToleranceReached
    const double cost_change = x_cost - candidate_cost;
    if (std::fabs(cost_change) <= o.function_tolerance * x_cost) {
      R.termination = LFR_TERM_FUNCTION_TOL;
      break;
    }
    // IsStepSuccessful (TrustRegionStepEvaluator::StepQuality)
    const double relative_decrease = (current_cost - candidate_cost) / model_cost_change;
    const double historical =
        (reference_cost - candidate_cost) / (acc_reference_mcc + model_cost_change);
    const double quality = std::max(relative_decrease, historical);
    if (quality > o.min_relative_decrease) {  // HandleSuccessfulStep
      x = candidate_x;
      x_norm = norm2(x);
      evaluate_gradient_and_jacobian(false);
      step_is_successful = true;
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * quality - 1.0, 3));
      radius = std::min(o.max_trust_region_radius, radius);
      decrease_factor = 2.0;
      reuse_diagonal = false;
      // TrustRegionStepEvaluator::StepAccepted
      current_cost = candidate_cost;
      acc_candidate_mcc += model_cost_change;
      acc_reference_mcc += model_cost_change;
      if (current_cost < se_minimum_cost) {
        se_minimum_cost = current_cost;
        num_nonmonotonic = 0;
        candidate_ref_cost = current_cost;
        acc_candidate_mcc = 0.0;
      } else {
        ++num_nonmonotonic;
        if (current_cost > candidate_ref_cost) {
          candidate_ref_cost = current_cost;
          acc_candidate_mcc = 0.0;
        }
      }
      if (num_nonmonotonic == 0) {  // == max_consecutive_nonmonotonic_steps (monotonic)
        reference_cost = candidate_ref_cost;
        acc_reference_mcc = acc_candidate_mcc;
      }
    } else {  // HandleUnsuccessfulStep
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = true;
    }
  }
  R.iterations = iteration;
  R.final_cost = minimum_cost;
  // solver.cc (Minimize): the user state is only overwritten when Summary::IsSolutionUsable(),
  // i.e. not after FAILURE (10 consecutive invalid steps) — then the ORIGINAL values stay.
  if (R.termination != LFR_TERM_FAILURE) {
    for (int f = 0; f < C.n_free; ++f) {  // parameters <- best x
      C.pos[2 * C.local_of_free[f]] = best[2 * f];
      C.pos[2 * C.local_of_free[f] + 1] = best[2 * f + 1];
    }
  }
  return R;
}

// solve.cc:98-143 — which residual blocks exist and which blocks are constant.
void build_component(const lfr_problem& p, uint32_t c, const std::vector<uint32_t>& local_of,
                     const double* positions, Component* C) {
  const uint32_t beg = p.comp_ptr[c], end = p.comp_ptr[c + 1];
  const int nl = (int)(end - beg);
  C->nodes.assign(p.comp_nodes + beg, p.comp_nodes + end);
  C->pos.resize(2 * nl);
  for (int l = 0; l < nl; ++l) {
    C->pos[2 * l] = positions[2 * (size_t)C->nodes[l]];
    C->pos[2 * l + 1] = positions[2 * (size_t)C->nodes[l] + 1];
  }
  C->free_of.assign(nl, -1);
  C->local_of_free.clear();
  C->blocks.clear();
  C->n_free = 0;
  auto touch = [&](int l) {  // parameter blocks in order of first appearance
    if (p.is_root[C->nodes[l]]) return -1;  // SetParameterBlockConstant, solve.cc:134-135
    if (C->free_of[l] < 0) {
      C->free_of[l] = C->n_free++;
      C->local_of_free.push_back(l);
    }
    return C->free_of[l];
  };
  for (int l = 0; l < nl; ++l) {
    const uint32_t v = C->nodes[l];
    for (uint32_t e = p.row_ptr[v]; e < p.row_ptr[v + 1]; ++e) {
      const lfr_edge& E = p.edges[e];
      int kind;
      if (p.track[v] == p.track[E.dst]) kind = LFR_EDGE_CAUCHY;       // solve.cc:105
      else if (p.comp[v] == p.comp[E.dst]) kind = LFR_EDGE_TUKEY;     // solve.cc:114
      else continue;                                                  // solve.cc:123
      const int dl = (int)local_of[E.dst];
      Block B;
      B.src_local = l;
      B.dst_local = dl;
      B.src_free = touch(l);
      B.dst_free = touch(dl);
      if (B.src_free < 0 && B.dst_free < 0) continue;  // all-constant block: removed by Ceres' preprocessor (A.1)
      B.kind = kind;
      B.sim = (double)E.sim;
      for (int t = 0; t < 18; ++t) B.D[t] = (double)E.flow[t];
      C->blocks.push_back(B);
    }
  }
}

int validate(const lfr_problem* p) {
  if (!p) return fail(LFR_EINVAL, "problem is NULL");
  if (p->n_nodes && (!p->row_ptr || !p->track || !p->comp || !p->is_root))
    return fail(LFR_EINVAL, "NULL per-node array");
  if (p->n_components && (!p->comp_ptr || !p->comp_nodes))
    return fail(LFR_EINVAL, "NULL component list");
  if (p->n_nodes && p->row_ptr[p->n_nodes] != p->n_edges)
    return fail(LFR_EINVAL, "row_ptr[n_nodes] != n_edges");
  if (p->n_edges && !p->edges) return fail(LFR_EINVAL, "edges is NULL");
  for (uint64_t e = 0; e < p->n_edges; ++e)
    if (p->edges[e].dst >= p->n_nodes) return fail(LFR_EINVAL, "edge dst out of range");
  for (uint32_t c = 0; c < p->n_components; ++c)
    if (p->comp_ptr[c + 1] < p->comp_ptr[c]) return fail(LFR_EINVAL, "comp_ptr not monotone");
  const uint32_t tot = p->n_components ? p->comp_ptr[p->n_components] : 0;
  for (uint32_t i = 0; i < tot; ++i)
    if (p->comp_nodes[i] >= p->n_nodes) return fail(LFR_EINVAL, "comp_nodes out of range");
  return LFR_OK;
}

}  // namespace

extern "C" {

int lfr_abi_version(void) { return LFR_ABI_VERSION; }
const char* lfr_backend(void) { return "cpu-oracle"; }
const char* lfr_last_error(void) { return g_last_error.c_str(); }

void lfr_options_default(lfr_options* o) {
  if (!o) return;
  std::memset(o, 0, sizeof *o);
  o->bound = 1.0;
  o->cauchy_a = 0.25;
  o->tukey_a = 0.0625;
  o->tukey_variant = 1;
  o->max_num_iterations = 100;
  o->max_num_consecutive_invalid_steps = 10;
  o->max_num_line_search_step_size_iterations = 20;
  o->function_tolerance = 1e-4;
  o->gradient_tolerance = 1e-8;
  o->parameter_tolerance = 1e-4;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
  o->line_search_sufficient_function_decrease = 1e-4;
  o->max_line_search_step_contraction = 1e-3;
  o->min_line_search_step_contraction = 0.6;
  o->min_line_search_step_size = 1e-9;
  o->n_threads = 8;
  o->device = 0;
  o->linear_solver = 0;
}

int lfr_solve(const lfr_problem* p, const lfr_options* opt, double* positions,
              lfr_stats* stats) {
  int rc = validate(p);
  if (rc) return rc;
  if (!positions && p->n_nodes) return fail(LFR_EINVAL, "positions is NULL");
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  std::vector<uint32_t> local_of(p->n_nodes, 0);
  for (uint32_t c = 0; c < p->n_components; ++c)
    for (uint32_t i = p->comp_ptr[c]; i < p->comp_ptr[c + 1]; ++i)
      local_of[p->comp_nodes[i]] = i - p->comp_ptr[c];

  std::atomic<uint32_t> next(0);
  std::atomic<uint64_t> tot_it(0), tot_ls(0);
  std::atomic<uint32_t> n_solved(0);
  const auto t0 = std::chrono::steady_clock::now();
  // colmap::ThreadPool over the size-descending dispatch list, one task per
  // component, each task single-threaded (solve.cc:617-635).
  auto worker = [&]() {
    Component C;
    for (;;) {
      const uint32_t c = next.fetch_add(1);
      if (c >= p->n_components) break;
      const uint32_t nl = p->comp_ptr[c + 1] - p->comp_ptr[c];
      SolveResult R;
      if (nl <= 1) {  // solve.cc:619-622
        R.termination = LFR_TERM_SKIPPED;
      } else {
        build_component(*p, c, local_of, positions, &C);
        R = minimize(C, o);
        for (uint32_t l = 0; l < nl; ++l) {
          if (C.free_of[l] < 0) continue;
          positions[2 * (size_t)C.nodes[l]] = C.pos[2 * l];
          positions[2 * (size_t)C.nodes[l] + 1] = C.pos[2 * l + 1];
        }
        tot_it += (uint64_t)R.iterations;
        tot_ls += (uint64_t)R.line_search_steps;
        ++n_solved;
      }
      if (stats) {
        if (stats->iterations) stats->iterations[c] = R.iterations;
        if (stats->termination) stats->termination[c] = R.termination;
        if (stats->initial_cost) stats->initial_cost[c] = R.initial_cost;
        if (stats->final_cost) stats->final_cost[c] = R.final_cost;
      }
    }
  };
  const int nt = std::max(1, o.n_threads);
  if (nt == 1) {
    worker();
  } else {
    std::vector<std::thread> pool;
    for (int t = 0; t < nt; ++t) pool.emplace_back(worker);
    for (auto& th : pool) th.join();
  }
  const auto t1 = std::chrono::steady_clock::now();
  if (stats) {
    stats->total_iterations = tot_it.load();
    stats->total_line_search_steps = tot_ls.load();
    stats->n_solved = n_solved.load();
    stats->n_kernel_launches = 0;
    stats->h2d_ms = stats->kernel_ms = stats->d2h_ms = 0.0;
    stats->total_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  }
  return LFR_OK;
}

int lfr_solve_multi(const lfr_problem* p, const lfr_options* opt, const int32_t*, int32_t, double* positions,
                    lfr_stats* stats, lfr_multi_info* info) {
  if (info) std::memset(info, 0, sizeof *info);
  return lfr_solve(p, opt, positions, stats);  // the CPU pool has no devices to partition over
}

void lfr_shutdown(void) {}

void* lfr_host_alloc(uint64_t bytes) { return std::aligned_alloc(64, ((size_t)bytes + 63) / 64 * 64 + 64); }
void lfr_host_free(void* p) { std::free(p); }

int lfr_plan_create(const lfr_problem*, const lfr_options*, const double*, lfr_plan**) {
  return fail(LFR_EUNSUPPORTED, "cpu-oracle has no device plans");
}
int lfr_plan_solve(lfr_plan*, void*) { return fail(LFR_EUNSUPPORTED, "cpu-oracle has no device plans"); }
int lfr_plan_download(lfr_plan*, void*, double*, lfr_stats*) {
  return fail(LFR_EUNSUPPORTED, "cpu-oracle has no device plans");
}
int lfr_plan_num_launches(const lfr_plan*) { return 0; }
int lfr_plan_traffic(lfr_plan*, void*, uint64_t*, uint64_t*) {
  return fail(LFR_EUNSUPPORTED, "cpu-oracle has no device plans");
}
void lfr_plan_destroy(lfr_plan*) {}

int lfr_debug_edge_eval(const lfr_edge* edges, const uint8_t* kind, uint64_t n,
                        const double* xs, const double* xd, const lfr_options* opt,
                        double* r, double* jac, double* rho) {
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  for (uint64_t e = 0; e < n; ++e) {
    double D[18], f[2], dr[2], dc[2];
    for (int t = 0; t < 18; ++t) D[t] = (double)edges[e].flow[t];
    interpolate(D, xs[2 * e], xs[2 * e + 1], f, dr, dc);
    const double r0 = xd[2 * e] - xs[2 * e] - f[0];
    const double r1 = xd[2 * e + 1] - xs[2 * e + 1] - f[1];
    r[2 * e] = r0;
    r[2 * e + 1] = r1;
    jac[4 * e] = (0.0 - 1.0) - dr[0];
    jac[4 * e + 1] = (0.0 - 0.0) - dc[0];
    jac[4 * e + 2] = (0.0 - 0.0) - dr[1];
    jac[4 * e + 3] = (0.0 - 1.0) - dc[1];
    loss_eval(kind[e], (double)edges[e].sim, r0 * r0 + r1 * r1, o, &rho[3 * e]);
  }
  return LFR_OK;
}

// ---- oracle-only hooks for the known-answer tests -------------------------
void lfr_ref_interpolate(const double* grid18, double row, double col, double* f,
                         double* dfdrow, double* dfdcol) {
  interpolate(grid18, row, col, f, dfdrow, dfdcol);
}

void lfr_ref_loss(int kind, double sim, double s, const lfr_options* opt, double* rho) {
  lfr_options o;
  if (opt) o = *opt; else lfr_options_default(&o);
  loss_eval(kind, sim, s, o, rho);
}

// samples: [n][5] = {x, value, gradient, value_valid, gradient_valid}; samples[0] is
// the line search's initial point (x = 0), n = 2 or 3, all entries valid.
void lfr_ref_minimize_interpolating_polynomial(const double* samples, int n, double x_min,
                                               double x_max, double* optimal_x,
                                               double* optimal_value) {
  if (g_ls_mode.load() == 0) {  // literal polynomial.cc
    ceres::shim::MinimizeInterpolatingPolynomial(samples, n, x_min, x_max, optimal_x, optimal_value);
    return;
  }
  const bool three = n >= 3;
  *optimal_x = hermite_minimizer(samples[1], samples[2], samples[5], samples[6], samples[7], three,
                                 three ? samples[10] : 0.0, three ? samples[11] : 0.0,
                                 three ? samples[12] : 0.0, x_min, x_max, optimal_value);
}

// line-search interpolation mode: 0 literal polynomial.cc (default), 1 the fast formulation the GPU mirrors
void lfr_ref_set_line_search_mode(int mode) { g_ls_mode.store(mode ? 1 : 0); }
int lfr_ref_get_line_search_mode(void) { return g_ls_mode.load(); }

// the FAST formulation, whatever the mode (same arguments as lfr_ref_minimize_interpolating_polynomial)
void lfr_ref_minimize_interpolating_polynomial_fast(const double* samples, int n, double x_min, double x_max,
                                                    double* optimal_x, double* optimal_value) {
  const bool three = n >= 3;
  *optimal_x = hermite_minimizer(samples[1], samples[2], samples[5], samples[6], samples[7], three,
                                 three ? samples[10] : 0.0, three ? samples[11] : 0.0,
                                 three ? samples[12] : 0.0, x_min, x_max, optimal_value);
}

// polynomial.cc FindPolynomialRoots, literal (balanced companion matrix eigenvalues): real and imaginary
// parts of all roots of coeffs[0..n) (highest degree first); returns the count or -1
int lfr_ref_find_polynomial_roots(const double* coeffs, int n, double* real, double* imag) {
  return ceres::shim::FindPolynomialRoots(coeffs, n, real, imag);
}

// harvest of line-search interpolation states (11 doubles each) from subsequent lfr_solve calls
void lfr_ref_harvest(int on) {
  std::lock_guard<std::mutex> lock(g_harvest_mutex);
  g_harvested.clear();
  g_harvest.store(on != 0);
}
uint64_t lfr_ref_harvest_take(double* out, uint64_t max_states) {
  std::lock_guard<std::mutex> lock(g_harvest_mutex);
  const uint64_t have = g_harvested.size() / 11;
  const uint64_t n = std::min(have, max_states);
  if (out && n) std::memcpy(out, g_harvested.data(), sizeof(double) * 11 * n);
  return have;
}

// real roots inside [lo, hi] of a polynomial given highest-degree-first (n <= 5 coefficients)
int lfr_ref_polynomial_roots(const double* coeffs, int n, double lo, double hi, double* real_out) {
  return real_roots_in(coeffs, n, lo, hi, real_out);
}

}  // extern "C"
