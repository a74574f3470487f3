// lfr_lm.cuh — the minimizer every solve tier runs: Ceres' TrustRegionMinimizer (LEVENBERG_MARQUARDT,
// SURVEY A.6) with the projected Armijo line search of the bounds-constrained problem (A.7b), from
// iteration 0 to the per-slot statistics, written once over a tier's primitives.
//
// A tier (Warp2Tier, TileTier, WarpTier, CtaTier: one per solve kernel) wraps its context `C` and
// supplies, with every thread of its warp / CTA calling each member together:
//   kStride, kTier, kPolyWord  threads per component, the profile's tier code, the word that takes
//                              the line search's polynomial cycles
//   tid(), lane(), lead()      thread index (< kStride), lane in the warp, writer of the scalars
//   eval_x()                   cost at x (and the staged evaluation the assembly reads)
//   assemble(first)            gradient and normal matrix at the staged evaluation -> |x - P(x - g)|_inf
//                              (first: also fixes the Jacobi scaling)
//   lm_step(radius, &mc, &gd, &dmax)
//                              the damped step dl -> validity, model cost change, g . dl, |dl|_inf
//   trial(alpha)               xc = P(x + alpha dl) and the cost there
//   trial_slope(alpha, &dphi)  the same plus phi'(alpha) = grad f(xc) . dl (only read if the cost is finite)
//   slope()                    phi' at the candidate of the last trial()
//   scale_step(s)              dl *= s
//   x_norm()                   |x| over the free coordinates
//   step_norm()                |x - xc| over the free coordinates
//   accept()                   x = xc -> the new |x|
//   counter()                  the tier's own profile counter (word 7)
// The tiers differ in how they reduce, fuse and synchronise; those choices stay inside their
// members, so each tier's sums are the same operations, in the same order, as before the driver
// existed, and the driver changes no bit of any result.
#pragma once
#include "lfr_math.cuh"

namespace lfr {

struct DevProblem {
  uint32_t n_nodes;
  int* err_flag;  // set by classify_edge on malformed input: a dst out of range, a self edge, or a
                  // component node list that disagrees with `comp`
  const uint32_t* row_ptr;
  const float4* edges;  // 5 x float4 per edge
  const uint32_t* track;
  const uint32_t* comp;
  const uint8_t* is_root;
  const uint32_t* comp_ptr;
  const uint32_t* comp_nodes;
  const uint32_t* local_of;  // node -> index inside its component's node list
  double* positions;         // [2N] start point (device memory)
  double* positions_out;     // [2N] results: `positions` itself, or the caller's pinned host buffer
                             // (zero-copy write-back: only free nodes are written, solve.cc:131-141)
  unsigned long long* pull_ctr;  // [2] bytes of staging pulls {ticketed, arrived} (zero-copy pacing, see stage_edges)
  unsigned pull_window;      // 0 = unpaced; else at most this many bytes of staging pulls are outstanding per device
  // per dispatch slot
  int32_t* st_iter;
  int32_t* st_term;
  double* st_cost0;
  double* st_cost1;
  uint32_t* st_ls;
  uint32_t* st_kept;  // kept directed edges E_c
  unsigned long long* st_cycles;  // optional (LFR_DBG_PROFILE): one LmProfile record per slot
  unsigned long long* st_times;   // optional [2 per slot]: %globaltimer (ns) when the component's solve started / finished
};

// The LFR_DBG_PROFILE record of one dispatch slot (8 x u64 at P.st_cycles + 8 * slot; copied out by
// lfr_debug_plan_cycles, decoded by capi.profile_record).  Every word means the same on every tier:
//   0 total cycles of the component (kernel entry to the statistics)
//   1 setup: from kernel entry to the first evaluation
//   2 evaluation of the cost at x and at the full step
//   3 assembly after an accepted step (and at iteration 0)
//   4 linear solve (lm_step)
//   5 line search and the rest of the loop
//   6 line-search steps << 32 | SM id
//   7 tier << 56 | tier counter: line-search polynomial cycles (warp2, tile, warp), CG iterations (CTA,
//     whose polynomial cycles count in word 5)
// Words 1-5 (and 7's cycles) add up to word 0.  Setup is everything before the driver runs: the staging
// and classification of the warp2 / tile / warp tiers, the start-point projection of the CTA tier (whose
// lists come from cta_prepare_kernel).  Each mark adds its interval to the record with two global
// atomics from the writing thread; that is part of what a profiled run measures, so its shares are not
// comparable with records taken before the driver existed (per-tier register counters).  A solve
// without LFR_DBG_PROFILE only tests P.st_cycles at each mark.
struct LmProfile {
  enum Word { kTotal = 0, kSetup, kEval, kAssemble, kSolve, kRest, kSteps, kTierWord };
  enum Tier : unsigned { kWarp2 = 1, kTile = 2, kWarp = 3, kCta = 4 };

  const DevProblem& P;  // the record of slot c is written when P.st_cycles is set (a kernel parameter: the
  uint32_t c;           // test costs no register), by the thread that writes the scalars
  bool lead;
  long long t_mark;

  // At kernel entry, before the tier's setup.
  __device__ __forceinline__ LmProfile(const DevProblem& P_, uint32_t c_, bool lead_)
      : P(P_), c(c_), lead(lead_), t_mark(0) {
    if (!P.st_cycles) return;
    if (lead) {
      for (int k = 0; k < 8; ++k) P.st_cycles[8 * (size_t)c + k] = 0;
      P.st_times[2 * (size_t)c] = globaltimer();
    }
    t_mark = clock64();
  }
  // Charges the cycles since the last mark to word `w` (and to the total).
  __device__ __forceinline__ void tick(int w) {
    if (!P.st_cycles) return;
    const long long now = clock64();
    if (lead) {
      unsigned long long* o = P.st_cycles + 8 * (size_t)c;
      const unsigned long long d = (unsigned long long)(now - t_mark);
      atomicAdd(o + w, d);  // result unused: a fire-and-forget reduction, nothing waits on it
      atomicAdd(o + kTotal, d);
    }
    t_mark = now;
  }
  __device__ __forceinline__ void finish(unsigned ls_steps, unsigned tier, unsigned long long counter) {
    if (!P.st_cycles) return;
    tick(kRest);
    if (!lead) return;
    unsigned long long* o = P.st_cycles + 8 * (size_t)c;
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    o[kSteps] = (unsigned long long)ls_steps << 32 | smid;
    atomicAdd(o + kTierWord, (unsigned long long)tier << 56 | counter);
    P.st_times[2 * (size_t)c + 1] = globaltimer();
  }
  __device__ __forceinline__ static unsigned long long globaltimer() {
    unsigned long long ns;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
    return ns;
  }
};

// A component without free nodes ("No non-constant parameter blocks found."): its statistics.
__device__ __forceinline__ void lm_empty(const DevProblem& P, uint32_t c) {
  P.st_iter[c] = 0;
  P.st_term[c] = LFR_TERM_EMPTY;
  P.st_cost0[c] = 0.0;
  P.st_cost1[c] = 0.0;
  P.st_ls[c] = 0;
}

// Solves component `c` once its tier's setup is done: iteration 0, the trust-region loop with the
// line search, write-back of the free nodes' positions (not after FAILURE), the statistics and the
// profile record.
template <class Tier>
__device__ __forceinline__ void lm_solve(Tier& T, const DevProblem& P, const DevConsts& K, uint32_t c,
                                         LmProfile& prof) {
  const auto& C = T.C;
  if (T.lead()) P.st_kept[c] = (uint32_t)C.Ec;
  if (C.nf == 0) {
    if (T.lead()) lm_empty(P, c);
    return;
  }
  prof.tick(LmProfile::kSetup);

  // ---- iteration 0 -----------------------------------------------------------------
  double cost = T.eval_x();
  prof.tick(LmProfile::kEval);
  double gmax = T.assemble(true);
  prof.tick(LmProfile::kAssemble);
  const double cost0 = cost;
  double radius = K.radius0, nu = 2.0;
  int iter = 0, n_invalid = 0, term = LFR_TERM_NO_CONVERGENCE;
  unsigned ls_steps = 0;
  bool success = true;
  double x_norm = T.x_norm();

  // ---- trust-region loop (A.6) ---------------------------------------------------------
  for (;;) {
    if (iter >= K.max_iter) { term = LFR_TERM_NO_CONVERGENCE; break; }
    if (success && gmax <= K.g_tol) { term = LFR_TERM_GRADIENT_TOL; break; }
    if (radius <= K.radius_min) { term = LFR_TERM_MIN_RADIUS; break; }
    ++iter;
    success = false;
    double model_change = 0.0, gd = 0.0, dmax = 0.0;
    prof.tick(LmProfile::kRest);
    bool valid = T.lm_step(radius, &model_change, &gd, &dmax);
    prof.tick(LmProfile::kSolve);
    valid = valid && (model_change > 0.0);
    if (!valid) {
      if (++n_invalid >= K.max_invalid) { term = LFR_TERM_FAILURE; break; }
      radius /= nu;
      nu *= 2.0;
      continue;
    }
    n_invalid = 0;
    // projected Armijo line search along dl (bounds-constrained problem, A.7b)
    double cost_c = T.trial(1.0);
    prof.tick(LmProfile::kEval);
    bool c_valid = isfinite(cost_c);
    if (!c_valid || cost_c > cost + K.ls_suff * gd * 1.0) {
      LsSample initial{0.0, cost, gd, true, true};
      LsSample previous{0.0, 0.0, 0.0, false, false};
      LsSample current{1.0, cost_c, 0.0, c_valid, false};
      if (c_valid) {
        current.gradient = T.slope();
        current.gradient_valid = isfinite(current.gradient);
      }
      int ls_iter = 0;
      bool ls_ok = false;
      for (;;) {
        ++ls_iter;
        ++ls_steps;
        if (ls_iter >= K.max_ls_iter) break;
        prof.tick(LmProfile::kRest);
        const double step = ls_next_step(initial, previous, current, K, T.lane());
        prof.tick(Tier::kPolyWord);
        if (step * dmax < K.ls_min_step) break;
        previous = current;
        double dphi;
        cost_c = T.trial_slope(step, &dphi);
        c_valid = isfinite(cost_c);
        current = LsSample{step, cost_c, 0.0, c_valid, false};
        if (c_valid) {
          current.gradient = dphi;
          current.gradient_valid = isfinite(dphi);
        }
        if (c_valid && !(cost_c > cost + K.ls_suff * gd * step)) { ls_ok = true; break; }
      }
      if (ls_ok) {
        T.scale_step(current.x);
      } else {  // line search failed: delta unchanged, candidate = P(x + delta)
        cost_c = T.trial(1.0);
        c_valid = isfinite(cost_c);
      }
    }
    if (!c_valid) cost_c = 1.7976931348623157e308;
    const double step_norm = T.step_norm();
    if (step_norm <= K.p_tol * (x_norm + K.p_tol)) { term = LFR_TERM_PARAMETER_TOL; break; }
    if (fabs(cost - cost_c) <= K.f_tol * cost) { term = LFR_TERM_FUNCTION_TOL; break; }
    const double rho = (cost - cost_c) / model_change;
    if (rho > K.min_rel_decrease) {
      x_norm = T.accept();
      cost = cost_c;
      prof.tick(LmProfile::kRest);
      gmax = T.assemble(false);
      prof.tick(LmProfile::kAssemble);
      success = true;
      const double t = 2.0 * rho - 1.0;
      radius = fmin(K.radius_max, radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
      nu = 2.0;
    } else {
      radius /= nu;
      nu *= 2.0;
    }
  }
  // ---- write back the last accepted x ---------------------------------------------------
  // (not after FAILURE: Ceres only commits a usable solution, solver.cc Minimize / IsSolutionUsable)
  if (term != LFR_TERM_FAILURE) {
    for (int i = T.tid(); i < C.n; i += Tier::kStride) {
      const int l = C.lof[i >> 1];
      P.positions_out[2 * (size_t)C.node[l] + (i & 1)] = C.x[2 * l + (i & 1)];
    }
  }
  if (T.lead()) {
    P.st_iter[c] = iter;
    P.st_term[c] = term;
    P.st_cost0[c] = cost0;
    P.st_cost1[c] = cost;
    P.st_ls[c] = ls_steps;
  }
  prof.finish(ls_steps, Tier::kTier, T.counter());
}

}  // namespace lfr
