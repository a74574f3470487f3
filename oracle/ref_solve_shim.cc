// ref_solve_shim.cc — a C entry point into the REFERENCE's own create_and_solve_problem.
//
// TEST INFRASTRUCTURE ONLY.  This translation unit #includes
// /root/reference/multi-view-refinement/solve.cc verbatim (found through -I; never copied into this
// repository; it #includes cost.cc and graph.h) with its main() renamed, and compiles it against the
// shim headers in oracle/ref_shims/.  What runs below is the reference author's
// create_and_solve_problem (solve.cc:79-160): which residual blocks, which loss, which nodes are
// constant (SetParameterBlockConstant on every node whose is_root entry is set, solve.cc:131-143),
// the bounds and the solver options, minimised by mini-Ceres (oracle/ref_shims/mini_ceres.cc).
//
// The constant mask and the start point are arguments of that function, so any mask (the reference's
// roots OR the nodes of fixed images) and any start can be handed to it: an independent statement of
// what holding an image fixed means.  Built by oracle/build_ref.py into oracle/_ref/libref_solve.so;
// used by tests/test_fixed_images_ref.py and tests/test_gpu_fixed_tiers.py.
#define main lfr_refsrc_solve_main
#include "solve.cc"
#undef main

#include <stdint.h>

#include <cstring>
#include <unordered_map>

#include "lfr.h"

namespace {

// the LFR_TERM_* code of a summary (include/lfr.h), from the message mini-Ceres' minimizer sets at each
// of Ceres' termination points; -1 for a message not listed here
int termination_code(const ceres::Solver::Summary& s) {
  static const struct { const char* prefix; int code; } kCodes[] = {
      {"Function tolerance reached. No non-constant", LFR_TERM_EMPTY},
      {"Gradient tolerance", LFR_TERM_GRADIENT_TOL},
      {"Parameter tolerance", LFR_TERM_PARAMETER_TOL},
      {"Function tolerance", LFR_TERM_FUNCTION_TOL},
      {"Minimum trust region radius", LFR_TERM_MIN_RADIUS},
      {"Maximum number of iterations", LFR_TERM_NO_CONVERGENCE},
      {"Number of consecutive invalid steps", LFR_TERM_FAILURE},
      {"Residual and Jacobian evaluation failed", LFR_TERM_FAILURE},
  };
  for (const auto& k : kCodes)
    if (s.message.compare(0, std::strlen(k.prefix), k.prefix) == 0) return k.code;
  return -1;
}

}  // namespace

extern "C" {

// Every dispatch slot of `p` with more than one node through create_and_solve_problem(graph, track,
// positions, is_const, comp, nodes, 1) on a pool of `n_threads` workers, as main() dispatches them
// (solve.cc:614-635), with is_root = `is_const` [n_nodes] and positions = `start` [n_nodes][2].
// p->is_root is not read.  Out: `positions` [n_nodes][2]; per slot (0 / SKIPPED for slots of one node)
// the summary's num_iterations, LFR_TERM_* code, num_line_search_steps, initial_cost, final_cost and
// fixed_cost (the cost of the residual blocks between two constant nodes, part of initial_cost).
// Returns the number of solved slots, or -1 when a summary cannot be matched to its slot.
int lfr_refsrc_solve(const lfr_problem* p, const uint8_t* is_const, const double* start, uint32_t n_threads,
                     double* positions, int32_t* iterations, int32_t* termination, int32_t* ls_steps,
                     double* initial_cost, double* final_cost, double* fixed_cost) {
  const size_t N = p->n_nodes;
  // the reference's Graph (graph.h), out-edges in CSR order = insertion order; flows and similarities
  // widened from float to double as solve.cc:458-472 reads them
  Graph graph;
  for (size_t v = 0; v < N; ++v) {
    PatchNode* node = new PatchNode(std::string(), (int)v);
    graph.add_node(node);
  }
  for (size_t v = 0; v < N; ++v) {
    for (uint32_t k = p->row_ptr[v]; k < p->row_ptr[v + 1]; ++k) {
      const lfr_edge& e = p->edges[k];
      std::vector<double> flow(2 * kNumSamples * kNumSamples);
      for (size_t i = 0; i < flow.size(); ++i) flow[i] = e.flow[i];
      graph.nodes[v]->add_edge(graph.nodes[e.dst], (double)e.sim, flow);
    }
  }
  std::vector<size_t> track(p->track, p->track + N), comp(p->comp, p->comp + N);
  std::vector<bool> is_root(N);
  std::vector<Eigen::Vector2d> pos(N);
  std::unordered_map<const double*, size_t> node_of;
  for (size_t v = 0; v < N; ++v) {
    is_root[v] = is_const[v] != 0;
    pos[v][0] = start[2 * v];
    pos[v][1] = start[2 * v + 1];
    node_of[pos[v].data()] = v;
  }
  std::vector<std::vector<size_t>> nodes(p->n_components);
  std::vector<int64_t> slot_of(N, -1);
  for (uint32_t c = 0; c < p->n_components; ++c) {
    nodes[c].assign(p->comp_nodes + p->comp_ptr[c], p->comp_nodes + p->comp_ptr[c + 1]);
    for (size_t v : nodes[c]) slot_of[v] = c;
    iterations[c] = termination[c] = ls_steps[c] = 0;
    initial_cost[c] = final_cost[c] = fixed_cost[c] = 0.0;
  }
  ceres::shim::SetRecording(true);
  ceres::shim::TakeRecords();
  int n_solved = 0;
  {
    colmap::ThreadPool pool((int)n_threads);
    for (uint32_t c = 0; c < p->n_components; ++c) {
      if (nodes[c].size() <= 1) continue;
      ++n_solved;
      pool.AddTask(create_and_solve_problem, std::ref(graph), std::ref(track), std::ref(pos), std::ref(is_root),
                   std::ref(comp), std::ref(nodes[c]), 1);
    }
    pool.Wait();
  }
  const std::vector<ceres::shim::Record> recs = ceres::shim::TakeRecords();
  ceres::shim::SetRecording(false);
  for (size_t v = 0; v < N; ++v) {
    positions[2 * v] = pos[v][0];
    positions[2 * v + 1] = pos[v][1];
  }
  for (PatchNode* node : graph.nodes) {
    for (Edge* e : node->out_edges) delete e;
    delete node;
  }
  if ((int)recs.size() != n_solved) return -1;
  for (const ceres::shim::Record& r : recs) {
    const auto it = node_of.find(r.first_parameter_block);
    if (it == node_of.end() || slot_of[it->second] < 0) return -1;
    const int64_t c = slot_of[it->second];
    iterations[c] = r.summary.num_iterations;
    termination[c] = termination_code(r.summary);
    ls_steps[c] = r.summary.num_line_search_steps;
    initial_cost[c] = r.summary.initial_cost;
    final_cost[c] = r.summary.final_cost;
    fixed_cost[c] = r.summary.fixed_cost;
  }
  return n_solved;
}

}  // extern "C"
