/*
 * lfr_graph.h — the graph stage on the GPU: from the decoded match arrays straight to a
 * device-resident plan (include/lfr.h).
 *
 * lfr_plan_create_from_matches() uploads the flat match arrays of lfr_host_input once and builds,
 * on the device, everything lfr_host_stage_create() + lfr_host_stage_export() produce (solve.cc:438-606):
 * node interning, the CSR edge lists and their 80-byte records, the constrained Kruskal, track ids and
 * roots, the track meta-graph and its components, the dispatch list.  Every array is bitwise equal to
 * the host stage's.  Only the recursive 2-way cut of oversized meta-components runs on the host, on
 * the downloaded edges of those components (the same code as the host stage, lfr_cut.h).  The edge
 * records never leave the device: the plan solves them in place (lfr_plan_solve / lfr_plan_download).
 *
 * `in->edges_out` is ignored.  `sizes` (may be NULL) receives every count lfr_host_stage_create()
 * reports; tracks_ms / graph_cut_ms / graph_ms / dispatch_ms time the device phases (host clock,
 * stream synchronised at each phase boundary).  Errors: LFR_EINVAL for an image id out of range or a
 * non-finite similarity, LFR_EUNSUPPORTED for more than 65 535 images (as the host stage) or more than
 * 2^31 - 1 directed edges.  Only liblfr_b200.so provides these two symbols; the CPU oracle has no
 * plans and does not (the Python binding refuses Plan.from_matches() on it with LFR_EUNSUPPORTED).
 *
 * Cost: the Kruskal runs in rounds over a window of pending edges (LFR_KRUSKAL_WINDOW in the
 * environment, default 262144 edges; results do not depend on it), and every round ends with one
 * host-device synchronisation to refill the window.  Only one edge per union-find root decides per
 * round, so a long run of edges on one root — a feature matched across hundreds of images whose unions
 * are refused by image clashes — costs one round each.  The stage also allocates and frees its scratch
 * buffers (a few dozen cudaMalloc / cudaFree pairs) on every call.
 */
#ifndef LFR_GRAPH_H_
#define LFR_GRAPH_H_

#include <stdint.h>

#include "lfr.h"
#include "lfr_host.h"

#ifdef __cplusplus
extern "C" {
#endif

int lfr_plan_create_from_matches(const lfr_host_input* in, const lfr_options* o,
                                 const double* initial_positions /* [2N] or NULL = zeros */,
                                 lfr_plan** out, lfr_host_sizes* sizes);

/* Copy the stage's arrays of a plan made by lfr_plan_create_from_matches() into caller-owned arrays;
 * the arguments mean what they mean in lfr_host_stage_export() (any pointer may be NULL; `edges` is a
 * device-to-host copy).  LFR_EINVAL for a plan made by lfr_plan_create(). */
int lfr_plan_export_graph(const lfr_plan* plan, uint32_t* row_ptr /* [N+1] */, lfr_edge* edges /* [E] */,
                          uint32_t* track /* [N] */, uint32_t* comp /* [N] */, uint8_t* is_root /* [N] */,
                          uint32_t* comp_ptr /* [C+1] */, uint32_t* comp_nodes /* [N] */,
                          uint32_t* comp_order /* [C] */, uint32_t* node_image /* [N] */,
                          uint32_t* node_feat /* [N] */);

#ifdef __cplusplus
}
#endif
#endif /* LFR_GRAPH_H_ */
