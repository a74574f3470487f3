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
 * 2^31 - 1 directed edges.  Only liblfr_b200.so provides this header's symbols; the CPU oracle has no
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

/* One MatchingFile part for lfr_plan_create_from_wire(): its bytes and the offset of each of its
 * matches' length prefix, as lfr_wire_walk_matches() (include/lfr_wire.h) records them. */
typedef struct lfr_wire_part {
  const uint8_t* buf;         /* [len] the part's bytes; may be pageable (e.g. a mapped file) */
  uint64_t len;
  const uint64_t* match_off;  /* [n_matches] */
  uint64_t n_matches;
} lfr_wire_part;

/* lfr_plan_create_from_matches() from the MatchingFile bytes: the matches are decoded on the device,
 * straight into the stage's input, and never exist on the host.  `in` carries the pair level only —
 * n_pairs, n_matches, n_images, pair_img1/2, pair_skip, pair_ptr, built by the caller from
 * lfr_wire_walk_matches() over the parts in order (pair_ptr global: part k's matches follow part k-1's);
 * in->feat1 ... in->disp2 and edges_out are ignored.  The parts' n_matches must add up to in->n_matches.
 * The bytes go up through page-locked staging.  Every match is decoded with the semantics of
 * lfr_wire_decode_matches(), those of banned pairs included, so the result — the plan, every
 * lfr_plan_export_graph() array and the solve — is bitwise that of lfr_plan_create_from_matches() on
 * the host decode of the same bytes.  Errors: LFR_EINVAL with lfr_last_error() = "malformed Match
 * message" when a match is malformed (exactly when lfr_wire_decode_matches() rejects its part), checked
 * before the stage runs; otherwise the codes of lfr_plan_create_from_matches(). */
int lfr_plan_create_from_wire(const lfr_host_input* in, const lfr_wire_part* parts, uint32_t n_parts,
                              const lfr_options* o, const double* initial_positions /* [2N] or NULL */,
                              lfr_plan** out, lfr_host_sizes* sizes);

/* Copy the stage's arrays of a plan made by lfr_plan_create_from_matches() or _from_wire() into caller-owned arrays;
 * the arguments mean what they mean in lfr_host_stage_export() (any pointer may be NULL; `edges` is a
 * device-to-host copy).  LFR_EINVAL for a plan made by lfr_plan_create(). */
int lfr_plan_export_graph(const lfr_plan* plan, uint32_t* row_ptr /* [N+1] */, lfr_edge* edges /* [E] */,
                          uint32_t* track /* [N] */, uint32_t* comp /* [N] */, uint8_t* is_root /* [N] */,
                          uint32_t* comp_ptr /* [C+1] */, uint32_t* comp_nodes /* [N] */,
                          uint32_t* comp_order /* [C] */, uint32_t* node_image /* [N] */,
                          uint32_t* node_feat /* [N] */);

/* Whether a solve of `in` on `n_devices` devices should run its graph stage on the device
 * (lfr_plan_create_from_matches) rather than on the host (lfr_host_stage_create): 1 or 0.  Decided from
 * sizes known before either stage runs — the directed edges (2 x the matches of the pairs not skipped),
 * the number of images and of devices — and from nothing else: it needs no device and makes no CUDA
 * call.  0 below a size threshold measured on an H100 (DESIGN.md §4), for more than one device
 * (lfr_solve_multi() takes a host lfr_problem; plans are single-device), for NULL or malformed input and
 * for inputs the device stage refuses. */
int lfr_graph_stage_on_device(const lfr_host_input* in, int32_t n_devices);

/* On the device route, whether the matches should be decoded on the device (lfr_plan_create_from_wire)
 * rather than on the host (lfr_wire_decode_matches + lfr_plan_create_from_matches): 1 or 0, from the
 * match count alone (all pairs, banned ones included: every match is decoded).  0 below a threshold
 * measured on an H100 (DESIGN.md §4).  Host code only, like lfr_graph_stage_on_device(). */
int lfr_wire_decode_on_device(uint64_t n_matches);

#ifdef __cplusplus
}
#endif
#endif /* LFR_GRAPH_H_ */
