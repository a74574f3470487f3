/*
 * lfr_host.h — C ABI of the native host graph stage (SURVEY 8f, "next" row 2).
 *
 * Everything solve.cc does between the parsed MatchingFile and the solves
 * (solve.cc:438-606): node interning and directed edge lists (:53-65, :474-478),
 * constrained Kruskal -> tracks (:489-549), root selection (:552-582), the track
 * meta-graph, its connected components and the size-capped recursive 2-way cut
 * (:252-373, :185-250) and the dispatch list (:594-604) — from the flat match
 * arrays lfr_wire_decode_matches() produces straight into the arrays of
 * lfr_problem (include/lfr.h).  Host code only; no GPU needed.
 *
 * The 2-way cut stands in for colmap::ComputeNormalizedMinGraphCut (solve.cc:192),
 * which is not part of the reference repository; it is the same deterministic
 * algorithm as local-feature-refinement_b200/graph.py::two_way_cut, and the two
 * implementations are tested to agree exactly.
 */
#ifndef LFR_HOST_H_
#define LFR_HOST_H_

#include <stdint.h>

#include "lfr.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lfr_host_stage lfr_host_stage;

typedef struct lfr_host_input {
  uint64_t n_pairs, n_matches;
  uint32_t n_images;            /* image ids are < n_images                      */
  const uint32_t* pair_img1;    /* [n_pairs] image id of side 1 (types.proto:5)   */
  const uint32_t* pair_img2;    /* [n_pairs]                                      */
  const uint8_t* pair_skip;     /* [n_pairs] 1 = pair touches a banned image (solve.cc:444-446), may be NULL */
  const uint64_t* pair_ptr;     /* [n_pairs+1]                                    */
  const uint32_t* feat1;        /* [n_matches]                                    */
  const uint32_t* feat2;
  const float* sim;
  const float* disp1;           /* [n_matches*18]                                 */
  const float* disp2;
  /* optional: caller-owned destination of the 80-byte edge records (the bulk of the output; their
   * number is known up front: 2 x the matches of the non-skipped pairs).  When given and large
   * enough the stage writes them there directly and lfr_host_stage_export() skips its copy. */
  lfr_edge* edges_out;
  uint64_t edges_out_capacity;  /* in records                                     */
  /* optional: [n_images] the sub-scene of every image id, or NULL: the whole input is one scene.  With
   * sub-scenes (--query_images, one query or with --joint_queries a group of queries each) every
   * non-skipped pair joins two images of one sub-scene (LFR_EINVAL otherwise), the cut cap of a
   * meta-component is the number of images its sub-scene's non-skipped pairs name (n_images_seen of that
   * sub-scene alone), and a union-find image set indexes images inside their sub-scene, so its storage
   * follows the largest sub-scene, not n_images.  Each sub-scene then gets the arrays a stage on its pairs
   * alone gives, under a renumbering that keeps their relative order.  The graph stage on the GPU
   * (lfr_plan_create_from_matches(), lfr_plan_create_from_wire()) takes sub-scenes as this stage does. */
  const uint32_t* image_group;
} lfr_host_input;

typedef struct lfr_host_sizes {
  uint32_t n_nodes, n_tracks, n_components, n_images_seen, max_track_size, max_component_size;
  uint32_t n_meta_components, n_oversized_meta_components, n_cut_groups, reserved;
  uint64_t n_edges;
  double tracks_ms, graph_cut_ms;   /* solve.cc:487-582 (sort, Kruskal, roots) and :585-589 ("Graph-cut time") */
  double graph_ms, dispatch_ms;     /* node interning + edge lists (:438-481); dispatch list (:594-604)     */
} lfr_host_sizes;

/* Run the whole stage.  Returns 0 or LFR_E*. */
int lfr_host_stage_create(const lfr_host_input* in, lfr_host_stage** out, lfr_host_sizes* sizes);

/* Copy the results into caller-owned arrays (any pointer may be NULL). */
int lfr_host_stage_export(const lfr_host_stage* hs,
                          uint32_t* row_ptr /* [N+1] */, lfr_edge* edges /* [E] */,
                          uint32_t* track /* [N] */, uint32_t* comp /* [N] */, uint8_t* is_root /* [N] */,
                          uint32_t* comp_ptr /* [C+1] */, uint32_t* comp_nodes /* [N] */,
                          uint32_t* comp_order /* [C] component id of each dispatch slot */,
                          uint32_t* node_image /* [N] */, uint32_t* node_feat /* [N] */);

void lfr_host_stage_destroy(lfr_host_stage* hs);

/* The host form of lfr_plan_update_solution_since() (include/lfr_graph.h, which states the rule), bit for
 * bit: `p` is this run's problem (the reference's is_root, not a constant mask) with node ids
 * node_image / node_feat, image names by id names / name_off (n_images); `previous` is the earlier
 * MatchingFile's lfr_host_input (its pair_skip and edges_out are ignored: the earlier run bans no image) with
 * its names prev_names / prev_name_off (previous->n_images).  Runs lfr_host_stage_create() on `previous`,
 * marks the components that are not unchanged, then joins the SolutionFile `buf` as
 * lfr_wire_update_solution() does with those components touched too: positions [2 n_nodes], held [n_nodes],
 * *n_held and *n_touched mean what they mean there; *n_changed (may be NULL) = the components that are not
 * unchanged.  LFR_EINVAL for malformed bytes, NULL or inconsistent arrays, or malformed or repeated earlier
 * names; the earlier stage's codes (lfr_host_stage_create) when it rejects `previous`.  Every output is
 * untouched on error. */
int lfr_wire_update_solution_since(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names,
                                   const uint64_t* name_off, const lfr_problem* p, const uint32_t* node_image,
                                   const uint32_t* node_feat, const lfr_host_input* previous, const uint8_t* prev_names,
                                   const uint64_t* prev_name_off, double* positions /* [2 n_nodes] */,
                                   uint8_t* held /* [n_nodes] */, uint64_t* n_held, uint32_t* n_touched,
                                   uint32_t* n_changed);

/* The host form of lfr_plan_problem_record() (include/lfr_graph.h states the record), byte for byte: the
 * record of problem `p` with node ids node_image / node_feat and image names by id names / name_off
 * (n_images).  `p->is_root` must be the reference's is_root (the graph stage's export), not a constant mask;
 * comp_ptr / comp_nodes are not read.  Returns the record's size, 16 + 16 p->n_components, and writes it to
 * `out` only when `cap` is at least that; LFR_EINVAL for NULL or inconsistent arrays.  The element hashes
 * run on up to 8 helper threads (LFR_HOST_THREADS overrides the count); the bytes do not depend on it. */
int64_t lfr_host_problem_record(const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat,
                                uint32_t n_images, const uint8_t* names, const uint64_t* name_off, uint8_t* out,
                                uint64_t cap);

/* The host form of lfr_plan_update_solution_since_record() (include/lfr_graph.h), bit for bit: as
 * lfr_wire_update_solution_since(), with the compare against the earlier run's record (record_len bytes)
 * in place of its MatchingFile: a component is changed when its digest is not in the record.  LFR_EINVAL
 * for malformed SolutionFile bytes, a malformed record, NULL or inconsistent arrays.  Every output is
 * untouched on error. */
int lfr_wire_update_solution_since_record(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names,
                                          const uint64_t* name_off, const lfr_problem* p, const uint32_t* node_image,
                                          const uint32_t* node_feat, const uint8_t* record, uint64_t record_len,
                                          double* positions /* [2 n_nodes] */, uint8_t* held /* [n_nodes] */,
                                          uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed);

/* The host form of lfr_plan_update_solution_groups() (include/lfr_graph.h), bit for bit: many scenes of one run,
 * image id k in scene group_of_image[k] < n_groups, each updated from its own SolutionFile (files[g], file_len[g]
 * bytes, decoded against scene g's image ids alone; NULL: no entry, so every component of the scene is touched)
 * and, where records[g] is not NULL, against its own earlier record (record_len[g] bytes; a component of scene g
 * is changed when its digest is not in records[g]).  `files` or `records` may be NULL for none at all.
 * *n_changed counts the changed components of the scenes with a record.  LFR_EINVAL for a SolutionFile that does
 * not parse, a malformed record, a group out of range, a component whose nodes span two scenes, NULL or
 * inconsistent arrays.  Every output is untouched on error. */
int lfr_wire_update_solution_groups(uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                                    const uint32_t* group_of_image, uint32_t n_groups, const uint8_t* const* files,
                                    const uint64_t* file_len, const uint8_t* const* records, const uint64_t* record_len,
                                    const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat,
                                    double* positions /* [2 n_nodes] */, uint8_t* held /* [n_nodes] */,
                                    uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed);

/* The host form of lfr_plan_problem_record_groups() (include/lfr_graph.h), the same bytes: the problem record of
 * every scene g < n_groups of `p` (image id k in scene group_of_image[k]), each what lfr_host_problem_record()
 * writes for the scene's own run, back to back; scene g's is out[group_off[g], group_off[g + 1]).
 * group_off[0..n_groups] is always filled; the records are written when `cap` holds them all.  Returns the total
 * size, or LFR_EINVAL as lfr_host_problem_record() and for a group out of range or a component whose nodes span
 * two scenes. */
int64_t lfr_host_problem_record_groups(const lfr_problem* p, const uint32_t* node_image, const uint32_t* node_feat,
                                       uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                                       const uint32_t* group_of_image, uint32_t n_groups, uint8_t* out, uint64_t cap,
                                       uint64_t* group_off);

#ifdef __cplusplus
}
#endif
#endif /* LFR_HOST_H_ */
