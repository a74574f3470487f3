/*
 * lfr_graph.h — the graph stage on the GPU: from the decoded match arrays straight to a
 * device-resident plan (include/lfr.h).
 *
 * lfr_plan_create_from_matches() uploads the flat match arrays of lfr_host_input once and builds,
 * on the device, everything lfr_host_stage_create() + lfr_host_stage_export() produce (solve.cc:438-606):
 * node interning, the CSR edge lists and their 80-byte records, the constrained Kruskal, track ids and
 * roots, the track meta-graph and its components, the dispatch list.  Every array is bitwise equal to
 * the host stage's.  Only the recursive 2-way cut of oversized meta-components runs on the host, on
 * the downloaded edges of those components (the same code as the host stage, lfr_cut.h).  Its device
 * twin (lfr_cut.cuh, the same groups, no host round trip) runs under LFR_DBG_DEVICE_CUT; it measured
 * slower on an H100 on every workload up to cfg5, so it is not the default.  The edge
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

/* lfr_plan_create_from_wire() for a batch whose pairs are listed out of one MatchingFile (--listed_pairs): the
 * file's matches are decoded once on the device, in file order, and the batch's match arrays are then built
 * there from the entry list.  Entry k (k < in->n_pairs) is the file's pair pair_src[k] (< n_src_pairs); entries
 * may repeat and reorder pairs.  src_pair_ptr [n_src_pairs + 1] is the file's pair level from
 * lfr_wire_walk_matches() over the parts in order (global match offsets, as in->pair_ptr of
 * lfr_plan_create_from_wire()); the parts' n_matches add up to src_pair_ptr[n_src_pairs].  `in` carries the
 * batch's pair level: entry k's images and sub-scene (pair_img1/2, pair_skip, image_group) and pair_ptr, which
 * must be the exclusive scan of the entries' match counts (in->n_matches its total).  The expand is a scan of
 * those counts on the device and a gather that copies each match's feature indices, similarity and two
 * 18-float grids to its entry, bit for bit, so the result is bitwise lfr_plan_create_from_matches() on the
 * host decode of the file with every entry's matches copied into place.  Errors: those of
 * lfr_plan_create_from_wire(), and LFR_EINVAL for NULL arrays, a source pair out of range, a decreasing
 * src_pair_ptr or a pair_ptr that is not that scan. */
int lfr_plan_create_from_wire_listed(const lfr_host_input* in, const lfr_wire_part* parts, uint32_t n_parts,
                                     const uint64_t* src_pair_ptr, uint64_t n_src_pairs, const uint64_t* pair_src,
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

/* The SolutionFile (types.proto:30-46) of a plan made by lfr_plan_create_from_matches() or _from_wire(),
 * encoded on the device from the plan's current positions (the last lfr_plan_solve()'s result; the
 * initial positions before the first solve).  names / name_off / fact are indexed by image id (the ids of
 * lfr_host_input, n_images at least its n_images), name k = names[name_off[k], name_off[k+1]).  The bytes
 * are those of the host assembly of solve.cc:643-679 — lfr_plan_download(), images in order of their
 * lowest node index, displacements in ascending node index, di / dj = (float) of the fp64 positions as
 * x86 rounds them (NaN payloads included) — passed to lfr_wire_encode_solution().  Returns the bytes
 * needed and writes them to `out` only when cap >= that (the size protocol of lfr_wire_encode_solution);
 * *n_outside (may be NULL) = "# points with at least one coordinate > 0.5" (solve.cc:666-670), counted on
 * the fp64 positions.  A plan with no node encodes to 0 bytes.  Negative LFR_E* on error; LFR_EINVAL for
 * a plan made by lfr_plan_create().  The node ids stay on the device for this (8 B per node). */
int64_t lfr_plan_encode_solution(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                 const uint64_t* name_off, const float* fact, uint8_t* out, uint64_t cap,
                                 uint64_t* n_outside);

/* lfr_plan_encode_solution() restricted to the images k with written[k] != 0 (--query_images writes the query
 * images only): the other images get no Image message, and the bytes are those of the full encoding with
 * their Image messages left out.  *n_outside still counts every node.  Same size protocol and errors, and
 * LFR_EINVAL for a NULL `written`. */
int64_t lfr_plan_encode_solution_images(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                        const uint64_t* name_off, const float* fact, const uint8_t* written, uint8_t* out,
                                        uint64_t cap, uint64_t* n_outside);

/* The SolutionFiles of a batch of scenes (--additional_scenes) in one device pass: image k belongs to group
 * group_of_image[k] (< n_groups).  Group g's bytes are out[group_off[g], group_off[g+1]), equal to
 * lfr_plan_encode_solution_images() with written = the images of group g, and n_outside[g] counts the nodes of
 * group g's images only.  A group with no node encodes to 0 bytes.  group_off [n_groups + 1] and n_outside
 * [n_groups] are filled on every successful call; the return value is the total, group_off[n_groups], and the
 * bytes are written only when cap >= that (the size protocol of lfr_plan_encode_solution).  The groups are
 * encoded together, not one after the other: a thousand groups cost one encode.  LFR_EINVAL as
 * lfr_plan_encode_solution(), or for NULL group_of_image / group_off / n_outside or a group id >= n_groups. */
int64_t lfr_plan_encode_solution_groups(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                        const uint64_t* name_off, const float* fact, const uint32_t* group_of_image,
                                        uint32_t n_groups, uint8_t* out, uint64_t cap, uint64_t* group_off /* [n_groups+1] */,
                                        uint64_t* n_outside /* [n_groups] */);

/* lfr_plan_encode_solution() merged with an earlier SolutionFile `file`: the scene's output, each scene
 * image followed by its carried entries, then the file's other winning Image messages — the bytes of
 * lfr_wire_encode_solution_carried() (include/lfr_wire.h, which states the rule) on the plan's host assembly
 * (lfr_plan_download() and the assembly lfr_plan_encode_solution() describes).  A scene image is one with at
 * least one node; a name among names / name_off without a node (every pair banned, no match) is not one,
 * so the file's entries for it come after the scene images, as for a name outside the scene.  The file is
 * decoded on the host (lfr_wire_decode_solution); keying, the stable sort, the winners, the join to the
 * nodes, the compaction and the encoding of the N node records plus the carried ones run on the device.
 * Size protocol, `stream` and *n_outside (the scene's nodes only) as lfr_plan_encode_solution();
 * *n_carried (may be NULL) = the carried entries.  The plan is not changed.  LFR_EINVAL for malformed bytes,
 * repeated image names, NULL arrays and a plan made by lfr_plan_create(); LFR_EUNSUPPORTED for 2^31 or
 * more nodes plus displacements. */
int64_t lfr_plan_encode_solution_carried(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                         const uint64_t* name_off, const float* fact, const uint8_t* file,
                                         uint64_t file_len, uint8_t* out, uint64_t cap, uint64_t* n_outside,
                                         uint64_t* n_carried);

/* Hold images fixed in a plan made by lfr_plan_create_from_matches() or _from_wire(): every node of an
 * image k with fixed_by_image_id[k] != 0 (ids of lfr_host_input, n_images at least its n_images) becomes
 * constant, as a root is (solve.cc:135): it keeps its start value, gets no bounds, and a block between two
 * constant nodes is dropped.  The mask (reference root OR node of a fixed image) is expanded on the device
 * over the plan's node ids and the schedule is built again on it (free-node counts move components between
 * tiers); lfr_plan_export_graph() still reports the reference's is_root.  A later call replaces the mask
 * (an all-zero one solves as a plan never given one).  A plan never given a mask reads is_root as before and
 * holds no mask buffer.  Synchronous on the legacy default stream.  LFR_EINVAL for a plan made by
 * lfr_plan_create(), whose lfr_problem.is_root already says which nodes are constant. */
int lfr_plan_fix_images(lfr_plan* plan, const uint8_t* fixed_by_image_id /* [n_images] */, uint32_t n_images);

/* Start a plan made by lfr_plan_create_from_matches() or _from_wire() from a SolutionFile (types.proto:30-46):
 * names / name_off are the scene's image names by id, as for lfr_plan_encode_solution().  The bytes are
 * decoded on the host (lfr_wire_decode_solution), the entries keyed (image id << 32 | feature_idx) and
 * joined to the plan's node ids on the device, with the rule of lfr_wire_join_solution()
 * (include/lfr_wire.h), whose positions these are bit for bit.  Writes the plan's start and working
 * positions (lfr_plan_download() and lfr_plan_encode_solution() see them before the next solve, which starts
 * from them: free nodes are projected onto the box, constant nodes keep them).  *n_started (may be NULL) =
 * the nodes with an entry.  Returns after the join, on `stream`.  LFR_EINVAL for malformed bytes (the plan is
 * not changed) and for a plan made by lfr_plan_create(), which takes its start point at creation. */
int lfr_plan_start_from_solution(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                                 const uint8_t* names, const uint64_t* name_off, uint64_t* n_started);

/* Keep what an earlier SolutionFile refined and refine everything else: lfr_plan_start_from_solution() (the
 * same single host decode and device join, the same start and working positions bit for bit), and every
 * node with an entry in the file (the rule of lfr_wire_join_solution_entries(), include/lfr_wire.h) becomes
 * constant, as a node of a fixed image is.  The mask is reference root OR node of an image fixed by
 * lfr_plan_fix_images() OR kept node; the per-image mask and the kept flags are separate inputs, so the two
 * calls compose in either order, and the schedule is built again on the mask.  A later call, or a later
 * lfr_plan_update_solution(), replaces the kept set (an empty SolutionFile clears it); a later lfr_plan_start_from_solution() changes only the start
 * values.  A plan never given a kept set holds no buffer for one.  *n_kept (may be NULL) = the nodes with an
 * entry.  Synchronous on `stream`.  LFR_EINVAL for malformed bytes (the plan is not changed) and for a plan
 * made by lfr_plan_create(). */
int lfr_plan_keep_solution(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                           const uint8_t* names, const uint64_t* name_off, uint64_t* n_kept);

/* Update an earlier SolutionFile with new keypoints: solve again, from scratch, every component a keypoint
 * without an entry in the file joins, and hold every other component at the file's values.  A component is
 * an entry of the plan's dispatch list (lfr_problem.comp: after the cut; a component of one node counts
 * too).  It is touched when at least one of its nodes has no entry (the rule of
 * lfr_wire_join_solution_entries(), include/lfr_wire.h).
 *   - a touched component's nodes start at 0 and are held only when the reference or lfr_plan_fix_images()
 *     says so: it solves bit for bit as in a plan never given a file;
 *   - an untouched component's nodes start at their entries and are all held: it ends LFR_TERM_EMPTY (or
 *     SKIPPED at one node) with the file's values.
 * The same single host decode and device join as lfr_plan_keep_solution(); one kernel marks the touched
 * components, one writes the start and working positions and the held flags (entry AND component not
 * touched) that the constant mask ORs in place of the kept flags, and the schedule is built again.  The held
 * set and the kept set are one input: the last lfr_plan_keep_solution() or lfr_plan_update_solution() call
 * wins, and an empty file clears it (every component is touched then).  It composes with
 * lfr_plan_fix_images() in either order.  A plan never given the call allocates nothing for it.
 * *n_held (may be NULL) = the held nodes, *n_touched (may be NULL) = the touched components; both are what
 * lfr_wire_update_solution() counts.  Synchronous on `stream`.  LFR_EINVAL for malformed bytes (the plan is
 * not changed) and for a plan made by lfr_plan_create(). */
int lfr_plan_update_solution(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                             const uint8_t* names, const uint64_t* name_off, uint64_t* n_held, uint32_t* n_touched);

/* lfr_plan_update_solution() that also sees every change of the matches since the earlier run: given the
 * MatchingFile that produced the SolutionFile, it holds a component only when its problem is the problem the
 * earlier run solved, and touches every other one.
 *
 * The rule.  The *earlier run* is the graph stage (solve.cc:438-606) over every pair of the earlier
 * MatchingFile OLD, no image banned (a run that banned images is described by a file without their pairs);
 * its cut cap is OLD's own image count.  A keypoint is identified by (exact image-name bytes, feature_idx).
 * A component C of this plan (lfr_problem.comp, after the cut; one-node components count) is *unchanged*
 * when the earlier run has a component C' such that
 *   1. C' has the same keypoints as C;
 *   2. the same keypoints are roots (the reference's is_root) in both;
 *   3. every keypoint has the same multiset of kept out-edges in both.  An edge is kept when its kind is not
 *      LFR_EDGE_SKIP (same track: Cauchy, same component: Tukey); it is compared on its destination keypoint,
 *      its kind and the bits of sim and of the 18 flow floats (-0.0 is not +0.0; NaN payloads count).
 * Skipped edges and the order of nodes and edges do not enter the rule, and the comparison is exact.  C is
 * *held* when it is unchanged AND every one of its keypoints has an entry in the SolutionFile (the rule of
 * lfr_wire_join_solution_entries()); every other component is *touched* and treated as
 * lfr_plan_update_solution() treats its touched components: it starts at 0 with the constant mask root OR
 * fixed image, and solves bit for bit as in a plan never given a file.  A held component's nodes are all
 * constant at the file's float bits.  The touched set contains lfr_plan_update_solution()'s.
 *
 * `previous` is a plan made by lfr_plan_create_from_matches() or _from_wire() from OLD on the same device;
 * it is read, not changed, and may be destroyed when the call returns.  prev_names / prev_name_off are its
 * image names by id (prev_n_images at least its n_images), mapped to this plan's names / name_off by their
 * bytes; names only the earlier run has get ids after this plan's.  Keys, sorts, joins and the exact compare
 * run on the device (csrc/lfr_diff.cuh); the held flags, start positions, constant mask and schedule are
 * lfr_plan_update_solution()'s.  *n_held, *n_touched (each may be NULL) as lfr_plan_update_solution();
 * *n_changed (may be NULL) = the components that are not unchanged.  Synchronous on `stream`.  LFR_EINVAL as
 * lfr_plan_update_solution(), for a `previous` not made from matches, on another device or equal to `plan`,
 * and for malformed or repeated earlier names (the plan is not changed then); LFR_EUNSUPPORTED for 2^31 or
 * more directed edges in the two plans together.  lfr_wire_update_solution_since() (include/lfr_host.h) is
 * the host form, bit for bit. */
int lfr_plan_update_solution_since(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                                   const uint8_t* names, const uint64_t* name_off, const lfr_plan* previous,
                                   uint32_t prev_n_images, const uint8_t* prev_names, const uint64_t* prev_name_off,
                                   uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed);

/* The problem record of a run: one 128-bit digest per component, so that a later update can ask "was this
 * exact problem solved before?" without the earlier MatchingFile or its graph stage (about 16 bytes per
 * component instead of the earlier run's arrays).  Each run writes the record the next one reads.
 *
 * The record, exactly (csrc/lfr_record.h has the code, for the host library and the kernels alike):
 *   - S(k, m) is SipHash-2-4 (Aumasson and Bernstein) with the 16-byte key k, the message m hashed as its
 *     little-endian bytes.  H(m) = (S(K0, m), S(K1, m)), K0 = the 16 ASCII bytes "lfr problem rec0",
 *     K1 = "lfr problem rec1".
 *   - The name id of an image is H(exact name bytes).  A keypoint is (name id, feature_idx).
 *   - The node element of node v is 4 little-endian u64 words [0x4e, id(v).0, id(v).1, feat(v) | root(v) << 32],
 *     root = the reference's is_root (not a constant mask).
 *   - The edge element of each kept out-edge v -> w is 16 little-endian u64 words [0x45, id(v).0, id(v).1,
 *     id(w).0, id(w).1, feat(v) | feat(w) << 32, kind | bits(sim) << 32, bits(flow[2i]) | bits(flow[2i+1]) << 32
 *     for i = 0..8], flow in lfr_edge.flow order.  Kept and kind as the solve classifies edges: same track
 *     gives LFR_EDGE_CAUCHY, otherwise same component LFR_EDGE_TUKEY, otherwise the edge is skipped.
 *   - Digest(C) = (sum H(x).0, sum H(x).1) mod 2^64 over the node elements of C's nodes and the edge elements
 *     of their kept out-edges.  It depends on neither node nor edge order, counts multiplicity, and is exact
 *     integer arithmetic: any reduction order gives the same bits.
 *   - The record is the 8 bytes "LFRPREC1", u64 C, then the C digests as (d0, d1) u64 pairs in ascending
 *     (d0, d1) order: 16 + 16 C bytes.  A reader refuses any other length or magic and digests out of order.
 * The record describes the graph stage as it ran (its banned images and its cut cap); it does not depend on
 * fixed images, on a kept or held set or on the start point.
 *
 * `plan` is made from matches.  Name ids are hashed on the host from names / name_off (n_images, at least
 * the plan's image count); elements are hashed and summed per component on the device (csrc/lfr_record.cuh)
 * and a radix sort orders the digests.  Returns the record's size and writes it to `out` only when `cap` is
 * at least that (lfr_plan_encode_solution's protocol); LFR_EINVAL for a plan made by lfr_plan_create() or
 * malformed names.  Synchronous on `stream`.  The plan is not changed: a solve after the call is bitwise the
 * same.  lfr_host_problem_record() (include/lfr_host.h) is the host form, byte for byte. */
int64_t lfr_plan_problem_record(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                const uint64_t* name_off, uint8_t* out, uint64_t cap);

/* lfr_plan_update_solution_since() against the earlier run's problem record instead of its MatchingFile.
 * The held rule is the same with the compare replaced by digest membership: C is *unchanged* when Digest(C)
 * appears in the record, *held* when it is unchanged and every keypoint of C has an entry in the SolutionFile;
 * every other component is *touched* and behaves as in lfr_plan_update_solution_since().  *n_changed counts
 * the components whose digest is absent.  The held flags, start positions, constant mask and schedule are the
 * same code as lfr_plan_update_solution_since()'s.  Errors as lfr_plan_update_solution(), plus LFR_EINVAL for a
 * malformed record; the plan is not changed on error.  lfr_wire_update_solution_since_record()
 * (include/lfr_host.h) is the host form, bit for bit.
 *
 * Limits.  Equal digests are not exact equality: two different problems share a digest only when two different
 * multisets of element hashes have equal sums in both lanes.  For a random function that has probability 2^-128
 * when some multiplicity differs by an odd count, and 2^-(128-2t) when every difference is divisible by 2^t.
 * lfr_plan_update_solution_since() stays the exact path and needs no record; it is the only option when the
 * SolutionFile came from an older build or from the reference binary.  When the record was written by a run on
 * OLD that banned no image, the two calls give identical results. */
int lfr_plan_update_solution_since_record(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len,
                                          uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                                          const uint8_t* record, uint64_t record_len, uint64_t* n_held,
                                          uint32_t* n_touched, uint32_t* n_changed);

/* Many scenes of one plan, each updated as its own run: image id k belongs to scene group_of_image[k] < n_groups
 * (as for lfr_plan_encode_solution_groups; every component lies in one scene).  Scene g's SolutionFile is files[g]
 * (file_len[g] bytes), decoded on the host against scene g's image ids alone, since scenes reuse image names; a
 * NULL file has no entry, so every component of the scene is touched and solves bit for bit as from zeros.  With
 * records[g] (record_len[g] bytes) scene g follows lfr_plan_update_solution_since_record() against that record,
 * looked up within the scene alone (one kernel binary-searches scene g's slice of all the records); a NULL record
 * gives scene g the rule of lfr_plan_update_solution().  `files` or `records` may be NULL for none at all.
 * Every scene's entries are keyed by scene image id and joined in one pass, and the touch, update and schedule
 * steps are those of lfr_plan_update_solution(): the kernel launches, CUB calls and copies do not grow with
 * n_groups.  *n_held and *n_touched are sums over the scenes; *n_changed counts the changed components of the
 * scenes with a record.  With n_groups == 1 the call is lfr_plan_update_solution() (NULL record) or
 * lfr_plan_update_solution_since_record(), bit for bit.  Errors as those calls, plus LFR_EINVAL for a group out of
 * range; the plan is not changed on error.  lfr_wire_update_solution_groups() (include/lfr_host.h) is the host
 * form, bit for bit. */
int lfr_plan_update_solution_groups(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                    const uint64_t* name_off, const uint32_t* group_of_image, uint32_t n_groups,
                                    const uint8_t* const* files, const uint64_t* file_len, const uint8_t* const* records,
                                    const uint64_t* record_len, uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed);

/* The problem record of every scene of a plan (scenes as for lfr_plan_update_solution_groups): scene g's is
 * out[group_off[g], group_off[g + 1]), byte for byte lfr_plan_problem_record() of a plan of scene g alone.  The
 * digests are computed once on the device, ordered by (scene, d0, d1) with three stable radix sorts, and every
 * header and digest is written in one device pass and copied out once; nothing grows with n_groups but the offsets.
 * group_off[0..n_groups] is always filled; the records are written when `cap` holds them all
 * (lfr_plan_encode_solution_groups' protocol).  Returns the total size, or the errors of lfr_plan_problem_record()
 * and LFR_EINVAL for a group out of range or a NULL group_off.  The plan is not changed.
 * lfr_host_problem_record_groups() (include/lfr_host.h) is the host form, byte for byte. */
int64_t lfr_plan_problem_record_groups(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                       const uint64_t* name_off, const uint32_t* group_of_image, uint32_t n_groups,
                                       uint8_t* out, uint64_t cap, uint64_t* group_off);

/* A test hook: the calling thread's device operations since the last reset, {kernel launch sites checked, CUB
 * calls, synchronising copies to the host}, into out3 (may be NULL); reset != 0 zeroes them. */
int lfr_debug_device_ops(unsigned long long* out3, int reset);

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
