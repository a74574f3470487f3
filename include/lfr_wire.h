/*
 * lfr_wire.h — C ABI of the protobuf wire codec for types.proto.
 *
 * The reference parses MatchingFile with libprotobuf's generated classes
 * (solve.cc:426-436) and walks the message tree match by match
 * (solve.cc:438-480); it writes SolutionFile with SerializeToOstream
 * (solve.cc:643-679).  These entry points decode the same bytes straight into
 * the flat arrays the solver consumes and encode the solution, without a
 * protobuf dependency.  Host-only code: no GPU needed.
 *
 * Wire facts (proto3): unknown fields are skipped; absent scalars default to 0
 * (the encoder omits zero scalars, so `Displacement{0,0}` is an empty message);
 * `disp1`/`disp2` shorter than 9 entries leave the remaining grid samples 0 and
 * entries beyond the 9th are ignored (solve.cc:460-472 would write out of
 * bounds there).
 */
#ifndef LFR_WIRE_H_
#define LFR_WIRE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Count image pairs and matches of one MatchingFile buffer (types.proto:3-28).
 * Walks the pair level only (a match is skipped by its length prefix); the
 * contents of the matches are validated by lfr_wire_decode_matches.  Returns 0,
 * or LFR_EINVAL on malformed input ("Failed to parse proto object.",
 * solve.cc:433-436) — a buffer is well-formed iff scan AND decode return 0. */
int lfr_wire_scan_matches(const uint8_t* buf, uint64_t len, uint64_t* n_pairs,
                          uint64_t* n_matches);

typedef struct lfr_wire_matches {
  uint64_t n_pairs, n_matches;     /* capacities, from lfr_wire_scan_matches */
  uint64_t* pair_ptr;              /* [n_pairs+1] matches of pair p           */
  float* fact1;                    /* [n_pairs]  types.proto:6                */
  float* fact2;                    /* [n_pairs]  types.proto:8                */
  uint64_t* name1_off;             /* [n_pairs]  image_name1 = buf[off, off+len) */
  uint32_t* name1_len;
  uint64_t* name2_off;
  uint32_t* name2_len;
  uint32_t* feat1;                 /* [n_matches] feature_idx1                */
  uint32_t* feat2;                 /* [n_matches] feature_idx2                */
  float* sim;                      /* [n_matches] similarity                  */
  float* disp1;                    /* [n_matches*18] (di, dj) x 9             */
  float* disp2;                    /* [n_matches*18]                          */
} lfr_wire_matches;

int lfr_wire_decode_matches(const uint8_t* buf, uint64_t len, lfr_wire_matches* out);

/* The pair level of lfr_wire_decode_matches without decoding any match: fills pair_ptr, fact1/2 and the
 * name offsets and lengths of `out` (feat1 ... disp2 are not touched and may be NULL), and
 * match_off[k] = the byte offset in `buf` of match k's length prefix (the byte after its tag), for
 * k < out->n_matches.  Same walk and same capacity rules as lfr_wire_decode_matches, so it returns
 * LFR_EINVAL exactly when lfr_wire_scan_matches does (or the capacities are wrong); the contents of the
 * matches are left to the decoder (lfr_plan_create_from_wire, include/lfr_graph.h). */
int lfr_wire_walk_matches(const uint8_t* buf, uint64_t len, lfr_wire_matches* out, uint64_t* match_off);

/* Encode a MatchingFile.  names are concatenated in `names`, name k =
 * names[name_off[k], name_off[k+1]).  pair_name1/2[p] index names.
 * Returns the number of bytes needed; writes only if cap is large enough. */
int64_t lfr_wire_encode_matches(uint64_t n_pairs, const uint64_t* pair_ptr,
                                const uint32_t* pair_name1, const uint32_t* pair_name2,
                                const float* fact1, const float* fact2,
                                const uint8_t* names, const uint64_t* name_off,
                                const uint32_t* feat1, const uint32_t* feat2, const float* sim,
                                const float* disp1, const float* disp2,
                                uint8_t* out, uint64_t cap);

/* Encode a SolutionFile (types.proto:30-46): image i has displacements
 * [img_ptr[i], img_ptr[i+1]) of (feature_idx, di, dj).  Same size protocol. */
int64_t lfr_wire_encode_solution(uint64_t n_images, const uint64_t* img_ptr,
                                 const uint8_t* names, const uint64_t* name_off,
                                 const float* fact, const uint32_t* feature_idx,
                                 const float* di, const float* dj,
                                 uint8_t* out, uint64_t cap);

/* Decode a SolutionFile into flat arrays (used by tests and by consumers).
 * Pass 1: out arrays NULL -> counts only. */
int lfr_wire_decode_solution(const uint8_t* buf, uint64_t len, uint64_t* n_images,
                             uint64_t* n_disp, uint64_t* img_ptr, uint64_t* name_off,
                             uint32_t* name_len, float* fact, uint32_t* feature_idx,
                             float* di, float* dj);

#ifdef __cplusplus
}
#endif
#endif /* LFR_WIRE_H_ */
