// lfr_join.h — the host half of a start point read from a SolutionFile (types.proto:30-46), shared by the
// host joins (lfr_wire_join_solution, _entries and lfr_wire_update_solution, lfr_wire.cc), the device join
// (lfr_plan_start_from_solution, lfr_plan_keep_solution and lfr_plan_update_solution, lfr_capi.cu) and the
// carried encoders
// (lfr_wire_encode_solution_carried, lfr_plan_encode_solution_carried): the decode with
// lfr_wire_decode_solution() and the image rule, and the host joins' node loop.  Header-only host code.
//
// The rule is that of the reference's own reader (reconstruction-scripts/colmap_utils.py:104-137): an
// Image message is matched to a scene image by its exact name bytes, and the last Image message with a
// given name wins as a whole; within it, the last displacement of a feature wins.  Each displacement of a
// winning message gets the key (image id << 32 | feature_idx), as the encoder keys its nodes; every other
// displacement gets kNoKey, which no node has (image ids are < 2^32 - 1).  Scene image ids that share a name
// (--query_images gives a database image one id per sub-scene) all join the entries of that name: a node of
// image k is keyed with the lowest id of k's name (Decoded::canon).
#ifndef LFR_JOIN_H_
#define LFR_JOIN_H_

#include <algorithm>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/lfr.h"
#include "../../include/lfr_wire.h"

namespace lfr {
namespace join {

constexpr uint32_t kNoImage = 0xffffffffu;
constexpr uint64_t kNoKey = ~0ull;

inline uint64_t node_key(uint32_t image, uint32_t feature) { return (uint64_t)image << 32 | feature; }

struct Decoded {
  uint64_t n_images = 0, n_disp = 0;
  std::vector<uint64_t> img_ptr, name_off;
  std::vector<uint32_t> name_len, feature_idx;
  std::vector<float> fact, di, dj;
  // per decoded Image message: the scene image id its displacements belong to, or kNoImage (a name not in
  // the scene, or a later message with the same name)
  std::vector<uint32_t> image_id;
  // per decoded Image message: 1 when it is the last one with its name (it wins as a whole), whether or not
  // the name is a scene image's
  std::vector<uint8_t> wins;
  // per scene image id: the lowest id with the same name, the image whose entries it joins; empty when every
  // scene name is distinct (then each id is its own)
  std::vector<uint32_t> canon;
};

// Decode `buf` and resolve its images against the scene's names (name k = names[name_off[k], name_off[k+1])).
// LFR_EINVAL when the bytes do not parse.
inline int decode(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                  Decoded& d) {
  if (lfr_wire_decode_solution(buf, len, &d.n_images, &d.n_disp, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                               nullptr) != LFR_OK)
    return LFR_EINVAL;
  const uint64_t I = d.n_images, D = d.n_disp;
  d.img_ptr.assign(I + 1, 0);
  d.name_off.assign(I, 0);
  d.name_len.assign(I, 0);
  d.fact.assign(I, 0.f);
  d.feature_idx.assign(D, 0);
  d.di.assign(D, 0.f);
  d.dj.assign(D, 0.f);
  if (lfr_wire_decode_solution(buf, len, &d.n_images, &d.n_disp, d.img_ptr.data(), d.name_off.data(), d.name_len.data(),
                               d.fact.data(), d.feature_idx.data(), d.di.data(), d.dj.data()) != LFR_OK)
    return LFR_EINVAL;
  std::unordered_map<std::string, uint32_t> id_of;
  id_of.reserve(n_images);
  d.canon.clear();
  for (uint32_t k = 0; k < n_images; ++k) {
    const auto it =
        id_of.emplace(std::string(reinterpret_cast<const char*>(names) + name_off[k], name_off[k + 1] - name_off[k]), k);
    if (!it.second && d.canon.empty()) {
      d.canon.resize(n_images);
      for (uint32_t j = 0; j < n_images; ++j) d.canon[j] = j;
    }
    if (!d.canon.empty()) d.canon[k] = it.first->second;
  }
  std::unordered_map<std::string, uint64_t> last;  // the last Image message of each name in the file
  last.reserve(I);
  for (uint64_t i = 0; i < I; ++i)
    last[std::string(reinterpret_cast<const char*>(buf) + d.name_off[i], d.name_len[i])] = i;
  d.image_id.assign(I, kNoImage);
  d.wins.assign(I, 0);
  for (const auto& nl : last) {
    d.wins[nl.second] = 1;
    const auto it = id_of.find(nl.first);
    if (it != id_of.end()) d.image_id[nl.second] = it->second;
  }
  return LFR_OK;
}

// The effective entries of decoded Image message i: the last displacement of each feature, in ascending
// feature_idx (indices into d.feature_idx / di / dj).
inline void effective_entries(const Decoded& d, uint64_t i, std::vector<uint64_t>& out) {
  out.clear();
  for (uint64_t k = d.img_ptr[i]; k < d.img_ptr[i + 1]; ++k) out.push_back(k);
  std::stable_sort(out.begin(), out.end(), [&d](uint64_t a, uint64_t b) { return d.feature_idx[a] < d.feature_idx[b]; });
  size_t w = 0;
  for (size_t j = 0; j < out.size(); ++j)
    if (j + 1 == out.size() || d.feature_idx[out[j + 1]] != d.feature_idx[out[j]]) out[w++] = out[j];
  out.resize(w);
}

// The host join of a decoded file: positions[2v .. 2v+1] from node v's entry, 0 without one; has_entry[v] (may be
// NULL) = whether it has one
inline void join_decoded(const Decoded& d, uint32_t n_nodes, const uint32_t* node_image, const uint32_t* node_feat,
                         double* positions, uint8_t* has_entry, uint64_t* n_started) {
  // (key, displacement) sorted by key, stably: the last entry of a run of equal keys is the last occurrence
  std::vector<std::pair<uint64_t, uint64_t>> keyed;
  keyed.reserve(d.n_disp);
  for (uint64_t i = 0; i < d.n_images; ++i)
    if (d.image_id[i] != kNoImage)
      for (uint64_t k = d.img_ptr[i]; k < d.img_ptr[i + 1]; ++k) keyed.emplace_back(node_key(d.image_id[i], d.feature_idx[k]), k);
  std::stable_sort(keyed.begin(), keyed.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  uint64_t started = 0;
  for (uint32_t v = 0; v < n_nodes; ++v) {
    const uint64_t key = node_key(d.canon.empty() ? node_image[v] : d.canon[node_image[v]], node_feat[v]);
    const auto it = std::upper_bound(keyed.begin(), keyed.end(), key,
                                     [](uint64_t x, const std::pair<uint64_t, uint64_t>& e) { return x < e.first; });
    double a = 0.0, b = 0.0;
    const bool hit = it != keyed.begin() && (it - 1)->first == key;
    if (hit) {
      a = (double)d.di[(it - 1)->second];
      b = (double)d.dj[(it - 1)->second];
      ++started;
    }
    positions[2 * (size_t)v] = a;
    positions[2 * (size_t)v + 1] = b;
    if (has_entry) has_entry[v] = hit ? 1 : 0;
  }
  if (n_started) *n_started = started;
}

// The checks of every host join on the scene's names: NULL arguments, descending name_off
inline bool names_ok(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                     uint32_t n_nodes, const uint32_t* node_image, const uint32_t* node_feat, const double* positions) {
  if ((!buf && len) || (n_images && !name_off) || (n_nodes && (!node_image || !node_feat || !positions))) return false;
  for (uint32_t k = 0; k < n_images; ++k)
    if (name_off[k + 1] < name_off[k]) return false;
  return !(n_images && name_off[n_images] && !names);
}

// The host join (lfr_wire_join_solution / _entries): join_decoded() of `buf`.  Every output is untouched when the
// arguments or the bytes are rejected (LFR_EINVAL).
inline int join_nodes(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                      uint32_t n_nodes, const uint32_t* node_image, const uint32_t* node_feat, double* positions,
                      uint8_t* has_entry, uint64_t* n_started) {
  if (!names_ok(buf, len, n_images, names, name_off, n_nodes, node_image, node_feat, positions)) return LFR_EINVAL;
  const uint8_t no_name = 0;
  Decoded d;
  if (decode(buf, len, n_images, names ? names : &no_name, name_off, d) != LFR_OK) return LFR_EINVAL;
  join_decoded(d, n_nodes, node_image, node_feat, positions, has_entry, n_started);
  return LFR_OK;
}

// The touch rule after a join whose has-entry flags are in `held`: every component with a node without an entry
// is touched, and so is every component with changed[c] != 0 (`changed` may be NULL: none); a touched component's
// nodes start at 0 and are not held.  held[v] = has entry AND component not touched.
inline void touch_components(uint32_t n_nodes, const uint32_t* node_comp, uint32_t n_components, double* positions,
                             uint8_t* held, uint64_t* n_held, uint32_t* n_touched, const uint8_t* changed) {
  std::vector<uint8_t> touched(n_components, 0);
  if (changed)
    for (uint32_t c = 0; c < n_components; ++c) touched[c] = changed[c] ? 1 : 0;
  for (uint32_t v = 0; v < n_nodes; ++v)
    if (!held[v]) touched[node_comp[v]] = 1;
  uint64_t nh = 0;
  for (uint32_t v = 0; v < n_nodes; ++v) {
    if (touched[node_comp[v]]) {
      positions[2 * (size_t)v] = 0.0;
      positions[2 * (size_t)v + 1] = 0.0;
      held[v] = 0;
    }
    nh += held[v];
  }
  if (n_held) *n_held = nh;
  if (n_touched) *n_touched = (uint32_t)std::count(touched.begin(), touched.end(), (uint8_t)1);
}

// The host update (lfr_wire_update_solution): join_nodes() with its flags, then touch_components() (`changed`:
// lfr_wire_update_solution_since).  Every output is untouched when the arguments or the bytes are rejected
// (LFR_EINVAL).
inline int update_nodes(const uint8_t* buf, uint64_t len, uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                        uint32_t n_nodes, const uint32_t* node_image, const uint32_t* node_feat, const uint32_t* node_comp,
                        uint32_t n_components, double* positions, uint8_t* held, uint64_t* n_held, uint32_t* n_touched,
                        const uint8_t* changed = nullptr) {
  if (n_nodes && (!node_comp || !held)) return LFR_EINVAL;
  for (uint32_t v = 0; v < n_nodes; ++v)
    if (node_comp[v] >= n_components) return LFR_EINVAL;
  const int rc = join_nodes(buf, len, n_images, names, name_off, n_nodes, node_image, node_feat, positions, held, nullptr);
  if (rc != LFR_OK) return rc;
  touch_components(n_nodes, node_comp, n_components, positions, held, n_held, n_touched, changed);
  return LFR_OK;
}

// The SolutionFiles of many scenes in one run (lfr_plan_update_solution_groups, lfr_wire_update_solution_groups):
// file g (files[g], file_len[g] bytes; NULL: no entries) is decoded and resolved against group g's image ids alone
// (group_of_image[id] < G), since scenes reuse image names, and the decodes are concatenated into `d` with every
// winning message keyed by its scene image id.  The keys of different groups differ, so one join of `d` gives every
// node its own scene's entry.  LFR_EINVAL, with *bad_group = g, when file g does not parse.
inline int decode_groups(uint32_t G, const uint8_t* const* files, const uint64_t* file_len, uint32_t n_images,
                         const uint8_t* names, const uint64_t* name_off, const uint32_t* group_of_image, Decoded& d,
                         uint32_t* bad_group = nullptr) {
  std::vector<uint32_t> start((size_t)G + 1, 0), ids(n_images);  // the ids of every group, ascending
  for (uint32_t k = 0; k < n_images; ++k) ++start[group_of_image[k] + 1];
  for (uint32_t g = 0; g < G; ++g) start[g + 1] += start[g];
  {
    std::vector<uint32_t> fill(start.begin(), start.end() - 1);
    for (uint32_t k = 0; k < n_images; ++k) ids[fill[group_of_image[k]]++] = k;
  }
  d = Decoded();
  d.img_ptr.assign(1, 0);
  std::vector<uint8_t> blob;
  std::vector<uint64_t> off;
  const uint8_t no_name = 0;
  for (uint32_t g = 0; g < G; ++g) {
    if (!files || !files[g]) continue;
    const uint32_t a = start[g], n = start[g + 1] - a;
    blob.clear();
    off.assign(1, 0);
    for (uint32_t j = 0; j < n; ++j) {
      const uint32_t k = ids[a + j];
      blob.insert(blob.end(), names + name_off[k], names + name_off[k + 1]);
      off.push_back(blob.size());
    }
    Decoded dg;
    if (decode(files[g], file_len[g], n, blob.empty() ? &no_name : blob.data(), off.data(), dg) != LFR_OK) {
      if (bad_group) *bad_group = g;
      return LFR_EINVAL;
    }
    if (!dg.canon.empty()) {  // names repeated within the group: each id joins through its group's lowest
      if (d.canon.empty()) {
        d.canon.resize(n_images);
        for (uint32_t k = 0; k < n_images; ++k) d.canon[k] = k;
      }
      for (uint32_t j = 0; j < n; ++j) d.canon[ids[a + j]] = ids[a + dg.canon[j]];
    }
    for (uint64_t i = 0; i < dg.n_images; ++i) {
      d.image_id.push_back(dg.image_id[i] == kNoImage ? kNoImage : ids[a + dg.image_id[i]]);
      d.img_ptr.push_back(d.n_disp + dg.img_ptr[i + 1]);
    }
    d.feature_idx.insert(d.feature_idx.end(), dg.feature_idx.begin(), dg.feature_idx.end());
    d.di.insert(d.di.end(), dg.di.begin(), dg.di.end());
    d.dj.insert(d.dj.end(), dg.dj.begin(), dg.dj.end());
    d.n_images += dg.n_images;
    d.n_disp += dg.n_disp;
  }
  return LFR_OK;
}

// The earlier run's image ids in this run's numbering, by exact name bytes (lfr_wire_update_solution_since,
// lfr_plan_update_solution_since): map[k] = the id of earlier name k among names / name_off, or, for a name
// this run does not have, n_images + (its rank among such names).  LFR_EINVAL for NULL or descending offsets
// and for a name repeated among the earlier names (it would give two earlier keypoints one key).
inline int map_previous_images(uint32_t n_images, const uint8_t* names, const uint64_t* name_off, uint32_t prev_n_images,
                               const uint8_t* prev_names, const uint64_t* prev_name_off, std::vector<uint32_t>& map) {
  if ((n_images && !name_off) || (prev_n_images && !prev_name_off)) return LFR_EINVAL;
  for (uint32_t k = 0; k < n_images; ++k)
    if (name_off[k + 1] < name_off[k]) return LFR_EINVAL;
  for (uint32_t k = 0; k < prev_n_images; ++k)
    if (prev_name_off[k + 1] < prev_name_off[k]) return LFR_EINVAL;
  if ((n_images && name_off[n_images] && !names) || (prev_n_images && prev_name_off[prev_n_images] && !prev_names))
    return LFR_EINVAL;
  std::unordered_map<std::string, uint32_t> id_of;
  id_of.reserve(n_images);
  for (uint32_t k = 0; k < n_images; ++k)
    id_of.emplace(std::string(reinterpret_cast<const char*>(names) + name_off[k], name_off[k + 1] - name_off[k]), k);
  std::unordered_map<std::string, uint32_t> seen;
  seen.reserve(prev_n_images);
  map.assign(prev_n_images, 0);
  uint32_t extra = 0;
  for (uint32_t k = 0; k < prev_n_images; ++k) {
    std::string s(reinterpret_cast<const char*>(prev_names) + prev_name_off[k], prev_name_off[k + 1] - prev_name_off[k]);
    if (!seen.emplace(s, k).second) return LFR_EINVAL;
    const auto it = id_of.find(s);
    map[k] = it != id_of.end() ? it->second : n_images + extra++;
  }
  return LFR_OK;
}

}  // namespace join
}  // namespace lfr

#endif  // LFR_JOIN_H_
