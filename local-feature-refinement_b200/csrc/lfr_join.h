// lfr_join.h — the host half of a start point read from a SolutionFile (types.proto:30-46), shared by the
// host join (lfr_wire_join_solution, lfr_wire.cc) and the device join (lfr_plan_start_from_solution,
// lfr_capi.cu): the decode with lfr_wire_decode_solution() and the image rule.  Header-only host code.
//
// The rule is that of the reference's own reader (reconstruction-scripts/colmap_utils.py:104-137): an
// Image message is matched to a scene image by its exact name bytes, and the last Image message with a
// given name wins as a whole; within it, the last displacement of a feature wins.  Each displacement of a
// winning message gets the key (image id << 32 | feature_idx), as the encoder keys its nodes; every other
// displacement gets kNoKey, which no node has (image ids are < 2^32 - 1).
#ifndef LFR_JOIN_H_
#define LFR_JOIN_H_

#include <cstdint>
#include <string>
#include <unordered_map>
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
  for (uint32_t k = 0; k < n_images; ++k)
    id_of.emplace(std::string(reinterpret_cast<const char*>(names) + name_off[k], name_off[k + 1] - name_off[k]), k);
  d.image_id.assign(I, kNoImage);
  std::vector<uint64_t> winner(n_images, ~0ull);  // last Image message of each scene image
  for (uint64_t i = 0; i < I; ++i) {
    const auto it = id_of.find(std::string(reinterpret_cast<const char*>(buf) + d.name_off[i], d.name_len[i]));
    if (it != id_of.end()) winner[it->second] = i;
  }
  for (uint32_t k = 0; k < n_images; ++k)
    if (winner[k] != ~0ull) d.image_id[winner[k]] = k;
  return LFR_OK;
}

}  // namespace join
}  // namespace lfr

#endif  // LFR_JOIN_H_
