// Host build of the cross-key batch's G2 grouping (marlin_b200/csrc/verify_layout.hpp) over a tiny C ABI for
// tests/test_verify_layout_host.py.
#include "../../marlin_b200/csrc/verify_layout.hpp"

#include <cstddef>
using namespace b2m;

// keys[k]: counts[k] points of point_bytes bytes.  Out: group[k]; point[]: every key's point indices, key after key;
// group_of_point[] and src_key[] / src_point[] for the call's set (at most sum(counts) entries).  Returns the group count and
// the call's point count in *n_points.
extern "C" size_t g2_layout_host(size_t n_keys, const uint8_t* const* keys, const size_t* counts, size_t point_bytes, uint32_t* group,
                                 uint32_t* point, uint32_t* group_of_point, uint32_t* src_key, uint32_t* src_point, size_t* n_points) {
  std::vector<std::pair<const uint8_t*, size_t>> in;
  for (size_t k = 0; k < n_keys; k++) in.push_back({keys[k], counts[k]});
  const G2Layout L = g2_layout(in, point_bytes);
  size_t o = 0;
  for (size_t k = 0; k < n_keys; k++) {
    group[k] = L.group[k];
    for (uint32_t q : L.point[k]) point[o++] = q;
  }
  for (size_t i = 0; i < L.src.size(); i++) {
    group_of_point[i] = L.group_of_point[i];
    src_key[i] = L.src[i].first;
    src_point[i] = L.src[i].second;
  }
  *n_points = L.src.size();
  return L.n_groups;
}
