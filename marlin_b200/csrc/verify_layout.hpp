// The G2 side of a batch over several verifier keys (host only; tests/host/verify_layout_host_shim.cpp builds it for the CPU
// tests).  A key's G2 points are h, beta h and, for SonicKZG10, one beta^-(D - d) h per degree bound d.  Keys whose (h, beta h)
// bytes are equal form one group: their KZG checks fold into the same A (against h) and B (against beta h) MSMs and end in one
// pairing product per group.  Within a group every distinct SonicKZG10 point gets one slot of that product.
#pragma once
#include <cstdint>
#include <map>
#include <string>
#include <utility>
#include <vector>

namespace b2m {

struct G2Layout {
  std::vector<uint32_t> group;               // per key: its group
  std::vector<std::vector<uint32_t>> point;  // per key and key point (0: h, 1: beta h, 2 + b: bound b): its index in the call's set
  std::vector<uint32_t> group_of_point;      // per point of the call's set: the group it belongs to
  std::vector<std::pair<uint32_t, uint32_t>> src;  // per point of the call's set: the (key, key point) it is taken from
  size_t n_groups = 0;
};

// keys[k]: key k's points as consecutive `point_bytes`-byte encodings (h, beta h, bounds), and their count (at least 2).
// The call's set lists a new group's h and beta h when its first key is met, then each new SonicKZG10 point of the group when
// it is first met, in key order: the set of one key is its own points in order (when its bound points are distinct).
inline G2Layout g2_layout(const std::vector<std::pair<const uint8_t*, size_t>>& keys, size_t point_bytes) {
  G2Layout L;
  std::map<std::string, uint32_t> group_of_hb;        // h || beta h bytes -> group
  std::vector<std::map<std::string, uint32_t>> slot;  // per group: point bytes -> index in the call's set
  auto add = [&](uint32_t g, size_t k, size_t j) {
    L.group_of_point.push_back(g);
    L.src.push_back({(uint32_t)k, (uint32_t)j});
    return (uint32_t)L.src.size() - 1;
  };
  for (size_t k = 0; k < keys.size(); k++) {
    const uint8_t* p = keys[k].first;
    auto it = group_of_hb.find(std::string(reinterpret_cast<const char*>(p), 2 * point_bytes));
    if (it == group_of_hb.end()) {
      it = group_of_hb.emplace(std::string(reinterpret_cast<const char*>(p), 2 * point_bytes), (uint32_t)L.n_groups++).first;
      slot.emplace_back();
    }
    const uint32_t g = it->second;
    L.group.push_back(g);
    std::vector<uint32_t> pts;
    for (size_t j = 0; j < keys[k].second; j++) {
      // h and beta h are slots too, keyed apart from the bound points (a bound point may equal h when d = D)
      const std::string q = std::string(1, (char)(j < 2 ? j : 2)) + std::string(reinterpret_cast<const char*>(p + j * point_bytes), point_bytes);
      auto s = slot[g].find(q);
      if (s == slot[g].end()) s = slot[g].emplace(q, add(g, k, j)).first;
      pts.push_back(s->second);
    }
    L.point.push_back(std::move(pts));
  }
  return L;
}

}  // namespace b2m
