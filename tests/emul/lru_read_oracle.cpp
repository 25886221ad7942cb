// lru_read_oracle.cpp — the CPU oracle (oracle/mm_oracle.cpp, compiled whole into this library) plus the read side of its
// time-ordered weighted LRU.  TEST INFRASTRUCTURE ONLY (tests/lru_read_oracle.py builds and binds it).
//
//   orc_lru_read       orderedMap(false, MAX, usedSince) (CLHM:1226-1260): the deque walked from its tail, stopping at the
//                      first node with 0 < lastUsed < usedSince; usedSince <= 0 is descendingLruMap() (CLHM:1087-1116)
//   orc_lru_last_used  getLastUsedTime (CLHM:742-746): -1 when absent or lastUsed <= 0
//   orc_lru_weight     getWeight (CLHM:768-771): -1 when absent
//   orc_sim_lru_read   orc_lru_read of one cache of the closed loop, with each copy's registration time (loadTs, -1 if absent)
//
// The walk follows the linked deque literally; it does not use the (ts, seq) derivation the device kernels use.
#include "../../oracle/mm_oracle.cpp"

namespace {
// CLHM:1239-1250: descendingIterator, the break rule, map.put
int64_t lru_read_walk(const Lru &l, int64_t used_since, int32_t *keys, int64_t *last_used, int64_t *weights,
                      const std::unordered_map<int32_t, int64_t> *load_ts_of, int64_t *load_ts, int64_t cap) {
  int64_t n = 0;
  for (auto it = l.deque.rbegin(); it != l.deque.rend(); ++it) {
    const int64_t lastUsed = it->lastUsed;
    if (lastUsed > 0 && lastUsed < used_since) break;
    if (n < cap) {
      keys[n] = it->key; last_used[n] = lastUsed; weights[n] = it->weight;
      if (load_ts) {
        auto f = load_ts_of->find(it->key);
        load_ts[n] = f != load_ts_of->end() ? f->second : -1;
      }
    }
    n++;
  }
  return n;
}
}  // namespace

extern "C" {

int64_t orc_lru_read(orc_lru *l, int64_t used_since, int32_t *keys, int64_t *last_used, int64_t *weights, int64_t cap) {
  return lru_read_walk(l->l, used_since, keys, last_used, weights, nullptr, nullptr, cap);
}
int64_t orc_lru_last_used(orc_lru *l, int32_t key) {
  auto it = l->l.data.find(key);
  const int64_t lut = it == l->l.data.end() ? -1 : it->second->lastUsed;
  return lut <= 0 ? -1 : lut;
}
int64_t orc_lru_weight(orc_lru *l, int32_t key) {
  auto it = l->l.data.find(key);
  return it == l->l.data.end() ? -1 : it->second->weight;
}
int64_t orc_sim_lru_read(orc_sim *s, int32_t instance, int64_t used_since, int32_t *keys, int64_t *last_used, int64_t *weights,
                         int64_t *load_ts, int64_t cap) {
  if (!s || instance < 0 || (size_t)instance >= s->lru.size()) return -1;
  return lru_read_walk(*s->lru[instance], used_since, keys, last_used, weights, &s->loadTs[instance], load_ts, cap);
}

}  // extern "C"
