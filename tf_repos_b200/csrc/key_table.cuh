// key_table.cuh -- the probe policy of the text pipelines' lock-free key tables (criteo_feature.cu,
// aliccp_sample.cu, smart_feature.cu).
//
// Open addressing without locks: every key word of a slot is set once, by a CAS from 0, and is final once non-zero.
// A key's walk starts at __umul64hi(hash, cap), probes linearly and wraps at cap; a key that finds no slot within
// min(cap, KT_MAX_PROBE) probes counts as dropped, and the host raises.  Every thread inserting one key takes the same
// decision at every slot it visits, so all of them end in the same slot.  Each table keeps its own layout, hash, slot
// comparison and what it does on a hit.
#pragma once
#include "common.cuh"

namespace ctr {

constexpr int64_t KT_MAX_PROBE = 1 << 15;           // a key that finds no slot within this many probes overflows
constexpr int64_t KT_MAX_CAP = (int64_t)1 << 31;    // slot numbers are uint32, sort positions int32

// the key word *p set to v if it is empty -> the value it now holds: v when the slot is (or has become) v's
__device__ __forceinline__ uint64_t claim(uint64_t* p, uint64_t v) {
  uint64_t k = *reinterpret_cast<volatile uint64_t*>(p);
  if (k == 0) {
    k = atomicCAS(reinterpret_cast<unsigned long long*>(p), 0ull, (unsigned long long)v);
    if (k == 0) k = v;
  }
  return k;
}

__device__ __forceinline__ uint32_t claim(uint32_t* p, uint32_t v) {
  uint32_t k = *reinterpret_cast<volatile uint32_t*>(p);
  if (k == 0) {
    k = atomicCAS(p, 0u, v);
    if (k == 0) k = v;
  }
  return k;
}

// the first slot of the walk of hash h over cap slots where hit(slot) holds; -1 = none within the probe limit
template <class Hit>
__device__ __forceinline__ int64_t probe(uint64_t h, int64_t cap, Hit&& hit) {
  uint64_t s = __umul64hi(h, (uint64_t)cap);
  const int64_t probes = cap < KT_MAX_PROBE ? cap : KT_MAX_PROBE;
  for (int64_t i = 0; i < probes; ++i) {
    if (hit(s)) return (int64_t)s;
    if (++s == (uint64_t)cap) s = 0;
  }
  return -1;
}

}  // namespace ctr
