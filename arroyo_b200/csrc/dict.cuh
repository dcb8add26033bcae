// The persistent key dictionary shared by the window-aggregate and session operators: open addressing with
// linear probing over 16-byte slots {key, dense id}.  Keys recur from pane to pane / session to session, so
// after warm-up a row costs one read-only 16-byte probe that hits L2; per-key state lives in dense arrays
// indexed by id.
#pragma once

#include <climits>
#include <cstdlib>

#include "common.cuh"

namespace ab {

#ifndef AB_ID_CONSTANTS
#define AB_ID_CONSTANTS
constexpr uint32_t ID_UNSET = 0xFFFFFFFFu;
constexpr uint32_t ID_OVERFLOW = 0xFFFFFFFEu;
constexpr long long EMPTY_KEY = LLONG_MIN;
#endif
constexpr int MAX_PROBE = 4096;

struct alignas(16) Slot {
  long long key;
  uint32_t id;
  uint32_t pad;
};

struct DictView {
  Slot* slots;
  long long* id_keys;
  unsigned int* n_keys;
  uint32_t cap;  // number of slots (any value: placement is multiply-shift, not a mask)
  uint32_t id_cap;
  // direct-mapped range: keys in [dbase, dbase + dn) own the ids [1, dn] without touching the slot array
  // (dense integer keys -- Nexmark's auction / bidder ids -- need no hashing at all); dn = 0 disables it
  long long dbase;
  uint32_t dn;
};

__device__ __forceinline__ bool dict_is_direct(const DictView& d, long long key) {
  return ((unsigned long long)key - (unsigned long long)d.dbase) < (unsigned long long)d.dn;
}

__host__ __device__ __forceinline__ uint32_t dict_home(uint64_t key, uint32_t cap) {
  return (uint32_t)(((mix64(key) >> 32) * (uint64_t)cap) >> 32);
}
__host__ __device__ __forceinline__ uint32_t dict_next(uint32_t pos, uint32_t cap) {
  return pos + 1 == cap ? 0u : pos + 1;
}

// -------------------------------------------------------------------------------------------
// dictionary
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t wait_id(const Slot* s) {
  uint32_t id;
  do {
    __nanosleep(20);
    id = *(volatile const uint32_t*)&s->id;
  } while (id == ID_UNSET);
  return id;
}

static __global__ void dict_init_kernel(Slot* slots, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    slots[i].key = EMPTY_KEY;
    slots[i].id = ID_UNSET;
    slots[i].pad = 0;
  }
}

// re-insert ids [first, n) after the slot array was replaced (ids below `first` are direct-mapped)
static __global__ void dict_rebuild_kernel(Slot* slots, uint32_t cap, const long long* id_keys, uint32_t n,
                                           uint32_t first) {
  uint32_t id = blockIdx.x * blockDim.x + threadIdx.x + first;
  uint32_t stride = gridDim.x * blockDim.x;
  for (; id < n; id += stride) {
    long long key = id_keys[id];
    uint32_t pos = dict_home((uint64_t)key, cap);
    while (true) {
      unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&slots[pos].key),
                                         (unsigned long long)EMPTY_KEY, (unsigned long long)key);
      if (old == (unsigned long long)EMPTY_KEY) {
        slots[pos].id = id;
        break;
      }
      pos = dict_next(pos, cap);
    }
  }
}

// First sighting of a key: claim the empty slot found at `pos` (or keep walking if somebody else took it).
static __device__ __noinline__ uint32_t dict_insert(const DictView& d, long long key, uint32_t pos) {
#pragma unroll 1
  for (int probe = 0; probe < MAX_PROBE; ++probe) {
    Slot* sp = d.slots + pos;
    ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(sp));
    long long k = (long long)raw.x;
    uint32_t id = (uint32_t)raw.y;
    if (k == key) {
      if (id == ID_UNSET) id = wait_id(sp);
      return id;
    }
    if (k == EMPTY_KEY) {
      unsigned long long old =
          atomicCAS(reinterpret_cast<unsigned long long*>(&sp->key), (unsigned long long)EMPTY_KEY, (unsigned long long)key);
      if (old == (unsigned long long)EMPTY_KEY) {
        uint32_t nid = atomicAdd(d.n_keys, 1u);
        if (nid >= d.id_cap) {
          nid = ID_OVERFLOW;
        } else {
          d.id_keys[nid] = key;
        }
        __threadfence();
        atomicExch(&sp->id, nid);
        return nid;
      }
      if ((long long)old == key) return wait_id(sp);
    }
    pos = dict_next(pos, d.cap);
  }
  return ID_OVERFLOW;
}

// Dense id of `key` given its home slot contents `raw` (already loaded).  Existing keys resolve with
// read-only probes inline; the insert path is out of line.
__device__ __forceinline__ uint32_t resolve_id(const DictView& d, long long key, unsigned long long k0, uint32_t id0) {
  if (dict_is_direct(d, key)) return (uint32_t)((unsigned long long)key - (unsigned long long)d.dbase) + 1u;
  if ((long long)k0 == key && id0 < ID_OVERFLOW) return id0;
  if (key == EMPTY_KEY) return 0;  // id 0 is reserved for the one key that equals the empty sentinel
  uint32_t pos = dict_home((uint64_t)key, d.cap);
  if ((long long)k0 == EMPTY_KEY || (long long)k0 == key) return dict_insert(d, key, pos);
#pragma unroll 1
  for (int probe = 1; probe < MAX_PROBE; ++probe) {
    pos = dict_next(pos, d.cap);
    const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(d.slots + pos));
    if ((long long)raw.x == key && (uint32_t)raw.y < ID_OVERFLOW) return (uint32_t)raw.y;
    if ((long long)raw.x == EMPTY_KEY || (long long)raw.x == key) return dict_insert(d, key, pos);
  }
  return ID_OVERFLOW;
}

// Id of `key`, inserting it on first sight (cold paths: restore, partial-state merge, sessions).
static __device__ __forceinline__ uint32_t dict_lookup_or_insert(const DictView& d, long long key) {
  if (dict_is_direct(d, key)) return (uint32_t)((unsigned long long)key - (unsigned long long)d.dbase) + 1u;
  if (key == EMPTY_KEY) return 0u;
  return dict_insert(d, key, dict_home((uint64_t)key, d.cap));
}

// slot count: 3.5 x ids => load factor 0.25 at the expected key count (0.29 when every id is used).
// The random 16-byte probe is faster at load 0.25 than at 0.5: shorter chains mean fewer divergent replays per
// warp.  ARROYO_B200_DICT_QUARTER_SLOTS_PER_ID
// (default 14 = 3.5 slots per id) trades chain length against L2 footprint for experiments.
inline uint64_t dict_slots_for(uint64_t ids) {
  static const uint64_t q = [] {
    const char* e = getenv("ARROYO_B200_DICT_QUARTER_SLOTS_PER_ID");
    uint64_t v = e ? strtoull(e, nullptr, 10) : 14;
    return v < 5 ? 5 : (v > 64 ? 64 : v);
  }();
  const uint64_t n = ids * q / 4;
  return n > 1024 ? n : 1024;
}

}  // namespace ab
