// The persistent key dictionary of the session operator: open addressing with linear probing over 16-byte slots
// {key, dense id}.  Keys recur from session to session, so after warm-up a row costs one read-only 16-byte probe that
// hits L2; per-key state lives in dense arrays indexed by id.
#pragma once

#include "common.cuh"

namespace ab {

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
};

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

// re-insert ids [first, n) after the slot array was replaced (id 0, the INT64_MIN key's, has no slot)
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

// First sighting of a key: claim the empty slot found at `pos` (or keep walking if somebody else took it).  The walk
// may visit every slot: the table is kept below 0.3 load (dict_slots_for), so it always ends at the key or at an empty
// slot, however long the key's chain is.  ID_OVERFLOW: the ids are used up, or (never, below full) no slot was found.
static __device__ __noinline__ uint32_t dict_insert(const DictView& d, long long key, uint32_t pos) {
#pragma unroll 1
  for (uint32_t probe = 0; probe < d.cap; ++probe) {
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

// slot count: 3.5 x ids => load factor 0.25 at the expected key count (0.29 when every id is used).
// The random 16-byte probe is faster at load 0.25 than at 0.5: shorter chains mean fewer divergent replays per
// warp.
inline uint64_t dict_slots_for(uint64_t ids) {
  const uint64_t n = ids * 14 / 4;
  return n > 1024 ? n : 1024;
}

}  // namespace ab
