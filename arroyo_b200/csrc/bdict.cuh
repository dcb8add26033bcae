// The window aggregate's key dictionary: a *bucketed* open-addressing table.
//
//   bucket(key) = mulhi32(bd_hash(key) >> 32, n_buckets)           BD_KS 16-byte slots {key, idx} per bucket,
//   slot0(key)  = (key * odd constant) >> 53                linear probing that wraps inside the bucket
//   id(key)     = BD_ID_BASE + bucket * BD_CAPB + idx       idx = arrival order inside the bucket
//
// Why buckets: the two-pass ingest (ingest_two_pass.cuh) radix-partitions a launch's rows by bucket and aggregates
// each bucket in shared memory.  A bucket's slice of the dictionary is one contiguous 32 KB block (one coalesced load
// into shared memory), and a bucket's ids are one contiguous range of every pane array (the block's flush is a
// coalesced vector add instead of a scatter of REDs).  Keys recur from pane to pane, so after warm-up the
// dictionary is read-only; a bucket holds ~BD_MEAN keys (Poisson, sigma ~32: BD_CAPB is 8 sigma above the mean).
// The direct kernel (one probe + REDs per row) uses the same table through bd_resolve.
//
// When a bucket runs out of ids or the table outgrows its mean fill, the host doubles n_buckets and rebuilds
// (ids change; pane blocks are permuted with the old->new id map, window_agg.cu::grow_ids).
#pragma once

#include <climits>

#include "common.cuh"

namespace ab {

constexpr int BD_KS = 2048;        // slots per bucket (power of two)
constexpr int BD_CAPB = 1280;      // ids per bucket
constexpr int BD_MEAN = 1024;      // target keys per bucket when sizing n_buckets
constexpr uint32_t BD_ID_BASE = 2;  // id 0 = the key that equals the empty sentinel, id 1 unused (keeps bucket ranges 16-byte aligned)

struct alignas(16) BSlot {
  long long key;
  uint32_t idx;  // index inside the bucket
  uint32_t pad;
};

struct BDict {
  BSlot* slots;           // [n_buckets][BD_KS]
  unsigned int* nkeys;    // [n_buckets] ids handed out per bucket
  long long* id_keys;     // [id_cap] key of each id (emission)
  unsigned int* n_total;  // total keys (statistics, growth policy)
  uint32_t n_buckets;
  uint32_t pad;
};

// The bucket hash: one 64-bit multiply after folding the high half into the low one (every key bit reaches the high
// product bits that select the bucket).  The partition kernel evaluates it once per row; a three-multiply finaliser
// (splitmix64) measured as a fifth of that kernel's instructions.
__host__ __device__ __forceinline__ uint64_t bd_hash(long long key) {
  const uint64_t k = (uint64_t)key;
  return (k ^ (k >> 32)) * 0x9E3779B97F4A7C15ull;
}
__host__ __device__ __forceinline__ uint32_t bd_bucket(uint64_t h, uint32_t n_buckets) {
  return (uint32_t)(((h >> 32) * (uint64_t)n_buckets) >> 32);
}
// slot inside the bucket: a second, cheap hash of the key itself (one multiply), independent of the bits that chose
// the bucket -- the aggregation kernel computes only this one per row (its rows already sit in their bucket)
constexpr int BD_KS_LOG2 = 11;
static_assert((1 << BD_KS_LOG2) == BD_KS, "BD_KS_LOG2");
// Home slots are aligned to groups of BD_GROUP slots (one 64-byte line): a key sits in its home group unless the
// group overflowed, so a lookup is BD_GROUP straight-line compares (no divergent probe loop) and only the rare
// overflow walks on.
constexpr int BD_GROUP = 4;
__host__ __device__ __forceinline__ uint32_t bd_slot0(long long key) {
  return (uint32_t)(((uint64_t)key * 0xD6E8FEB86659FD93ull) >> (64 - BD_KS_LOG2)) & ~(uint32_t)(BD_GROUP - 1);
}
__host__ __device__ __forceinline__ uint32_t bd_id(uint32_t bucket, uint32_t idx) { return BD_ID_BASE + bucket * BD_CAPB + idx; }
inline uint64_t bd_id_cap(uint64_t n_buckets) { return ((BD_ID_BASE + n_buckets * BD_CAPB + 1023) / 1024) * 1024; }
inline uint64_t bd_buckets_for(uint64_t keys) {
  const uint64_t b = (keys + BD_MEAN - 1) / BD_MEAN;
  return b < 1 ? 1 : b;
}

static __global__ void bd_init_kernel(BSlot* slots, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    slots[i].key = EMPTY_KEY;
    slots[i].idx = ID_UNSET;
    slots[i].pad = 0;
  }
}

static __global__ void bd_fill_keys_kernel(long long* id_keys, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) id_keys[i] = EMPTY_KEY;  // "no key yet": readers of a bucket's id range skip these
}

__device__ __forceinline__ uint32_t bd_wait_idx(const BSlot* s) {
  uint32_t idx;
  do {
    __nanosleep(20);
    idx = *(volatile const uint32_t*)&s->idx;
  } while (idx == ID_UNSET);
  return idx;
}

// Lookup-or-insert in bucket `b`, starting at slot `s`.  Returns the id, or ID_OVERFLOW when the bucket is out of
// ids / slots (the caller defers the row; the host grows the dictionary).  Safe against concurrent inserts from any
// number of blocks: the slot is claimed with a CAS on the key, the index is published afterwards.
static __device__ __noinline__ uint32_t bd_insert(const BDict& d, uint32_t b, long long key, uint32_t s) {
  BSlot* tab = d.slots + (size_t)b * BD_KS;
#pragma unroll 1
  for (int probe = 0; probe < BD_KS; ++probe) {
    BSlot* sp = tab + s;
    const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(sp));
    long long k = (long long)raw.x;
    uint32_t idx = (uint32_t)raw.y;
    if (k == EMPTY_KEY) {
      const unsigned long long old =
          atomicCAS(reinterpret_cast<unsigned long long*>(&sp->key), (unsigned long long)EMPTY_KEY, (unsigned long long)key);
      if (old == (unsigned long long)EMPTY_KEY) {
        uint32_t nidx = atomicAdd(d.nkeys + b, 1u);
        if (nidx >= (uint32_t)BD_CAPB) {
          nidx = ID_OVERFLOW;  // the slot stays claimed for this key: every later row of the key overflows too
        } else {
          d.id_keys[bd_id(b, nidx)] = key;
          atomicAdd(d.n_total, 1u);
        }
        __threadfence();
        atomicExch(&sp->idx, nidx);
        return nidx == ID_OVERFLOW ? ID_OVERFLOW : bd_id(b, nidx);
      }
      k = (long long)old;
      idx = ID_UNSET;
    }
    if (k == key) {
      if (idx == ID_UNSET) idx = bd_wait_idx(sp);
      return idx >= ID_OVERFLOW ? ID_OVERFLOW : bd_id(b, idx);
    }
    s = (s + 1) & (BD_KS - 1);
  }
  return ID_OVERFLOW;
}

// Id of `key` given the contents of the first two slots of its home group (already loaded: the hot path issues those
// loads early; they share one 32-byte sector).  Known keys resolve with read-only probes inline; first sightings go
// out of line.
__device__ __forceinline__ uint32_t bd_resolve(const BDict& d, long long key, uint64_t h, unsigned long long k0,
                                               uint32_t idx0, unsigned long long k1, uint32_t idx1) {
  if (key == EMPTY_KEY) return 0;  // id 0 is reserved for the one key that equals the empty sentinel
  const uint32_t b = bd_bucket(h, d.n_buckets);
  if ((long long)k0 == key && idx0 < ID_OVERFLOW) return bd_id(b, idx0);
  if ((long long)k1 == key && idx1 < ID_OVERFLOW) return bd_id(b, idx1);
  uint32_t s = bd_slot0(key);
  if ((long long)k0 != EMPTY_KEY && (long long)k0 != key && (long long)k1 != EMPTY_KEY && (long long)k1 != key) {
    const BSlot* tab = d.slots + (size_t)b * BD_KS;
    s += 1;
#pragma unroll 1
    for (int probe = 2; probe < BD_KS; ++probe) {
      s = (s + 1) & (BD_KS - 1);
      const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(tab + s));
      if ((long long)raw.x == key && (uint32_t)raw.y < ID_OVERFLOW) return bd_id(b, (uint32_t)raw.y);
      if ((long long)raw.x == EMPTY_KEY || (long long)raw.x == key) break;
    }
  }
  return bd_insert(d, b, key, s);
}

__device__ __forceinline__ const BSlot* bd_home(const BDict& d, long long key, uint64_t h) {
  return d.slots + (size_t)bd_bucket(h, d.n_buckets) * BD_KS + bd_slot0(key);
}

// Id of `key`, inserting it on first sight (cold paths: restore, partial-state merge).
static __device__ __forceinline__ uint32_t bd_lookup_or_insert(const BDict& d, long long key) {
  if (key == EMPTY_KEY) return 0u;
  const uint64_t h = bd_hash(key);
  return bd_insert(d, bd_bucket(h, d.n_buckets), key, bd_slot0(key));
}

// Rebuild after growth: every key of the old dictionary gets an id in the new one; map[old id] = new id
// (ID_UNSET for ids that hold no key).
static __global__ void bd_rehash_kernel(BDict old_d, BDict new_d, uint32_t old_id_cap, uint32_t* map) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (; i < old_id_cap; i += stride) {
    uint32_t nid = ID_UNSET;
    if (i == 0) {
      nid = 0;
    } else if (i >= BD_ID_BASE) {
      const uint32_t b = (i - BD_ID_BASE) / BD_CAPB, idx = (i - BD_ID_BASE) % BD_CAPB;
      if (b < old_d.n_buckets && idx < min(old_d.nkeys[b], (unsigned)BD_CAPB)) nid = bd_lookup_or_insert(new_d, old_d.id_keys[i]);
    }
    map[i] = nid;
  }
}

}  // namespace ab
