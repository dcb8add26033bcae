// The key dictionary of the window and updating aggregates: a *bucketed* open-addressing table.
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
// The updating aggregate (updating_agg.cu) uses the same table for its dense ids, without the two-pass ingest.
//
// BucketDict, at the end of this file, is the host side both operators share: it owns the device buffers, and when a
// bucket runs out of ids or the table outgrows its mean fill it doubles n_buckets and rebuilds.  Ids change: each
// operator moves its own per-id state with the old->new id map (the window's pane blocks, the updating aggregate's
// accumulators).  BucketDict::place gives restored keys their ids before anything is merged; BucketDict::rebuild
// makes a fresh, smaller table from the keys of chosen ids (the updating aggregate gives back the ids of expired keys).
#pragma once

#include <algorithm>
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

// Restore: the id of every row's key, inserted on first sight; ID_OVERFLOW (counted in *overflow) when the key's
// bucket is out of ids.  keys == nullptr (an unkeyed plan): every row has id 0.
static __global__ void __launch_bounds__(256) bd_place_kernel(const BDict d, const long long* keys, long long n, uint32_t* ids,
                                                              unsigned long long* overflow) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const uint32_t id = keys ? bd_lookup_or_insert(d, keys[i]) : 0u;
    ids[i] = id;
    if (id >= ID_OVERFLOW) atomicAdd(overflow, 1ull);
  }
}

// Rebuild from a subset: the keys of the ids [BD_ID_BASE, n_ids) that hold a key and have keep[id] != 0, with their
// old ids, compacted with one atomic per warp.  Thread 0 also maps id 0 (the INT64_MIN key's) to itself.
static __global__ void __launch_bounds__(256) bd_gather_kernel(const long long* id_keys, const unsigned char* keep,
                                                               uint32_t n_ids, long long* keys, uint32_t* old_ids,
                                                               unsigned int* count, uint32_t* map) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t stride = gridDim.x * blockDim.x;
  const unsigned int lane = threadIdx.x & 31;
  if (i == 0) map[0] = 0;
  for (; i < n_ids; i += stride) {
    const bool mine = i >= BD_ID_BASE && keep[i] && id_keys[i] != EMPTY_KEY;
    const unsigned int active = __activemask();
    const unsigned int mask = __ballot_sync(active, mine);
    if (!mask) continue;
    const int leader = __ffs(active) - 1;
    unsigned int base = 0;
    if ((int)lane == leader) base = atomicAdd(count, (unsigned int)__popc(mask));
    base = __shfl_sync(active, base, leader);
    if (!mine) continue;
    const unsigned int o = base + __popc(mask & ((1u << lane) - 1u));
    keys[o] = id_keys[i];
    old_ids[o] = i;
  }
}
static __global__ void bd_map_kernel(const uint32_t* old_ids, const uint32_t* new_ids, unsigned int n, uint32_t* map) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; i < n; i += stride) map[old_ids[i]] = new_ids[i];
}

// What BucketDict::grow and ::rebuild hand back: map[old id] = new id (ID_UNSET: the id held no key, or a key that
// was not kept) for the old ids [0, old_ids), and the old id capacity (the stride of the caller's per-id arrays
// before the change).
struct BdGrowth {
  DevBuf map;
  uint32_t old_ids;
  uint64_t old_cap;
};

// The host side of one dictionary.  The key counter (BDict::n_total) stays where its operator reads it back with the
// rest of its bookkeeping; the owner only takes its address.  An unkeyed plan keeps one bucket's id range and no slots.
class BucketDict {
 public:
  // `launches` counts the kernels launched here (the operator's statistic)
  void init(cudaStream_t stream, int num_sms, bool keyed, unsigned int* n_total, uint64_t* launches) {
    stream_ = stream;
    num_sms_ = num_sms;
    keyed_ = keyed;
    n_total_ = n_total;
    launches_ = launches;
  }
  uint64_t n_buckets() const { return n_buckets_; }
  uint64_t id_cap() const { return id_cap_; }
  // the id range: every bucket's ids, used or not
  uint32_t n_ids() const { return (uint32_t)(BD_ID_BASE + n_buckets_ * BD_CAPB); }
  const long long* id_keys() const { return id_keys_.as<long long>(); }

  // A dictionary of `n_buckets` empty buckets.  Ids are 32-bit with two values reserved: refused at 2^31.
  void alloc(uint64_t n_buckets) {
    AB_REQUIRE(bd_id_cap(n_buckets) < (1ull << 31), ARROYO_B200_RUNTIME, "key dictionary too large");
    n_buckets_ = n_buckets;
    id_cap_ = bd_id_cap(n_buckets);
    id_keys_.alloc(id_cap_ * sizeof(long long));
    bd_fill_keys_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(id_keys_.as<long long>(), id_cap_);
    AB_CUDA(cudaGetLastError());
    nkeys_.alloc(n_buckets_ * sizeof(unsigned int));
    AB_CUDA(cudaMemsetAsync(nkeys_.p, 0, n_buckets_ * sizeof(unsigned int), stream_));
    if (keyed_) {
      slots_.alloc(n_buckets_ * BD_KS * sizeof(BSlot));
      bd_init_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(slots_.as<BSlot>(), n_buckets_ * BD_KS);
      AB_CUDA(cudaGetLastError());
    }
    *launches_ += keyed_ ? 2 : 1;
  }

  BDict view() const {
    BDict d{};
    d.slots = slots_.as<BSlot>();
    d.nkeys = nkeys_.as<unsigned int>();
    d.id_keys = id_keys_.as<long long>();
    d.n_total = n_total_;
    d.n_buckets = (uint32_t)n_buckets_;
    return d;
  }

  // Doubles the bucket count and re-inserts every key: ids change, the key counter is recounted.  A bucket's keys split
  // between the two buckets that replace it, so the rehash itself never runs out of ids.  Refused before anything
  // moves: the dictionary stays usable.  Returns with the stream drained.
  BdGrowth grow() {
    AB_REQUIRE(keyed_, ARROYO_B200_RUNTIME, "growth of an unkeyed dictionary");
    AB_REQUIRE(bd_id_cap(n_buckets_ * 2) < (1ull << 31), ARROYO_B200_RUNTIME, "key dictionary too large");
    BdGrowth g{DevBuf((size_t)id_cap_ * sizeof(uint32_t)), n_ids(), id_cap_};
    const BDict old_d = view();
    const DevBuf old_slots = std::move(slots_), old_nkeys = std::move(nkeys_), old_keys = std::move(id_keys_);
    AB_CUDA(cudaMemsetAsync(n_total_, 0, sizeof(unsigned int), stream_));
    alloc(n_buckets_ * 2);
    bd_rehash_kernel<<<grid(g.old_ids), 256, 0, stream_>>>(old_d, view(), g.old_ids, g.map.as<uint32_t>());
    AB_CUDA(cudaGetLastError());
    ++*launches_;
    AB_CUDA(cudaStreamSynchronize(stream_));  // the old buffers go when this returns
    return g;
  }

  // Gives each of `n` restored keys (device memory) its id, ids[i], before the caller merges anything.  When a bucket
  // runs out of ids, `grow_step()` -- grow() plus the move of the operator's own per-id state -- doubles the dictionary
  // and every row looks its key up again (a placed key keeps its place, under a new id).  A dictionary sized for few
  // rows has few buckets, each covering a wide hash range, so crowded keys may need several doublings to split: below
  // the default size (2^16 keys) it doubles freely; from there on, RESTORE_STALLS doublings in a row that place none
  // of the rest give up with RUNTIME.
  template <class GrowStep>
  void place(const long long* keys, long long n, uint32_t* ids, GrowStep grow_step) {
    constexpr int RESTORE_STALLS = 4;
    const uint64_t free_buckets = bd_buckets_for(1ull << 16);
    DevBuf overflow(sizeof(unsigned long long));
    for (uint64_t left = UINT64_MAX, stalls = 0;;) {
      AB_CUDA(cudaMemsetAsync(overflow.p, 0, sizeof(unsigned long long), stream_));
      bd_place_kernel<<<grid(n), 256, 0, stream_>>>(view(), keys, n, ids, overflow.as<unsigned long long>());
      AB_CUDA(cudaGetLastError());
      ++*launches_;
      unsigned long long over = 0;
      AB_CUDA(cudaMemcpyAsync(&over, overflow.p, sizeof over, cudaMemcpyDeviceToHost, stream_));
      AB_CUDA(cudaStreamSynchronize(stream_));
      if (over == 0) return;
      stalls = over < left || n_buckets_ < free_buckets ? 0 : stalls + 1;
      left = over;
      AB_REQUIRE(stalls < RESTORE_STALLS, ARROYO_B200_RUNTIME,
                 "restored keys whose dictionary bucket is out of ids still do not fit after the dictionary grew");
      grow_step();
    }
  }

  // A fresh dictionary holding only the keys of the ids with keep[id] != 0 (device, one byte per id of n_ids()), with
  // at least `min_buckets` buckets and room for the kept keys at the mean fill: what was handed out to keys that are
  // gone is reclaimed.  The kept keys are placed like restored ones (place, doubling when a bucket runs out of ids).
  // Id 0 maps to itself.  Returns with the stream drained.
  BdGrowth rebuild(const unsigned char* keep, uint64_t min_buckets) {
    AB_REQUIRE(keyed_, ARROYO_B200_RUNTIME, "rebuild of an unkeyed dictionary");
    BdGrowth g{DevBuf((size_t)id_cap_ * sizeof(uint32_t)), n_ids(), id_cap_};
    DevBuf keys((size_t)g.old_ids * sizeof(long long)), old_ids((size_t)g.old_ids * sizeof(uint32_t)),
        count(sizeof(unsigned int));
    AB_CUDA(cudaMemsetAsync(g.map.p, 0xFF, (size_t)id_cap_ * sizeof(uint32_t), stream_));  // ID_UNSET
    AB_CUDA(cudaMemsetAsync(count.p, 0, sizeof(unsigned int), stream_));
    bd_gather_kernel<<<grid(g.old_ids), 256, 0, stream_>>>(id_keys(), keep, g.old_ids, keys.as<long long>(),
                                                          old_ids.as<uint32_t>(), count.as<unsigned int>(),
                                                          g.map.as<uint32_t>());
    AB_CUDA(cudaGetLastError());
    ++*launches_;
    unsigned int n = 0;
    AB_CUDA(cudaMemcpyAsync(&n, count.p, sizeof n, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    AB_CUDA(cudaMemsetAsync(n_total_, 0, sizeof(unsigned int), stream_));
    alloc(std::max<uint64_t>(min_buckets, bd_buckets_for(n)));
    DevBuf new_ids((size_t)std::max(n, 1u) * sizeof(uint32_t));
    place(keys.as<long long>(), n, new_ids.as<uint32_t>(), [&] { grow(); });
    if (n) {
      bd_map_kernel<<<grid(n), 256, 0, stream_>>>(old_ids.as<uint32_t>(), new_ids.as<uint32_t>(), n, g.map.as<uint32_t>());
      AB_CUDA(cudaGetLastError());
      ++*launches_;
    }
    AB_CUDA(cudaStreamSynchronize(stream_));
    return g;
  }

 private:
  cudaStream_t stream_ = nullptr;
  int num_sms_ = 0;
  bool keyed_ = false;
  unsigned int* n_total_ = nullptr;
  uint64_t* launches_ = nullptr;
  uint64_t n_buckets_ = 0, id_cap_ = 0;
  DevBuf slots_, nkeys_, id_keys_;

  int grid(uint64_t items) const { return (int)std::max<uint64_t>(1, std::min<uint64_t>((items + 255) / 256, (uint64_t)num_sms_ * 8)); }
};

}  // namespace ab
