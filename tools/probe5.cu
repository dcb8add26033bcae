// probe5: (1) SM-side cost of the primitives a shared-memory aggregation could be built from, and
//         (2) a standalone prototype of the two-pass ingest: radix partition by dictionary bucket with
//             shared-memory write-combining -> per-bucket aggregation in warp-private shared-memory tables
//             fed by cp.async.bulk (TMA) + mbarrier rings.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -o tools/bin/probe5 tools/probe5.cu
// Run:   tools/bin/probe5 [rows_log2=23] [keys_log2=20] [hot=0]
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define CK(x)                                                                               \
  do {                                                                                      \
    cudaError_t e_ = (x);                                                                   \
    if (e_ != cudaSuccess) {                                                                \
      fprintf(stderr, "CUDA %s at %s:%d: %s\n", cudaGetErrorName(e_), __FILE__, __LINE__, #x); \
      exit(1);                                                                              \
    }                                                                                       \
  } while (0)

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// ------------------------------------------------------------------------------------------------
// (1) primitive micro-benchmarks: cycles per warp-instruction at nw warps per SM
// ------------------------------------------------------------------------------------------------
constexpr int MB_ITERS = 2048;

__global__ void mb_match32(unsigned* out, unsigned seed) {
  unsigned x = (threadIdx.x * 2654435761u) ^ seed, acc = 0;
  for (int i = 0; i < MB_ITERS; ++i) {
    x = x * 1664525u + 1013904223u;
    acc += __match_any_sync(0xffffffffu, x >> 22);  // 1024 values
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}
__global__ void mb_match64(unsigned* out, unsigned seed) {
  unsigned x = (threadIdx.x * 2654435761u) ^ seed, acc = 0;
  for (int i = 0; i < MB_ITERS; ++i) {
    x = x * 1664525u + 1013904223u;
    acc += __match_any_sync(0xffffffffu, ((unsigned long long)x << 20) | (x >> 12));
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}
__global__ void mb_alu_only(unsigned* out, unsigned seed) {
  unsigned x = (threadIdx.x * 2654435761u) ^ seed, acc = 0;
  for (int i = 0; i < MB_ITERS; ++i) {
    x = x * 1664525u + 1013904223u;
    acc += x >> 22;
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}
// shared atomics, spread addresses over `span` words
template <int MODE>  // 0 = atomicAdd u32 no return, 1 = atomicAdd u32 with return, 2 = atomicAdd u64 (CAS loop), 3 = plain LDS+STS u64 RMW, 4 = plain LDS u64 only, 5 = LDS.128 only
__global__ void mb_smem(unsigned* out, unsigned seed, unsigned span) {
  extern __shared__ unsigned long long sm64[];
  unsigned* sm32 = reinterpret_cast<unsigned*>(sm64);
  for (unsigned i = threadIdx.x; i < span * 2; i += blockDim.x) sm32[i] = 0;
  __syncthreads();
  unsigned x = (threadIdx.x * 2654435761u) ^ seed, acc = 0;
  for (int i = 0; i < MB_ITERS; ++i) {
    x = x * 1664525u + 1013904223u;
    const unsigned a = (x >> 8) % span;
    if (MODE == 0) atomicAdd(&sm32[a], 1u);
    if (MODE == 1) acc += atomicAdd(&sm32[a], 1u);
    if (MODE == 2) atomicAdd(&sm64[a], (unsigned long long)x);
    if (MODE == 3) {
      unsigned long long v = sm64[a];
      sm64[a] = v + x;
    }
    if (MODE == 4) acc += (unsigned)sm64[a];
    if (MODE == 5) {
      const ulonglong2 v = reinterpret_cast<const ulonglong2*>(sm64)[a >> 1];
      acc += (unsigned)(v.x + v.y);
    }
  }
  __syncthreads();
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc + sm32[threadIdx.x % (span * 2)];
}

template <class F>
float time_ms(F f, int reps = 5) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  f();
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    CK(cudaEventRecord(a));
    f();
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms;
    CK(cudaEventElapsedTime(&ms, a, b));
    best = std::min(best, ms);
  }
  CK(cudaEventDestroy(a));
  CK(cudaEventDestroy(b));
  return best;
}

void run_micro(int sms, double ghz) {
  unsigned* out;
  CK(cudaMalloc(&out, sizeof(unsigned) * sms * 1024));
  printf("---- primitives: SM-cycles per warp instruction (chip-wide, %d SMs, %.2f GHz assumed) ----\n", sms, ghz);
  for (int threads : {256, 512, 1024}) {
    auto report = [&](const char* name, float ms, float base_ms) {
      const double warp_instr_per_sm = (double)MB_ITERS * (threads / 32);
      const double cyc = (ms - base_ms) * 1e-3 * ghz * 1e9 / warp_instr_per_sm;
      printf("%-44s thr=%4d  %8.3f ms  %6.2f cyc/warp-instr  (%5.2f cyc/lane)\n", name, threads, ms, cyc, cyc / 32);
    };
    float base = time_ms([&] { mb_alu_only<<<sms, threads>>>(out, 1); });
    report("alu only (baseline, subtracted below)", base, 0);
    report("MATCH.ANY.U32 (1024 values)", time_ms([&] { mb_match32<<<sms, threads>>>(out, 1); }), base);
    report("MATCH.ANY.U64", time_ms([&] { mb_match64<<<sms, threads>>>(out, 1); }), base);
    const unsigned span = 4096;
    const size_t sh = span * 8;
    report("ATOMS.ADD.32 no return, spread 4096", time_ms([&] { mb_smem<0><<<sms, threads, sh>>>(out, 1, span); }), base);
    report("ATOMS.ADD.32 with return, spread 4096", time_ms([&] { mb_smem<1><<<sms, threads, sh>>>(out, 1, span); }), base);
    report("atomicAdd u64 shared (CAS loop), spread", time_ms([&] { mb_smem<2><<<sms, threads, sh>>>(out, 1, span); }), base);
    report("plain LDS.64 + STS.64 RMW, random", time_ms([&] { mb_smem<3><<<sms, threads, sh>>>(out, 1, span); }), base);
    report("plain LDS.64 random", time_ms([&] { mb_smem<4><<<sms, threads, sh>>>(out, 1, span); }), base);
    report("plain LDS.128 random", time_ms([&] { mb_smem<5><<<sms, threads, sh>>>(out, 1, span); }), base);
  }
  CK(cudaFree(out));
}

// ------------------------------------------------------------------------------------------------
// (2) two-pass prototype
// ------------------------------------------------------------------------------------------------
struct alignas(16) Rec {
  long long key;
  long long val;
};
struct alignas(16) KSlot {
  long long key;
  uint32_t idx;
  uint32_t pad;
};
constexpr long long EMPTY_KEY = LLONG_MIN;
constexpr uint32_t IDX_UNSET = 0xFFFFFFFFu;
__device__ unsigned long long g_trap_code;

// bucketed dictionary: B buckets x KS slots (global), ids = b * CAPB + idx
constexpr int KS = 2048;
constexpr int CAPB = 1280;

struct BDict {
  KSlot* slots;       // [B][KS]
  unsigned* nkeys;    // [B]
  long long* id_keys; // [B * CAPB]
  int log2b;
};

__device__ __forceinline__ uint32_t bucket_of(uint64_t h, int log2b) { return (uint32_t)(h >> (64 - log2b)); }
__device__ __forceinline__ uint32_t slot_of(uint64_t h) { return (uint32_t)h & (KS - 1); }

// global lookup-or-insert; returns idx within the bucket (or IDX_UNSET on overflow)
__device__ __noinline__ uint32_t bdict_insert(const BDict& d, uint32_t b, long long key, uint32_t s) {
  KSlot* tab = d.slots + (size_t)b * KS;
  for (int probe = 0; probe < KS; ++probe) {
    KSlot* sp = tab + s;
    const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(sp));
    long long k = (long long)raw.x;
    uint32_t idx = (uint32_t)raw.y;
    if (k == EMPTY_KEY) {
      unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&sp->key), (unsigned long long)EMPTY_KEY,
                                         (unsigned long long)key);
      if (old == (unsigned long long)EMPTY_KEY) {
        uint32_t nid = atomicAdd(d.nkeys + b, 1u);
        if (nid >= CAPB) nid = IDX_UNSET - 1;
        else d.id_keys[(size_t)b * CAPB + nid] = key;
        __threadfence();
        atomicExch(&sp->idx, nid);
        return nid;
      }
      k = (long long)old;
      idx = IDX_UNSET;
    }
    if (k == key) {
      for (long long spin = 0; idx == IDX_UNSET; ++spin) {
        __nanosleep(20);
        idx = *(volatile uint32_t*)&sp->idx;
        if (spin > (1ll << 22)) {
          g_trap_code = 0x1D2ull;
          __threadfence_system();
          __trap();
        }
      }
      return idx;
    }
    s = (s + 1) & (KS - 1);
  }
  return IDX_UNSET - 1;
}

__global__ void bdict_init(KSlot* slots, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i < n; i += (size_t)gridDim.x * blockDim.x) {
    slots[i].key = EMPTY_KEY;
    slots[i].idx = IDX_UNSET;
    slots[i].pad = 0;
  }
}

// ---------------- pass 1: partition ----------------
struct Part1Params {
  const long long* key;
  const long long* val;
  const long long* ts;
  long long n;
  int log2b;
  unsigned long long slide_magic;  // stand-in for the pane assignment arithmetic
  long long q0;
  Rec* out;            // [NR][cap]
  unsigned* cursor;    // [NR]
  unsigned cap;        // rows per region
  unsigned long long* overflow;  // counter
};

template <int THREADS, int RPT, int NR_MAX>
__global__ void __launch_bounds__(THREADS, 1) part1_kernel(const __grid_constant__ Part1Params p) {
  constexpr int TILE = THREADS * RPT;
  constexpr int NWARP = THREADS / 32;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Rec* reorder = reinterpret_cast<Rec*>(smem_raw);                                  // TILE x 16
  uint16_t* rid = reinterpret_cast<uint16_t*>(smem_raw + (size_t)TILE * 16);        // TILE x 2
  uint16_t* wh = rid + TILE;                                                        // NWARP x NR_MAX x 2
  uint32_t* toff = reinterpret_cast<uint32_t*>(wh + (size_t)NWARP * NR_MAX);        // NR_MAX
  uint32_t* gdelta = toff + NR_MAX;                                                 // NR_MAX  (global pos - tile offset)
  __shared__ uint32_t s_wsum[NWARP];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int NR = 1 << p.log2b;
  const unsigned lt = (1u << lane) - 1u;
  const long long n_tiles = (p.n + TILE - 1) / TILE;
  uint16_t* mywh = wh + (size_t)w * NR_MAX;

  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = tile * TILE;
    const int cnt = (int)min((long long)TILE, p.n - base);
    // zero the warp-private histograms
    for (int i = tid; i < NWARP * NR_MAX / 2; i += THREADS) reinterpret_cast<uint32_t*>(wh)[i] = 0;
    long long k[RPT], v[RPT];
    uint32_t rr[RPT];  // region | rank << 16
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const int i = j * THREADS + tid;
      k[j] = 0;
      v[j] = 0;
      long long t = 0;
      if (i < cnt) {
        k[j] = __ldcs(p.key + base + i);
        v[j] = __ldcs(p.val + base + i);
        t = __ldcs(p.ts + base + i);
      }
      const uint64_t q = __umul64hi((uint64_t)t, p.slide_magic);
      const bool on = i < cnt && (long long)q >= p.q0;
      rr[j] = on ? bucket_of(mix64((uint64_t)k[j]), p.log2b) : 0xFFFFu;
    }
    __syncthreads();
    // rank inside the warp-private histogram (no atomics: one leader per distinct region per step)
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const uint32_t r = rr[j];
      const unsigned peers = __match_any_sync(0xffffffffu, r);
      const int lead = __ffs(peers) - 1;
      unsigned old = 0;
      if (lane == lead && r != 0xFFFFu) {
        old = mywh[r];
        mywh[r] = (uint16_t)(old + __popc(peers));
      }
      old = __shfl_sync(0xffffffffu, old, lead);
      rr[j] = r | ((old + __popc(peers & lt)) << 16);
    }
    __syncthreads();
    // per region: exclusive prefix over the warps; thread t owns regions 2t, 2t+1 (one 32-bit word per warp row)
    uint32_t c0 = 0, c1 = 0;
    if (2 * tid < NR) {
#pragma unroll 4
      for (int ww = 0; ww < NWARP; ++ww) {
        uint32_t* cell = reinterpret_cast<uint32_t*>(wh + (size_t)ww * NR_MAX) + tid;
        const uint32_t x = *cell;
        *cell = (c0 & 0xFFFFu) | (c1 << 16);
        c0 += x & 0xFFFFu;
        c1 += x >> 16;
      }
    }
    // block exclusive scan of the per-region tile counts
    uint32_t tsum = c0 + c1, incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) s_wsum[w] = incl;
    __syncthreads();
    uint32_t wbase = 0;
    for (int ww = 0; ww < w; ++ww) wbase += s_wsum[ww];
    const uint32_t ex = wbase + incl - tsum;
    if (2 * tid < NR) {
      toff[2 * tid] = ex;
      toff[2 * tid + 1] = ex + c0;
      uint32_t g0 = 0, g1 = 0;
      if (c0) g0 = atomicAdd(p.cursor + 2 * tid, c0);
      if (c1) g1 = atomicAdd(p.cursor + 2 * tid + 1, c1);
      gdelta[2 * tid] = g0 - ex;
      gdelta[2 * tid + 1] = g1 - (ex + c0);
    }
    __syncthreads();
    // scatter into the tile's reorder buffer
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const uint32_t r = rr[j] & 0xFFFFu;
      if (r != 0xFFFFu) {
        const uint32_t pos = toff[r] + wh[(size_t)w * NR_MAX + r] + (rr[j] >> 16);
        reorder[pos] = Rec{k[j], v[j]};
        rid[pos] = (uint16_t)r;
      }
    }
    __syncthreads();
    const uint32_t total = wbase;  // not the tile total; recompute
    (void)total;
    uint32_t n_on = 0;
    for (int ww = 0; ww < NWARP; ++ww) n_on += s_wsum[ww];
    for (uint32_t i = tid; i < n_on; i += THREADS) {
      const Rec rec = reorder[i];
      const uint32_t r = rid[i];
      const uint32_t dst = gdelta[r] + i;
      if (dst < p.cap) p.out[(size_t)r * p.cap + dst] = rec;
      else atomicAdd(p.overflow, 1ull);
    }
    __syncthreads();
  }
}

// ---------------- pass 2: aggregate one region per CTA in warp-private tables ----------------
struct Agg2Params {
  const Rec* in;       // [NR][cap]
  const unsigned* cursor;
  unsigned cap;
  BDict dict;
  unsigned long long* pane_rows;  // [B * CAPB]
  unsigned long long* pane_sum;   // [B * CAPB]
  unsigned long long* misses;     // rows that took the global insert path
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  for (long long spin = 0; !mbar_try(bar, parity); ++spin) {
    if (spin > (1ll << 24)) {  // a second or so: the copy never completed
      g_trap_code = 0xBA2ull;
      __threadfence_system();
      __trap();
    }
  }
}

template <int NW, int NST, int CH>
__global__ void __launch_bounds__(NW * 32, 1) agg2_kernel(const __grid_constant__ Agg2Params p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  KSlot* ktab = reinterpret_cast<KSlot*>(smem_raw);                                          // KS x 16
  unsigned long long* ssum = reinterpret_cast<unsigned long long*>(smem_raw + (size_t)KS * 16);  // NW x CAPB x 8
  uint32_t* scnt = reinterpret_cast<uint32_t*>(ssum + (size_t)NW * CAPB);                     // NW x CAPB x 4
  Rec* ring = reinterpret_cast<Rec*>(scnt + (size_t)NW * CAPB);                               // NW x NST x CH x 16
  unsigned long long* bars = reinterpret_cast<unsigned long long*>(ring + (size_t)NW * NST * CH);  // NW x NST
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int B = 1 << p.dict.log2b;
  unsigned long long* mysum = ssum + (size_t)w * CAPB;
  uint32_t* mycnt = scnt + (size_t)w * CAPB;
  Rec* myring = ring + (size_t)w * NST * CH;
  const uint32_t bar0 = smem_u32(bars + (size_t)w * NST);
  if (lane == 0)
    for (int s = 0; s < NST; ++s) mbar_init(bar0 + 8 * s, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  uint32_t phase = 0;  // bit s = parity of stage s
  unsigned long long miss = 0;

  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const unsigned n = min(p.cursor[b], p.cap);
    // dictionary slice -> shared, private tables zeroed
    {
      const ulonglong2* src = reinterpret_cast<const ulonglong2*>(p.dict.slots + (size_t)b * KS);
      ulonglong2* dst = reinterpret_cast<ulonglong2*>(ktab);
      for (int i = tid; i < KS; i += NW * 32) dst[i] = __ldcg(src + i);
      for (int i = tid; i < NW * CAPB; i += NW * 32) {
        ssum[i] = 0;
        scnt[i] = 0;
      }
    }
    __syncthreads();
    const Rec* rows = p.in + (size_t)b * p.cap;
    const unsigned n_chunks = (n + CH - 1) / CH;
    // this warp's chunks: w, w + NW, ...
    const unsigned my_chunks = n_chunks > (unsigned)w ? (n_chunks - w + NW - 1) / NW : 0;
    auto issue = [&](unsigned ci, int s) {
      const unsigned c = w + ci * NW;
      const unsigned r0 = c * CH;
      const unsigned nr = min((unsigned)CH, n - r0);
      if (lane == 0) {
        mbar_expect_tx(bar0 + 8 * s, nr * 16);
        tma_load_1d(smem_u32(myring + (size_t)s * CH), rows + r0, nr * 16, bar0 + 8 * s);
      }
    };
    for (unsigned ci = 0; ci < (unsigned)NST && ci < my_chunks; ++ci) issue(ci, (int)ci);
    for (unsigned ci = 0; ci < my_chunks; ++ci) {
      const int s = (int)(ci % NST);
      mbar_wait(bar0 + 8 * s, (phase >> s) & 1u);
      phase ^= 1u << s;
      const unsigned c = w + ci * NW;
      const unsigned nr = min((unsigned)CH, n - c * CH);
      const Rec* chunk = myring + (size_t)s * CH;
#pragma unroll
      for (int sub = 0; sub < CH / 32; ++sub) {
        const unsigned ri = sub * 32 + lane;
        const bool valid = ri < nr;
        Rec rec{0, 0};
        if (valid) rec = chunk[ri];
        // probe the shared dictionary slice
        uint32_t idx = IDX_UNSET;
        if (valid) {
          const uint64_t h = mix64((uint64_t)rec.key);
          uint32_t sl = slot_of(h);
          for (int probe = 0; probe < KS; ++probe) {
            const ulonglong2 e = *reinterpret_cast<const ulonglong2*>(ktab + sl);
            if ((long long)e.x == rec.key && (uint32_t)e.y != IDX_UNSET) {
              idx = (uint32_t)e.y;
              break;
            }
            if ((long long)e.x == EMPTY_KEY || (long long)e.x == rec.key) {
              // first sight in this slice: global insert (race-free across CTAs), then publish locally
              idx = bdict_insert(p.dict, (uint32_t)b, rec.key, slot_of(h));
              ++miss;
              if ((long long)e.x == EMPTY_KEY) {
                unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(&ktab[sl].key),
                                                   (unsigned long long)EMPTY_KEY, (unsigned long long)rec.key);
                if (old == (unsigned long long)EMPTY_KEY) *(volatile uint32_t*)&ktab[sl].idx = idx;
              }
              break;
            }
            sl = (sl + 1) & (KS - 1);
          }
        }
        const bool ok = valid && idx < (uint32_t)CAPB;
        // intra-warp duplicates: combine onto the first lane of each group, then one plain RMW per group
        const uint32_t gk = ok ? idx : (0x80000000u | (uint32_t)lane);
        const unsigned peers = __match_any_sync(0xffffffffu, gk);
        unsigned long long sv = (unsigned long long)rec.val;
        uint32_t cv = 1;
        if (__any_sync(0xffffffffu, peers & (peers - 1))) {
          unsigned long long acc = 0;
          for (unsigned m = peers; m; m &= m - 1) acc += __shfl_sync(peers, sv, __ffs(m) - 1);  // mask = the group: trip counts differ between groups
          sv = acc;
          cv = __popc(peers);
        }
        if (ok && (__ffs(peers) - 1) == lane) {
          mysum[idx] += sv;
          mycnt[idx] += cv;
        }
      }
      __syncwarp();
      if (ci + NST < my_chunks) issue(ci + NST, s);
    }
    __syncthreads();
    // reduce the NW private tables and add into the pane block (this CTA owns the bucket's ids in this launch)
    const unsigned nk = min(*(volatile unsigned*)(p.dict.nkeys + b), (unsigned)CAPB);
    for (unsigned i = tid; i < nk; i += NW * 32) {
      unsigned long long s = 0;
      uint32_t c = 0;
#pragma unroll
      for (int ww = 0; ww < NW; ++ww) {
        s += ssum[(size_t)ww * CAPB + i];
        c += scnt[(size_t)ww * CAPB + i];
      }
      if (c) {
        const size_t id = (size_t)b * CAPB + i;
        p.pane_rows[id] += c;
        p.pane_sum[id] += s;
      }
    }
    __syncthreads();
  }
  if (miss) atomicAdd(p.misses, miss);
}

// smallest possible TMA round trip: one warp, one bulk copy, one mbarrier
__global__ void tma_selftest(const Rec* src, Rec* dst, int n) {
  __shared__ __align__(128) Rec buf[64];
  __shared__ __align__(8) unsigned long long bar;
  const uint32_t b = smem_u32(&bar);
  if (threadIdx.x == 0) mbar_init(b, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(b, n * 16);
    tma_load_1d(smem_u32(buf), src, n * 16, b);
  }
  mbar_wait(b, 0);
  if ((int)threadIdx.x < n) dst[threadIdx.x] = buf[threadIdx.x];
}

// reference: direct global atomics through the same dictionary
__global__ void direct_kernel(const long long* key, const long long* val, long long n, BDict d, unsigned long long* rows,
                              unsigned long long* sum) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long k = key[i];
    const uint64_t h = mix64((uint64_t)k);
    const uint32_t b = bucket_of(h, d.log2b);
    const uint32_t idx = bdict_insert(d, b, k, slot_of(h));
    if (idx < (uint32_t)CAPB) {
      atomicAdd(rows + (size_t)b * CAPB + idx, 1ull);
      atomicAdd(sum + (size_t)b * CAPB + idx, (unsigned long long)val[i]);
    }
  }
}

__global__ void gen_kernel(long long* key, long long* val, long long* ts, long long n, unsigned long long n_keys, int hot,
                           unsigned long long seed) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint64_t r = mix64((uint64_t)i * 0x9E3779B97F4A7C15ull + seed);
    uint64_t kid = r % n_keys;
    if (hot && (mix64(r) & 3) != 0) kid = 7;
    key[i] = (long long)(kid * 0x9E3779B97F4A7C15ull);
    val[i] = (long long)((r >> 40) % 100000000ull) + 100;
    ts[i] = 1700000000000000000ll + i * 59;
  }
}

int main(int argc, char** argv) {
  setvbuf(stdout, nullptr, _IOLBF, 0);
  const int rows_log2 = argc > 1 ? atoi(argv[1]) : 23;
  const int keys_log2 = argc > 2 ? atoi(argv[2]) : 20;
  const int hot = argc > 3 ? atoi(argv[3]) : 0;
  const char* mode = argc > 4 ? argv[4] : "all";  // micro | tma | p1 | p2 | all
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  const double ghz = prop.clockRate * 1e-6;
  printf("device %s, %d SMs, %.3f GHz, mode %s\n", prop.name, sms, ghz, mode);
  auto is = [&](const char* m) { return !strcmp(mode, m) || !strcmp(mode, "all"); };
  if (is("micro")) run_micro(sms, ghz);
  if (is("tma")) {
    Rec *a, *b;
    CK(cudaMalloc(&a, 64 * sizeof(Rec)));
    CK(cudaMalloc(&b, 64 * sizeof(Rec)));
    std::vector<Rec> h(64);
    for (int i = 0; i < 64; ++i) h[i] = Rec{i, 100 + i};
    CK(cudaMemcpy(a, h.data(), 64 * sizeof(Rec), cudaMemcpyHostToDevice));
    tma_selftest<<<1, 64>>>(a, b, 64);
    CK(cudaDeviceSynchronize());
    std::vector<Rec> g(64);
    CK(cudaMemcpy(g.data(), b, 64 * sizeof(Rec), cudaMemcpyDeviceToHost));
    int ok = 1;
    for (int i = 0; i < 64; ++i) ok &= g[i].key == i && g[i].val == 100 + i;
    printf("tma self test: %s\n", ok ? "ok" : "WRONG DATA");
  }
  if (!is("p1") && !is("p2")) return 0;

  const long long n = 1ll << rows_log2;
  const unsigned long long n_keys = 1ull << keys_log2;
  const int log2b = std::max(1, keys_log2 - 10);  // ~1024 keys per bucket
  const int B = 1 << log2b;
  printf("---- two-pass prototype: %lld rows, %llu keys, B=%d buckets (KS=%d, CAPB=%d), hot=%d ----\n", n, n_keys, B, KS, CAPB,
         hot);
  long long *key, *val, *ts;
  CK(cudaMalloc(&key, n * 8));
  CK(cudaMalloc(&val, n * 8));
  CK(cudaMalloc(&ts, n * 8));
  gen_kernel<<<sms * 8, 256>>>(key, val, ts, n, n_keys, hot, 42);
  BDict d{};
  d.log2b = log2b;
  CK(cudaMalloc(&d.slots, (size_t)B * KS * sizeof(KSlot)));
  CK(cudaMalloc(&d.nkeys, B * sizeof(unsigned)));
  CK(cudaMalloc(&d.id_keys, (size_t)B * CAPB * 8));
  bdict_init<<<sms * 8, 256>>>(d.slots, (size_t)B * KS);
  CK(cudaMemset(d.nkeys, 0, B * sizeof(unsigned)));
  const unsigned cap = (unsigned)(n / B + n / B / 4 + 1024);
  Rec* part;
  unsigned* cursor;
  unsigned long long *overflow, *misses;
  CK(cudaMalloc(&part, (size_t)B * cap * sizeof(Rec)));
  CK(cudaMalloc(&cursor, B * sizeof(unsigned)));
  CK(cudaMalloc(&overflow, 8));
  CK(cudaMalloc(&misses, 8));
  CK(cudaMemset(overflow, 0, 8));
  CK(cudaMemset(misses, 0, 8));
  const size_t ids = (size_t)B * CAPB;
  unsigned long long *rows_a, *sum_a, *rows_b, *sum_b;
  CK(cudaMalloc(&rows_a, ids * 8));
  CK(cudaMalloc(&sum_a, ids * 8));
  CK(cudaMalloc(&rows_b, ids * 8));
  CK(cudaMalloc(&sum_b, ids * 8));
  CK(cudaMemset(rows_a, 0, ids * 8));
  CK(cudaMemset(sum_a, 0, ids * 8));
  CK(cudaMemset(rows_b, 0, ids * 8));
  CK(cudaMemset(sum_b, 0, ids * 8));

  Part1Params p1{};
  p1.key = key;
  p1.val = val;
  p1.ts = ts;
  p1.n = n;
  p1.log2b = log2b;
  p1.slide_magic = 18446744074ull;  // ~ 2^64 / 1e9
  p1.q0 = 0;
  p1.out = part;
  p1.cursor = cursor;
  p1.cap = cap;
  p1.overflow = overflow;
  Agg2Params p2{};
  p2.in = part;
  p2.cursor = cursor;
  p2.cap = cap;
  p2.dict = d;
  p2.pane_rows = rows_a;
  p2.pane_sum = sum_a;
  p2.misses = misses;

  constexpr int P1_THREADS = 512, P1_RPT = 16, NR_MAX = 1024;
  constexpr int P1_TILE = P1_THREADS * P1_RPT;
  const size_t sh1 = (size_t)P1_TILE * 16 + (size_t)P1_TILE * 2 + (size_t)(P1_THREADS / 32) * NR_MAX * 2 + NR_MAX * 8;
  auto k1 = part1_kernel<P1_THREADS, P1_RPT, NR_MAX>;
  CK(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh1));
  constexpr int NW = 8, NST = 4, CH = 64;
  const size_t sh2 = (size_t)KS * 16 + (size_t)NW * CAPB * 12 + (size_t)NW * NST * CH * 16 + (size_t)NW * NST * 8;
  auto k2 = agg2_kernel<NW, NST, CH>;
  CK(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh2));
  printf("pass1: %d threads, tile %d rows, %zu B smem; pass2: %d warps, %zu B smem; region cap %u rows\n", P1_THREADS, P1_TILE,
         sh1, NW, sh2, cap);
  if (B > NR_MAX) {
    printf("B > NR_MAX: prototype limit\n");
    return 1;
  }

  int runs = 0;
  auto two_pass = [&] {
    CK(cudaMemsetAsync(cursor, 0, B * sizeof(unsigned)));
    k1<<<sms, P1_THREADS, sh1>>>(p1);
    k2<<<std::min(B, sms), NW * 32, sh2>>>(p2);
    ++runs;
  };
  {
    float t1only = time_ms([&] {
      CK(cudaMemsetAsync(cursor, 0, B * sizeof(unsigned)));
      k1<<<sms, P1_THREADS, sh1>>>(p1);
    }, 5);
    std::vector<unsigned> hc(B);
    CK(cudaMemcpy(hc.data(), cursor, B * 4, cudaMemcpyDeviceToHost));
    unsigned long long tot = 0;
    unsigned mx = 0;
    for (unsigned c : hc) {
      tot += c;
      mx = std::max(mx, c);
    }
    printf("pass 1 alone: %8.3f ms  %7.2f G rows/s; partitioned rows %llu of %lld, max region %u (cap %u)\n", t1only,
           (double)n / (t1only * 1e-3) / 1e9, tot, n, mx, cap);
  }
  if (!strcmp(mode, "p1")) return 0;
  // cold run (every key is new), then timed warm runs
  float cold = time_ms(two_pass, 1);
  printf("cold two-pass done: %.3f ms\n", cold);
  runs = 0;
  CK(cudaMemset(rows_a, 0, ids * 8));
  CK(cudaMemset(sum_a, 0, ids * 8));
  float t12 = time_ms(two_pass, 5);
  const int runs_two = runs;
  float t1 = time_ms([&] {
    CK(cudaMemsetAsync(cursor, 0, B * sizeof(unsigned)));
    k1<<<sms, P1_THREADS, sh1>>>(p1);
  }, 5);
  float t2 = time_ms([&] { k2<<<std::min(B, sms), NW * 32, sh2>>>(p2); }, 5);
  CK(cudaMemset(rows_a, 0, ids * 8));
  CK(cudaMemset(sum_a, 0, ids * 8));
  two_pass();
  CK(cudaDeviceSynchronize());
  (void)runs_two;
  int ref_runs = 0;
  float td = time_ms([&] {
    direct_kernel<<<sms * 8, 256>>>(key, val, n, d, rows_b, sum_b);
    ++ref_runs;
  }, 3);
  CK(cudaDeviceSynchronize());
  // compare: rows_b / sum_b hold ref_runs identical passes
  std::vector<unsigned long long> ha(ids), hb(ids), hsa(ids), hsb(ids);
  CK(cudaMemcpy(ha.data(), rows_a, ids * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hb.data(), rows_b, ids * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hsa.data(), sum_a, ids * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hsb.data(), sum_b, ids * 8, cudaMemcpyDeviceToHost));
  size_t bad = 0;
  unsigned long long tot = 0;
  for (size_t i = 0; i < ids; ++i) {
    tot += ha[i];
    if (ha[i] * ref_runs != hb[i] || hsa[i] * ref_runs != hsb[i]) ++bad;
  }
  unsigned long long h_over = 0, h_miss = 0;
  CK(cudaMemcpy(&h_over, overflow, 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&h_miss, misses, 8, cudaMemcpyDeviceToHost));
  unsigned maxc = 0;
  {
    std::vector<unsigned> hc(B);
    CK(cudaMemcpy(hc.data(), cursor, B * 4, cudaMemcpyDeviceToHost));
    for (unsigned c : hc) maxc = std::max(maxc, c);
  }
  auto rate = [&](float ms) { return (double)n / (ms * 1e-3) / 1e9; };
  printf("cold two-pass (all keys new)   %8.3f ms  %7.2f G rows/s\n", cold, rate(cold));
  printf("two-pass (p1 + p2)             %8.3f ms  %7.2f G rows/s   frac(24B/row @3350 GB/s, H100 SXM data sheet) %.3f\n", t12, rate(t12),
         24.0 * rate(t12) / 3350.0);
  printf("  pass 1 partition alone       %8.3f ms  %7.2f G rows/s   (%.0f GB/s of 40 B/row)\n", t1, rate(t1), 40.0 * rate(t1));
  printf("  pass 2 aggregate alone       %8.3f ms  %7.2f G rows/s\n", t2, rate(t2));
  printf("direct (probe + 2 atomics)     %8.3f ms  %7.2f G rows/s\n", td, rate(td));
  printf("check: rows aggregated %llu of %lld, mismatching ids %zu, region overflow rows %llu, max region fill %u / %u, "
         "global-insert rows %llu\n",
         tot, n, bad, h_over, maxc, cap, h_miss);
  return bad == 0 ? 0 : 2;
}
