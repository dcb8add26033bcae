// What the instant join (join.cu) and the join with expiration (ttl_join.cu) share: a join side's device arenas and
// the host batches it accepts, which input feeds which side, the count of a probe's output pairs, and the writer of the
// output batch of a pair list.
#pragma once

#include <algorithm>
#include <climits>
#include <string>
#include <vector>

#include "op.h"
#include "scan.cuh"
#include "validity.cuh"

namespace ab {

constexpr int JOIN_THREADS = 256;

// ---- output kernels -----------------------------------------------------------------------
struct GatherParams {
  const int* idx;          // pair side to read
  const long long* src;    // source column
  long long* dst;
  unsigned char* valid;    // optional validity bytes
  long long n;
};
static __global__ void gather_kernel(const __grid_constant__ GatherParams p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    int j = p.idx[i];
    p.dst[i] = j >= 0 ? p.src[j] : 0;
    if (p.valid) p.valid[i] = j >= 0 ? 1 : 0;
  }
}
static __global__ void gather_ts_kernel(const int* __restrict__ il, const int* __restrict__ ir, const long long* __restrict__ lts,
                                        const long long* __restrict__ rts, long long* __restrict__ dst, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    int a = il[i], b = ir[i];
    long long ta = a >= 0 ? lts[a] : LLONG_MIN, tb = b >= 0 ? rts[b] : LLONG_MIN;
    dst[i] = max(ta, tb);
  }
}
// ---- join sides ---------------------------------------------------------------------------
// The joins compare raw 64-bit key patterns, which is equality only for integer-like keys of one type: an Int64,
// UInt64 or timestamp[ns] key, the same type on both sides (INTEGRATION.md §1).  A Float64 key (-0.0 = 0.0) or an
// Int64 key against a UInt64 key is refused.  `seen_*`: the key format an earlier batch of this / the other side
// carried ("" while unknown).
inline int join_key_class(const std::string& f) {
  if (f == "l") return 1;
  if (f == "L") return 2;
  if (f.compare(0, 4, "tsn:") == 0) return 3;
  return 0;
}
inline void require_join_key_type(const std::string& f, const std::string& seen_this, const std::string& seen_other) {
  const int k = join_key_class(f);
  if (k == 0) throw Error(ARROYO_B200_UNSUPPORTED, "join key of type '" + f + "' (supported: l, L, tsn:)");
  for (const std::string* s : {&seen_this, &seen_other})
    if (!s->empty() && join_key_class(*s) != k)
      throw Error(ARROYO_B200_UNSUPPORTED, "join key of type '" + f + "' after keys of type '" + *s + "'");
}

// A host batch a join side has accepted: its columns and the first element of each.
struct JoinBatch {
  std::vector<InColumn> cols;
  int64_t n = 0;
  const uint64_t* data[ARROYO_B200_MAX_COLS] = {};
};

// One input of a join: its columns are the leading `_key_*` routing copies (`n_routing` of them), then the key, the
// timestamp and the payload in any order.  The routing copies are stripped from the output like `unkeyed_batch`
// does (arroyo-rpc/src/df.rs:359-367) and never reach the device.  Rows [0, n) of every other column sit in a device
// arena of `cap` rows.
struct JoinSide {
  int n_cols = 0, ts_col = 0, key_col = 0, n_routing = 0;
  std::vector<int> payload;          // input column indices that appear in the output
  std::vector<std::string> formats;  // Arrow format per input column
  std::string key_format;            // the key's format once a host batch has shown it
  std::vector<DevBuf> cols;          // device columns (the routing columns stay empty)
  int64_t n = 0, cap = 0;

  // Imports a host batch for this side and checks it before anything changes: its column count (`count_msg` refuses
  // it) and its key type against `seen_key`, the key this side has shown so far, and the other side's.
  JoinBatch import(const ArrowArray* a, const ArrowSchema* s, const std::string& seen_key, const JoinSide& other,
                   const char* count_msg = "join side has the wrong number of columns") const {
    JoinBatch b;
    b.cols = import_batch(a, s, &b.n);
    AB_REQUIRE((int)b.cols.size() == n_cols, ARROYO_B200_INVALID_ARGUMENT, count_msg);
    require_join_key_type(b.cols[key_col].format, seen_key, other.key_format);
    for (int c = 0; c < n_cols; ++c) b.data[c] = b.cols[c].data;
    return b;
  }

  // Records the formats of an accepted batch: the output columns carry them.
  void take_formats(const std::vector<InColumn>& in) {
    for (int c = 0; c < n_cols; ++c) formats[c] = in[c].format;
    key_format = in[key_col].format;
  }

  // Makes room for `extra` more rows: the arenas double from 2^16 rows.  `links` (4 bytes per row) grows with them;
  // `stale` holds buffers sized for the old capacity, which are released.
  void reserve(int64_t extra, cudaStream_t stream, DevBuf* links = nullptr, std::vector<DevBuf>* stale = nullptr) {
    if (n + extra <= cap) return;
    int64_t nc = std::max<int64_t>(cap * 2, 1 << 16);
    while (nc < n + extra) nc *= 2;
    // rows are numbered as int (pairs, links) and as row + 1 in 32 bits (table slots)
    AB_REQUIRE(nc < (1ll << 31), ARROYO_B200_RUNTIME, "join side holds more than 2^31 rows");
    if (stale)
      for (DevBuf& b : *stale) b.release();
    auto grow = [&](DevBuf& b, size_t elem) {
      DevBuf nb((size_t)nc * elem);
      if (n) AB_CUDA(cudaMemcpyAsync(nb.p, b.p, (size_t)n * elem, cudaMemcpyDeviceToDevice, stream));
      AB_CUDA(cudaStreamSynchronize(stream));
      b = std::move(nb);
    };
    for (int c = n_routing; c < n_cols; ++c) grow(cols[c], 8);
    if (links) grow(*links, 4);
    cap = nc;
  }

  // Copies `rows` rows of every non-routing column `src[c]` (host or device memory) to the end of the arenas, which
  // have room for them.
  void append(const uint64_t* const* src, int64_t rows, bool host, cudaStream_t stream, ArroyoB200Stats& st) {
    for (int c = n_routing; c < n_cols; ++c)
      AB_CUDA(cudaMemcpyAsync(cols[c].as<long long>() + n, src[c], (size_t)rows * 8,
                              host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, stream));
    if (host) st.h2d_bytes += (uint64_t)rows * 8 * (uint64_t)(n_cols - n_routing);
    n += rows;
  }
};

inline void init_join_side(JoinSide& s, int n_cols, int ts_col, int key_col, int n_routing) {
  AB_REQUIRE(n_cols >= 2 && n_cols <= ARROYO_B200_MAX_COLS, ARROYO_B200_INVALID_ARGUMENT, "bad join side n_cols");
  AB_REQUIRE(ts_col >= 0 && ts_col < n_cols && key_col >= 0 && key_col < n_cols && n_routing >= 0 && n_routing < n_cols,
             ARROYO_B200_INVALID_ARGUMENT, "bad join side columns");
  AB_REQUIRE(key_col >= n_routing && ts_col >= n_routing, ARROYO_B200_INVALID_ARGUMENT,
             "join key or timestamp column among the routing columns");
  s.n_cols = n_cols;
  s.ts_col = ts_col;
  s.key_col = key_col;
  s.n_routing = n_routing;
  for (int i = n_routing; i < n_cols; ++i)
    if (i != ts_col) s.payload.push_back(i);
  s.formats.assign(n_cols, "l");
  s.formats[ts_col] = "tsn:";
  s.cols.resize(n_cols);
}

// ---- the operators' shared part -------------------------------------------------------------
// Makes `b` hold at least `bytes`, doubling: buffers that follow a growing stream are reallocated a few times only.
inline void grow(DevBuf& b, size_t bytes) {
  if (b.bytes < bytes) b.alloc(std::max(bytes, b.bytes * 2));
}

class JoinOpBase : public OpBase {
 public:
  void stats(ArroyoB200Stats* out) override { *out = st_; }

 protected:
  ArroyoB200Stats st_{};
  DevBuf sums_;      // scan scratch
  DevBuf pairs_[2];  // the pair list: the left / right row of each output row (-1: none)

  int grid_for(int64_t n) const {
    return (int)std::max<int64_t>(1, std::min<int64_t>((n + JOIN_THREADS - 1) / JOIN_THREADS, (int64_t)num_sms_ * 8));
  }

  // Input index -> side (instant_join.rs:249-253): the first half of the inputs feed the left side.
  static int side_of(uint32_t index, uint32_t in_partitions) {
    AB_REQUIRE(in_partitions >= 2 && in_partitions % 2 == 0, ARROYO_B200_INVALID_ARGUMENT, "join needs an even number of inputs");
    const int sd = (int)(index / (in_partitions / 2));
    AB_REQUIRE(sd == 0 || sd == 1, ARROYO_B200_INVALID_ARGUMENT, "bad input index");
    return sd;
  }

  // The output pairs of `n` probe rows: `count` launches the kernel that writes their counts to cnt[0, n), the
  // exclusive scan of the counts goes to `off`, and the total comes back through `total_dev` to `*total_host`.
  template <class Count>
  int64_t count_pairs(Count&& count, const unsigned int* cnt, int64_t n, unsigned long long* off,
                      unsigned long long* total_dev, unsigned long long* total_host) {
    count();
    AB_CUDA(cudaGetLastError());
    device_exclusive_scan(cnt, n, off, total_dev, sums_, stream_);
    AB_CUDA(cudaMemcpyAsync(total_host, total_dev, 8, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    st_.kernel_launches += 4;
    return (int64_t)*total_host;
  }

  void reserve_pairs(int64_t n) {
    for (DevBuf& p : pairs_) grow(p, (size_t)n * 4);
  }

  // Writes the output of the first `n` pairs: the columns [left payload..., right payload..., _timestamp = max(l, r)]
  // (arroyo-planner/src/plan/join.rs:165-185), named l<c> / r<c> after their input column.  A nullable side may be
  // missing from a pair: its columns carry validity.  The output is one host batch appended to `out_host` or, when that
  // is null, one device batch appended to `out_dev` (no nullable side), which points into buffers the next call reuses.
  void write_output(const JoinSide& L, const JoinSide& R, int64_t n, bool l_nullable, bool r_nullable,
                    BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>* out_dev) {
    const JoinSide* side[2] = {&L, &R};
    const bool nullable[2] = {l_nullable, r_nullable};
    out_cols_.resize(L.payload.size() + R.payload.size());
    out_valid_.resize(out_cols_.size());
    std::vector<OutColumn> cols;
    size_t oc = 0;
    for (int sd = 0; sd < 2; ++sd) {
      for (int c : side[sd]->payload) {
        grow(out_cols_[oc], (size_t)n * 8);
        if (nullable[sd]) grow(out_valid_[oc], (size_t)n + 64);
        GatherParams gp{pairs_[sd].as<int>(), side[sd]->cols[c].as<long long>(), out_cols_[oc].as<long long>(),
                        nullable[sd] ? out_valid_[oc].as<unsigned char>() : nullptr, n};
        gather_kernel<<<grid_for(n), JOIN_THREADS, 0, stream_>>>(gp);
        AB_CUDA(cudaGetLastError());
        ++st_.kernel_launches;
        if (out_host) {
          OutColumn o;
          o.name = std::string(sd == 0 ? "l" : "r") + std::to_string(c);
          o.format = side[sd]->formats[c];
          o.data = d2h_pinned(out_cols_[oc].p, (size_t)n * 8, stream_, &st_.d2h_bytes);
          if (nullable[sd]) {
            grow(out_bits_, (size_t)((n + 31) / 32) * 4);
            export_validity(o, out_valid_[oc].as<unsigned char>(), n, out_bits_.as<unsigned int>(), grid_for(n),
                            JOIN_THREADS, stream_, st_);
          }
          cols.push_back(o);
        }
        ++oc;
      }
    }
    grow(out_ts_, (size_t)n * 8);
    gather_ts_kernel<<<grid_for(n), JOIN_THREADS, 0, stream_>>>(pairs_[0].as<int>(), pairs_[1].as<int>(),
                                                               L.cols[L.ts_col].as<long long>(),
                                                               R.cols[R.ts_col].as<long long>(), out_ts_.as<long long>(), n);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    st_.rows_out += (uint64_t)n;
    ++st_.windows_out;
    if (out_host) {
      OutColumn t;
      t.name = "_timestamp";
      t.format = "tsn:";
      t.data = d2h_pinned(out_ts_.p, (size_t)n * 8, stream_, &st_.d2h_bytes);
      cols.push_back(t);
      AB_CUDA(cudaStreamSynchronize(stream_));
      out_host->arrays.emplace_back();
      out_host->schemas.emplace_back();
      export_batch(cols, n, &out_host->arrays.back(), &out_host->schemas.back());
    } else {
      ArroyoB200DeviceBatch d{};
      d.n_rows = n;
      for (const DevBuf& b : out_cols_) d.cols[d.n_cols++] = (uint64_t)b.p;
      d.cols[d.n_cols++] = (uint64_t)out_ts_.p;
      out_dev->push_back(d);
      AB_CUDA(cudaStreamSynchronize(stream_));
    }
  }

 private:
  std::vector<DevBuf> out_cols_, out_valid_;  // one per payload column of both sides
  DevBuf out_ts_, out_bits_;
};

}  // namespace ab
