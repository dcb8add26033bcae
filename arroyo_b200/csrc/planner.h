// Host-side window state machines: *when* panes close and *which* panes make up each emitted
// window.  Pure C++ (no CUDA) so the control flow can be tested on a box without a GPU
// (arroyo_b200_plan_sliding / arroyo_b200_plan_tumbling in the C ABI).
//
// They follow the reference's control flow statement by statement, including what it does with
// panes that are buffered while the window store runs empty:
//   tumbling: arroyo-worker/src/arrow/tumbling_aggregating_window.rs:250-392, :430-467
//   sliding : arroyo-worker/src/arrow/sliding_aggregating_window.rs:102-210, :556-737
//   state view keys: arroyo-state/src/tables/expiring_time_key_map.rs:833-929
#pragma once

#include <stdint.h>

#include <climits>
#include <map>
#include <set>
#include <vector>

namespace ab {

constexpr int64_t NO_TIME = INT64_MIN;

// Floor division: a negative watermark (the first timestamps of a stream are smaller than the watermark delay) bins
// below zero, so it makes no row late and closes no window.  Truncation would round it up towards zero.
inline int64_t bin_start(int64_t ts, int64_t width) {
  if (width == 0) return ts;
  int64_t r = ts % width;
  if (r < 0) r += width;
  return ts - r;
}

struct PlanStep {
  enum Kind : int64_t { EMIT = 1, JOIN = 2, LEAVE = 3, CHECKPOINT_PANE = 4 };
  int64_t kind;
  int64_t a, b, c;
};

// The keys of ExpiringTimeKeyView that the operators' control flow observes.
struct TableKeys {
  int64_t retention = 0;
  std::set<int64_t> flushed, to_flush;

  void insert(int64_t t) { to_flush.insert(t); }
  void flush(bool has_wm, int64_t wm) {
    for (int64_t t : to_flush) {
      if (has_wm && t < sat_sub(wm, retention)) continue;
      flushed.insert(t);
    }
    to_flush.clear();
    if (has_wm) {
      int64_t cutoff = sat_sub(wm, retention);
      flushed.erase(flushed.begin(), flushed.lower_bound(cutoff));
    }
  }
  void flush_timestamp(int64_t t) {
    if (to_flush.erase(t)) flushed.insert(t);
  }
  void expire_timestamp(int64_t t) {
    flushed.erase(t);
    to_flush.erase(t);
  }
  bool get_min_time(int64_t* out) const {
    bool any = false;
    int64_t m = INT64_MAX;
    if (!flushed.empty()) { m = *flushed.begin(); any = true; }
    if (!to_flush.empty()) { m = any ? std::min(m, *to_flush.begin()) : *to_flush.begin(); any = true; }
    *out = m;
    return any;
  }
  static int64_t sat_sub(int64_t a, int64_t b) {
    __int128 r = (__int128)a - b;
    if (r < INT64_MIN) return INT64_MIN;
    if (r > INT64_MAX) return INT64_MAX;
    return (int64_t)r;
  }
};

struct ExecFlags {
  bool active = false;    // rows received since the last drain
  bool finished = false;  // has drained partial batches (checkpoint / restore)
};

class TumblingPlanner {
 public:
  explicit TumblingPlanner(int64_t width) : width_(width) {}

  // on-time rows arrived for pane `bin` (process_batch, :282-318)
  void touch(int64_t bin) { execs_[bin].active = true; }
  void restore(int64_t bin) { execs_[bin].finished = true; }

  // handle_watermark (:321-392): pop every bin < bin(watermark), ascending
  void watermark(int64_t wm, std::vector<PlanStep>& out) {
    int64_t wbin = bin_start(wm, width_);
    while (!execs_.empty()) {
      auto it = execs_.begin();
      if (!(it->first < wbin)) break;
      int64_t b = it->first;
      execs_.erase(it);
      out.push_back({PlanStep::EMIT, b, b + width_, b});
    }
  }
  // handle_checkpoint (:430-467): every exec with undrained rows writes a partial batch
  void checkpoint(std::vector<PlanStep>& out) {
    for (auto& kv : execs_) {
      if (!kv.second.active) continue;
      kv.second.active = false;
      kv.second.finished = true;
      out.push_back({PlanStep::CHECKPOINT_PANE, kv.first, 0, 0});
    }
  }
  const std::map<int64_t, ExecFlags>& execs() const { return execs_; }

 private:
  int64_t width_;
  std::map<int64_t, ExecFlags> execs_;
};

class SlidingPlanner {
 public:
  enum State { NO_DATA, ONLY_BUFFERED, IN_MEMORY };

  SlidingPlanner(int64_t width, int64_t slide) : width_(width), slide_(slide) { table_.retention = width; }

  // process_batch, per on-time bin range (:627-672)
  void touch(int64_t bin) {
    if (state_ == NO_DATA) {
      state_ = ONLY_BUFFERED;
      t_ = bin;
    } else if (state_ == ONLY_BUFFERED) {
      t_ = std::min(t_, bin);
    }
    execs_[bin].active = true;
  }

  // on_start (:556-595)
  void restore_begin(bool has_wm, int64_t wm) {
    restore_wbin_ = bin_start(has_wm ? wm : 0, slide_);
  }
  // returns true if the pane goes straight to the window store (bin < watermark bin)
  bool restore_pane(int64_t ts) {
    int64_t b = bin_start(ts, slide_);
    table_.flushed.insert(ts);
    if (b < restore_wbin_) {
      tier_.insert(b);
      return true;
    }
    execs_[b].finished = true;
    return false;
  }
  void restore_end(bool has_min, int64_t table_min_time) {
    if (tier_.empty()) {
      if (has_min) {
        state_ = ONLY_BUFFERED;
        t_ = bin_start(table_min_time, slide_);
      } else {
        state_ = NO_DATA;
      }
    } else {
      state_ = IN_MEMORY;
      t_ = restore_wbin_;
    }
  }

  bool should_advance(int64_t wm) const {
    if (state_ == NO_DATA) return false;
    return (__int128)t_ + slide_ <= (__int128)bin_start(wm, slide_);
  }

  // advance (:115-210)
  void advance(std::vector<PlanStep>& out) {
    int64_t b = t_;
    int64_t bin_end = b + slide_;
    table_.flush(true, bin_end);
    int64_t closed = NO_TIME;
    auto it = execs_.find(b);
    if (it != execs_.end()) {
      if (it->second.active) table_.insert(b);
      execs_.erase(it);
      tier_.insert(b);
      closed = b;
      out.push_back({PlanStep::JOIN, b, 0, 0});
    }
    table_.flush_timestamp(bin_end);
    table_.expire_timestamp(bin_end - width_ + slide_);
    out.push_back({PlanStep::EMIT, bin_end - width_, bin_end, closed});
    int64_t cutoff = bin_start(bin_end + slide_ - width_, slide_);
    while (!tier_.empty() && *tier_.begin() < cutoff) {
      out.push_back({PlanStep::LEAVE, *tier_.begin(), 0, 0});
      tier_.erase(tier_.begin());
    }
    if (tier_.empty()) {
      // The reference looks only at the table here, so panes that received rows while the store was non-empty and
      // were never checkpointed (the first batch after a gap longer than the window, rows far ahead) would never be
      // emitted.  Their earliest bin is a candidate too: no on-time row is lost.
      int64_t mt;
      bool has = table_.get_min_time(&mt);
      if (!execs_.empty() && (!has || execs_.begin()->first < mt)) {
        mt = execs_.begin()->first;
        has = true;
      }
      if (has) {
        state_ = ONLY_BUFFERED;
        t_ = bin_start(mt, slide_);
      } else {
        state_ = NO_DATA;
      }
    } else {
      state_ = IN_MEMORY;
      t_ = bin_end;
    }
  }

  // handle_watermark (:676-691)
  void watermark(int64_t wm, std::vector<PlanStep>& out) {
    while (should_advance(wm)) advance(out);
  }

  // handle_checkpoint (:693-737)
  void checkpoint(bool has_wm, int64_t wm, std::vector<PlanStep>& out) {
    for (auto& kv : execs_) {
      if (!kv.second.active) continue;
      kv.second.active = false;
      kv.second.finished = true;
      table_.insert(kv.first);
      out.push_back({PlanStep::CHECKPOINT_PANE, kv.first, 0, 0});
    }
    table_.flush(has_wm, wm);
  }

  State state() const { return state_; }
  int64_t state_time() const { return t_; }
  const std::set<int64_t>& tier() const { return tier_; }
  const std::map<int64_t, ExecFlags>& execs() const { return execs_; }

 private:
  int64_t width_, slide_;
  State state_ = NO_DATA;
  int64_t t_ = 0;
  int64_t restore_wbin_ = 0;
  std::map<int64_t, ExecFlags> execs_;
  std::set<int64_t> tier_;  // panes in the TieredRecordBatchHolder (single tier, :519-521)
  TableKeys table_;
};

}  // namespace ab
