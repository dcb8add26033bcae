// extern "C" entry points of libarroyo_b200.so (see include/arroyo_b200.h for the contract and the
// reference interfaces each one replaces).  Nothing unwinds across this boundary.
#include <algorithm>
#include <chrono>
#include <new>

#include "op.h"
#include "planner.h"

using namespace ab;

struct ArroyoB200Op {
  OpBase* impl;
  double host_process_ms = 0, host_watermark_ms = 0;
};

namespace {
struct WallTimer {
  double& acc;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  explicit WallTimer(double& a) : acc(a) {}
  ~WallTimer() { acc += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};
}  // namespace

namespace {

template <class F>
int32_t guarded(ArroyoB200Op* op, F&& f) {
  if (!op || !op->impl) return ARROYO_B200_INVALID_ARGUMENT;
  try {
    f(op->impl);
    return ARROYO_B200_OK;
  } catch (const Error& e) {
    op->impl->last_error = e.what();
    return e.status;
  } catch (const std::bad_alloc&) {
    op->impl->last_error = "out of host memory";
    return ARROYO_B200_RUNTIME;
  } catch (const std::exception& e) {
    op->impl->last_error = e.what();
    return ARROYO_B200_RUNTIME;
  } catch (...) {
    op->impl->last_error = "unknown C++ exception";
    return ARROYO_B200_RUNTIME;
  }
}

void set_err(char* err, uint64_t len, const char* msg) {
  if (err && len) {
    snprintf(err, (size_t)len, "%s", msg);
  }
}

// Writes the first max_out windows of `v` to `out`; the rest stay queued, in order, for the next
// handle_watermark_device_poll.  The emission has already left the operator, so nothing may be dropped here.
int64_t hand_out(OpBase* o, std::vector<ArroyoB200DeviceBatch>& v, ArroyoB200DeviceBatch* out, int64_t max_out) {
  const size_t n = (size_t)std::min<int64_t>((int64_t)v.size(), std::max<int64_t>(max_out, 0));
  for (size_t i = 0; i < n; ++i) out[i] = v[i];
  o->pending_dev.assign(v.begin() + n, v.end());
  return (int64_t)n;
}

}  // namespace

extern "C" {

int32_t arroyo_b200_abi_version(void) { return 1; }

int32_t arroyo_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

void* arroyo_b200_host_alloc(uint64_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, (size_t)bytes, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}

void arroyo_b200_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

int32_t arroyo_b200_op_create(const ArroyoB200OpConfig* config, ArroyoB200Op** out, char* err, uint64_t err_len) {
  if (!config || !out) {
    set_err(err, err_len, "null config or out pointer");
    return ARROYO_B200_INVALID_ARGUMENT;
  }
  *out = nullptr;
  try {
    OpBase* impl = nullptr;
    switch (config->kind) {
      case ARROYO_B200_TUMBLING_AGGREGATE:
      case ARROYO_B200_SLIDING_AGGREGATE:
        impl = make_window_agg_op(*config);
        break;
      case ARROYO_B200_SESSION_AGGREGATE:
        impl = make_session_op(*config);
        break;
      case ARROYO_B200_INSTANT_JOIN:
        impl = make_instant_join_op(*config);
        break;
      case ARROYO_B200_UPDATING_AGGREGATE:
        impl = make_updating_agg_op(*config);
        break;
      case ARROYO_B200_TTL_JOIN:
        impl = make_ttl_join_op(*config);
        break;
      default:
        set_err(err, err_len, "unknown operator kind");
        return ARROYO_B200_INVALID_ARGUMENT;
    }
    auto* h = new ArroyoB200Op();
    h->impl = impl;
    *out = h;
    return ARROYO_B200_OK;
  } catch (const Error& e) {
    set_err(err, err_len, e.what());
    return e.status;
  } catch (const std::exception& e) {
    set_err(err, err_len, e.what());
    return ARROYO_B200_RUNTIME;
  } catch (...) {
    set_err(err, err_len, "unknown C++ exception");
    return ARROYO_B200_RUNTIME;
  }
}

void arroyo_b200_op_destroy(ArroyoB200Op* op) {
  if (!op) return;
  try {
    if (op->impl && op->impl->pending_out) {
      // an emission that was begun and never collected: wait for its copies, give the buffers back
      op->impl->poll_watermark(true);
      ArroyoB200Batches tmp{};
      batches_finish(op->impl->pending_out, &tmp);
      batches_release(&tmp);
      op->impl->pending_out = nullptr;
    }
    delete op->impl;
  } catch (...) {
  }
  delete op;
}

const char* arroyo_b200_op_last_error(const ArroyoB200Op* op) {
  if (!op || !op->impl) return "invalid handle";
  return op->impl->last_error.c_str();
}

const char* arroyo_b200_op_name(const ArroyoB200Op* op) {
  if (!op || !op->impl) return "";
  return op->impl->name.c_str();
}

int32_t arroyo_b200_op_on_start(ArroyoB200Op* op, struct ArrowArray* state, struct ArrowSchema* schemas, int64_t n,
                                int64_t watermark_ns, int64_t table_min_time_ns) {
  return guarded(op, [&](OpBase* o) { o->on_start(state, schemas, n, watermark_ns, table_min_time_ns); });
}

int32_t arroyo_b200_op_process_batch(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                     struct ArrowArray* batch, const struct ArrowSchema* schema) {
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_process_ms);
  return guarded(op, [&](OpBase* o) { o->process_batch(input_index, in_partitions, batch, schema); });
}

int32_t arroyo_b200_op_process_batch_emit(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                          struct ArrowArray* batch, const struct ArrowSchema* schema, ArroyoB200Batches* out) {
  if (out) memset(out, 0, sizeof *out);
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_process_ms);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(out != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null out");
    auto* priv = new BatchesPriv();
    try {
      o->process_batch_emit(input_index, in_partitions, batch, schema, priv);
    } catch (...) {
      ArroyoB200Batches tmp{};
      batches_finish(priv, &tmp);
      batches_release(&tmp);
      throw;
    }
    batches_finish(priv, out);
  });
}

int32_t arroyo_b200_op_process_device_batch(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                            const uint64_t* cols, int32_t n_cols, int64_t n_rows) {
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(cols != nullptr && n_cols > 0, ARROYO_B200_INVALID_ARGUMENT, "null column list");
    o->process_device_batch(input_index, in_partitions, cols, n_cols, n_rows);
  });
}

int32_t arroyo_b200_op_process_device_batches(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                              const uint64_t* cols, int32_t n_cols, const int64_t* n_rows,
                                              int64_t n_batches) {
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_process_ms);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(cols != nullptr && n_rows != nullptr && n_cols > 0 && n_batches >= 0, ARROYO_B200_INVALID_ARGUMENT,
               "null batch list");
    for (int64_t b = 0; b < n_batches; ++b)
      o->process_device_batch(input_index, in_partitions, cols + b * n_cols, n_cols, n_rows[b]);
  });
}

int32_t arroyo_b200_op_handle_watermark(ArroyoB200Op* op, int64_t watermark_ns, ArroyoB200Batches* out) {
  if (out) memset(out, 0, sizeof *out);
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_watermark_ms);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(out != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null out");
    auto* priv = new BatchesPriv();
    try {
      o->handle_watermark(watermark_ns, priv, nullptr);
    } catch (...) {
      ArroyoB200Batches tmp{};
      batches_finish(priv, &tmp);
      batches_release(&tmp);
      throw;
    }
    batches_finish(priv, out);
  });
}

int32_t arroyo_b200_op_handle_tick(ArroyoB200Op* op, ArroyoB200Batches* out) {
  if (out) memset(out, 0, sizeof *out);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(out != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null out");
    auto* priv = new BatchesPriv();
    try {
      o->handle_tick(priv);
    } catch (...) {
      ArroyoB200Batches tmp{};
      batches_finish(priv, &tmp);
      batches_release(&tmp);
      throw;
    }
    batches_finish(priv, out);
  });
}

int32_t arroyo_b200_op_handle_watermark_begin(ArroyoB200Op* op, int64_t watermark_ns) {
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_watermark_ms);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(o->pending_out == nullptr, ARROYO_B200_INVALID_ARGUMENT,
               "the previous emission has not been collected (handle_watermark_poll)");
    o->pending_out = new BatchesPriv();
    try {
      o->begin_watermark(watermark_ns);
    } catch (...) {
      o->poll_watermark(true);
      ArroyoB200Batches tmp{};
      batches_finish(o->pending_out, &tmp);
      batches_release(&tmp);
      o->pending_out = nullptr;
      throw;
    }
  });
}

int32_t arroyo_b200_op_handle_watermark_poll(ArroyoB200Op* op, int32_t block, ArroyoB200Batches* out, int32_t* ready) {
  if (out) memset(out, 0, sizeof *out);
  if (ready) *ready = 0;
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_watermark_ms);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(out != nullptr && ready != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null out");
    if (!o->pending_out) {
      *ready = 1;  // nothing outstanding: an empty list
      return;
    }
    if (!o->poll_watermark(block != 0)) return;
    batches_finish(o->pending_out, out);
    o->pending_out = nullptr;
    *ready = 1;
  });
}

int32_t arroyo_b200_op_run_batches(ArroyoB200Op* op, struct ArrowArray* batches, const struct ArrowSchema* schema,
                                    int64_t n_batches, const int64_t* watermarks, int32_t async_emit,
                                    ArroyoB200Batches* out, int64_t* n_consumed) {
  if (out) memset(out, 0, sizeof *out);
  if (n_consumed) *n_consumed = 0;
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  auto* acc = new BatchesPriv();
  int32_t st = guarded(op, [&](OpBase* o) {
    AB_REQUIRE(out != nullptr && n_consumed != nullptr && (n_batches == 0 || (batches != nullptr && schema != nullptr)),
               ARROYO_B200_INVALID_ARGUMENT, "null argument");
    // the windows of an emission that has been begun: hand them on once their copies have completed
    auto collect = [&](bool block) {
      if (!o->pending_out || !o->poll_watermark(block)) return;
      for (auto& a : o->pending_out->arrays) acc->arrays.push_back(a);
      for (auto& s : o->pending_out->schemas) acc->schemas.push_back(s);
      delete o->pending_out;
      o->pending_out = nullptr;
    };
    for (int64_t i = 0; i < n_batches; ++i) {
      {
        WallTimer wt(op->host_process_ms);
        o->process_batch(0, 1, &batches[i], schema);
      }
      ++*n_consumed;
      const int64_t wm = watermarks ? watermarks[i] : INT64_MIN;
      WallTimer wt(op->host_watermark_ms);
      if (wm == INT64_MIN) {
        if (async_emit && (i & 7) == 0) collect(false);
        continue;
      }
      if (async_emit) {
        collect(true);  // windows leave in order: the previous emission first
        o->pending_out = new BatchesPriv();
        try {
          o->begin_watermark(wm);
        } catch (...) {
          // same clean-up as arroyo_b200_op_handle_watermark_begin: nothing half-emitted stays pending
          o->poll_watermark(true);
          ArroyoB200Batches tmp{};
          batches_finish(o->pending_out, &tmp);
          batches_release(&tmp);
          o->pending_out = nullptr;
          throw;
        }
      } else {
        o->handle_watermark(wm, acc, nullptr);
      }
    }
    if (async_emit) collect(false);
  });
  if (out) {
    batches_finish(acc, out);
  } else {
    // null `out` was rejected above: drop whatever was accumulated instead of writing through it
    ArroyoB200Batches tmp{};
    batches_finish(acc, &tmp);
    batches_release(&tmp);
  }
  return st;
}

int32_t arroyo_b200_op_handle_watermark_device(ArroyoB200Op* op, int64_t watermark_ns, ArroyoB200DeviceBatch* out,
                                               int64_t max_out, int64_t* n_out) {
  if (n_out) *n_out = 0;
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_watermark_ms);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(n_out != nullptr && (out != nullptr || max_out <= 0), ARROYO_B200_INVALID_ARGUMENT, "null out");
    // the queued windows live in the output buffers the next emission would write
    AB_REQUIRE(o->pending_dev.empty(), ARROYO_B200_INVALID_ARGUMENT,
               "windows of the previous emission are still queued (handle_watermark_device_poll)");
    std::vector<ArroyoB200DeviceBatch> v;
    o->handle_watermark(watermark_ns, nullptr, &v);
    *n_out = hand_out(o, v, out, max_out);
  });
}

int32_t arroyo_b200_op_handle_watermark_device_begin(ArroyoB200Op* op, int64_t watermark_ns) {
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_watermark_ms);
  return guarded(op, [&](OpBase* o) {
    // the queued windows live in the output buffers the next emission would write (every operator kind)
    AB_REQUIRE(o->pending_dev.empty(), ARROYO_B200_INVALID_ARGUMENT,
               "windows of the previous emission are still queued (handle_watermark_device_poll)");
    o->begin_watermark_device(watermark_ns);
  });
}

int32_t arroyo_b200_op_handle_watermark_device_poll(ArroyoB200Op* op, ArroyoB200DeviceBatch* out, int64_t max_out,
                                                    int64_t* n_out) {
  if (n_out) *n_out = 0;
  if (!op) return ARROYO_B200_INVALID_ARGUMENT;
  WallTimer wt(op->host_watermark_ms);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(n_out != nullptr && (out != nullptr || max_out <= 0), ARROYO_B200_INVALID_ARGUMENT, "null out");
    std::vector<ArroyoB200DeviceBatch> v;
    o->poll_watermark_device(&v);
    *n_out = hand_out(o, v, out, max_out);
  });
}

int32_t arroyo_b200_op_handle_checkpoint(ArroyoB200Op* op, int64_t watermark_ns, ArroyoB200Batches* state_out) {
  if (state_out) memset(state_out, 0, sizeof *state_out);
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(state_out != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null out");
    auto* priv = new BatchesPriv();
    try {
      o->handle_checkpoint(watermark_ns, priv);
    } catch (...) {
      ArroyoB200Batches tmp{};
      batches_finish(priv, &tmp);
      batches_release(&tmp);
      throw;
    }
    batches_finish(priv, state_out);
  });
}

int32_t arroyo_b200_op_on_close(ArroyoB200Op* op, int32_t end_of_data, ArroyoB200Batches* out) {
  if (out) memset(out, 0, sizeof *out);
  return guarded(op, [&](OpBase* o) {
    auto* priv = new BatchesPriv();
    try {
      o->on_close(end_of_data, priv);
    } catch (...) {
      ArroyoB200Batches tmp{};
      batches_finish(priv, &tmp);
      batches_release(&tmp);
      throw;
    }
    if (out) {
      batches_finish(priv, out);
    } else {
      ArroyoB200Batches tmp{};
      batches_finish(priv, &tmp);
      batches_release(&tmp);
    }
  });
}

int32_t arroyo_b200_op_flush(ArroyoB200Op* op) {
  return guarded(op, [&](OpBase* o) { o->flush(); });
}

int32_t arroyo_b200_op_submit(ArroyoB200Op* op) {
  return guarded(op, [&](OpBase* o) { o->submit(); });
}

void arroyo_b200_release_batches(ArroyoB200Batches* batches) { batches_release(batches); }

int32_t arroyo_b200_op_stats(ArroyoB200Op* op, ArroyoB200Stats* out) {
  return guarded(op, [&](OpBase* o) {
    AB_REQUIRE(out != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null out");
    o->stats(out);
    out->host_process_ms = op->host_process_ms;
    out->host_watermark_ms = op->host_watermark_ms;
  });
}

uint64_t arroyo_b200_hash_key(int64_t key) { return mix64((uint64_t)key); }

uint32_t arroyo_b200_server_for_hash(uint64_t h, uint32_t n) {
  if (n == 0) return 0;
  uint64_t range = UINT64_MAX / (uint64_t)n;
  return (uint32_t)((h / range) % (uint64_t)n);
}

int64_t arroyo_b200_bin_start(int64_t ts_ns, int64_t width_ns) {
  if (width_ns < 2 || ts_ns < 0) return width_ns <= 0 ? ts_ns : ts_ns - ts_ns % width_ns;
  FastDivU64 d = FastDivU64::make((uint64_t)width_ns);
  return (int64_t)(d.div_host((uint64_t)ts_ns) * (uint64_t)width_ns);
}

// ---- host-only planner hooks ----------------------------------------------------------------
static int64_t write_steps(const std::vector<PlanStep>& steps, int64_t* out, int64_t cap) {
  if ((int64_t)steps.size() * 4 > cap) return -1;
  for (size_t i = 0; i < steps.size(); ++i) {
    out[4 * i + 0] = steps[i].kind;
    out[4 * i + 1] = steps[i].a;
    out[4 * i + 2] = steps[i].b;
    out[4 * i + 3] = steps[i].c;
  }
  return (int64_t)steps.size();
}

int64_t arroyo_b200_plan_sliding(int64_t width_ns, int64_t slide_ns, const int64_t* events, int64_t n_events,
                                 int64_t* out, int64_t out_cap) {
  if (slide_ns <= 0 || width_ns <= 0 || width_ns % slide_ns) return -2;
  SlidingPlanner pl(width_ns, slide_ns);
  std::vector<PlanStep> steps;
  bool has_wm = false;
  int64_t wm = 0;
  for (int64_t i = 0; i < n_events; ++i) {
    int64_t kind = events[2 * i], v = events[2 * i + 1];
    if (kind == 0) {
      // late test as in process_batch (:631-633)
      if (has_wm && v < bin_start(wm, slide_ns)) continue;
      pl.touch(v);
    } else if (kind == 1) {
      has_wm = true;
      wm = v;
      pl.watermark(v, steps);
    } else if (kind == 2) {
      pl.checkpoint(has_wm, wm, steps);
    }
  }
  return write_steps(steps, out, out_cap);
}

int64_t arroyo_b200_plan_tumbling(int64_t width_ns, const int64_t* events, int64_t n_events, int64_t* out,
                                  int64_t out_cap) {
  if (width_ns <= 0) return -2;
  TumblingPlanner pl(width_ns);
  std::vector<PlanStep> steps;
  bool has_wm = false;
  int64_t wm = 0;
  for (int64_t i = 0; i < n_events; ++i) {
    int64_t kind = events[2 * i], v = events[2 * i + 1];
    if (kind == 0) {
      if (has_wm && v < bin_start(wm, width_ns)) continue;
      pl.touch(v);
    } else if (kind == 1) {
      has_wm = true;
      wm = v;
      pl.watermark(v, steps);
    } else if (kind == 2) {
      pl.checkpoint(steps);
    }
  }
  return write_steps(steps, out, out_cap);
}

}  // extern "C"
