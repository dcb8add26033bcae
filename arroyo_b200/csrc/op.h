// Operator base class behind the C ABI: one virtual per ArrowOperator trait method
// (arroyo-operator/src/operator.rs:1143-1257).
#pragma once

#include <string>
#include <vector>

#include "arrow_io.h"
#include "common.cuh"

namespace ab {

class OpBase {
 public:
  ArroyoB200OpConfig cfg{};
  std::string last_error;
  std::string name;

  // Destroys the stream the operator created.  Each operator's own destructor calls drain_stream() first: nothing may
  // still run on the stream when its buffers and input batches are released.
  virtual ~OpBase() {
    if (own_stream_) cudaStreamDestroy(stream_);
  }
  virtual void on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t watermark, int64_t table_min) = 0;
  virtual void process_batch(uint32_t index, uint32_t in_partitions, ArrowArray* batch, const ArrowSchema* schema) = 0;
  // process_batch for operators that emit from it (the TTL join); everything else emits nothing here
  virtual void process_batch_emit(uint32_t index, uint32_t in_partitions, ArrowArray* batch, const ArrowSchema* schema,
                                  BatchesPriv* /*out*/) {
    process_batch(index, in_partitions, batch, schema);
  }
  virtual void process_device_batch(uint32_t index, uint32_t in_partitions, const uint64_t* cols, int32_t n_cols,
                                    int64_t n_rows) = 0;
  // exactly one of out_host / out_dev is non-null
  virtual void handle_watermark(int64_t watermark, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>* out_dev) = 0;
  virtual void handle_checkpoint(int64_t watermark, BatchesPriv* out) = 0;
  virtual void on_close(int end_of_data, BatchesPriv* out) = 0;
  virtual void handle_tick(BatchesPriv* /*out*/) {}
  // the key-value state table the updating aggregate writes at a checkpoint; every other operator has none
  virtual void checkpoint_state(BatchesPriv* /*out*/) {}
  // stores rows of a join side's key-time table without probing (the TTL join); every other operator has none
  virtual void restore_side(uint32_t /*side*/, ArrowArray* /*batches*/, ArrowSchema* /*schemas*/, int64_t /*n*/) {
    throw Error(ARROYO_B200_UNSUPPORTED, name + ": restore_side is only for the join with expiration");
  }
  // the clock the updating aggregate's time-to-idle runs on; every other operator has none
  virtual void set_clock(int64_t /*now_ns*/) {
    throw Error(ARROYO_B200_UNSUPPORTED, name + ": set_clock is only for the updating aggregate");
  }
  virtual void flush() = 0;
  // enqueue whatever input is still being batched on the host side; does not wait
  virtual void submit() {}
  // handle_watermark split in two, the way the reference's operators hand long-running work to
  // ArrowOperator::future_to_poll / handle_future_result (operator.rs:1190-1204): `begin` enqueues the emission and
  // the device->host copies of its windows into `pending_out`, `poll` says whether those copies have completed.
  BatchesPriv* pending_out = nullptr;
  virtual void begin_watermark(int64_t watermark) { handle_watermark(watermark, pending_out, nullptr); }
  virtual bool poll_watermark(bool /*block*/) { return true; }
  // handle_watermark with device-resident output, split the same way: `begin` enqueues the emission and returns
  // without waiting for the windows' row counts; `poll` waits for them and hands the windows out.  Operators without
  // their own implementation emit in `begin`.
  std::vector<ArroyoB200DeviceBatch> pending_dev;
  virtual void begin_watermark_device(int64_t watermark) {
    pending_dev.clear();
    handle_watermark(watermark, nullptr, &pending_dev);
  }
  virtual void poll_watermark_device(std::vector<ArroyoB200DeviceBatch>* out) {
    out->swap(pending_dev);
    pending_dev.clear();
  }
  virtual void stats(ArroyoB200Stats* out) = 0;

 protected:
  int device_ = 0;
  cudaStream_t stream_ = nullptr;
  bool own_stream_ = false;
  int num_sms_ = 132;  // set from the device by open_device

  // Every constructor calls this once its config is valid, so a bad config is refused without touching CUDA: takes
  // device `c.device` and the caller's stream `c.stream`, or a new non-blocking stream when none is given.
  void open_device(const ArroyoB200OpConfig& c) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0)
      throw Error(ARROYO_B200_FATAL, "no CUDA device available: libarroyo_b200 has no CPU fallback");
    AB_REQUIRE(c.device >= 0 && c.device < count, ARROYO_B200_INVALID_ARGUMENT, "bad device ordinal");
    device_ = c.device;
    set_device();
    cudaDeviceProp prop{};
    AB_CUDA(cudaGetDeviceProperties(&prop, device_));
    num_sms_ = prop.multiProcessorCount;
    if (c.stream) {
      stream_ = (cudaStream_t)c.stream;
    } else {
      AB_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
      own_stream_ = true;
    }
  }
  void set_device() const { AB_CUDA(cudaSetDevice(device_)); }
  // first step of a destructor (errors are ignored there)
  void drain_stream() const {
    cudaSetDevice(device_);
    cudaStreamSynchronize(stream_);
  }
};

OpBase* make_window_agg_op(const ArroyoB200OpConfig& cfg);
OpBase* make_instant_join_op(const ArroyoB200OpConfig& cfg);
OpBase* make_session_op(const ArroyoB200OpConfig& cfg);
OpBase* make_updating_agg_op(const ArroyoB200OpConfig& cfg);
OpBase* make_ttl_join_op(const ArroyoB200OpConfig& cfg);
OpBase* make_instant_agg_op(const ArroyoB200OpConfig& cfg);
OpBase* make_window_fn_op(const ArroyoB200OpConfig& cfg);

}  // namespace ab
