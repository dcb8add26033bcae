// Minimal Arrow C Data Interface import / export for 64-bit fixed-width columns and one level of
// struct nesting (the `window{start,end}` column, arroyo-planner/src/schemas.rs:7-23).
// This is the same mechanism the reference uses for its UDF dylib boundary
// (arroyo-udf/arroyo-udf-common/src/lib.rs:12-69).
#pragma once

#include <algorithm>
#include <deque>
#include <string>
#include <vector>

#include "common.cuh"

namespace ab {

// ---- import -------------------------------------------------------------------------------
struct InColumn {
  const uint64_t* data;  // first logical element (offsets applied)
  std::string format;
  const uint8_t* validity = nullptr;  // import_batch's `nullable_col` only, when it has nulls: bit validity_bit + row
  int64_t validity_bit = 0;
};

inline bool format_is_64bit(const char* f) {
  if (!f) return false;
  if (!strcmp(f, "l") || !strcmp(f, "L") || !strcmp(f, "g")) return true;
  if (!strncmp(f, "tsn:", 4)) return true;  // timestamp[ns]
  if (!strcmp(f, "tDn")) return true;       // duration[ns]
  return false;
}

// A struct column of a batch imported with its structs flattened: its children are flat columns
// [first, first + names.size()).
struct Nest {
  int first;
  std::string name;
  std::vector<std::string> names, formats;
};

// Validates a record batch exported as a struct array and returns its columns.  Nulls are refused, except in column
// `nullable_col`, whose validity bitmap is then handed back.  With `nests`, a struct column whose children are all
// 64-bit takes their places among the columns and is recorded there (one level; the window function's input);
// without it, as everywhere else, a struct column is refused.
inline std::vector<InColumn> import_batch(const ArrowArray* a, const ArrowSchema* s, int64_t* n_rows,
                                          int64_t nullable_col = -1, std::vector<Nest>* nests = nullptr) {
  AB_REQUIRE(a && s, ARROYO_B200_INVALID_ARGUMENT, "null batch or schema");
  AB_REQUIRE(s->format && !strcmp(s->format, "+s"), ARROYO_B200_INVALID_ARGUMENT,
             "batch must be exported as a struct array (format +s)");
  AB_REQUIRE(a->n_children == s->n_children, ARROYO_B200_INVALID_ARGUMENT, "array/schema children mismatch");
  AB_REQUIRE(a->null_count <= 0 || a->n_buffers == 0 || a->buffers[0] == nullptr, ARROYO_B200_UNSUPPORTED,
             "null rows at the struct level are not supported");
  if (nests) {
    nests->clear();
    // the struct array's children become the batch's: its offset adds to theirs (the batch's is kept separately)
    std::vector<const ArrowArray*> arrays;
    std::vector<const ArrowSchema*> schemas;
    std::vector<int64_t> offsets;
    std::vector<ArrowArray> flat_storage;
    for (int64_t i = 0; i < a->n_children; ++i) {
      const ArrowArray* c = a->children[i];
      const ArrowSchema* cs = s->children[i];
      AB_REQUIRE(c && cs, ARROYO_B200_INVALID_ARGUMENT, "null child");
      if (!cs->format || strcmp(cs->format, "+s") != 0) {
        arrays.push_back(c);
        schemas.push_back(cs);
        offsets.push_back(0);
        continue;
      }
      AB_REQUIRE(c->n_children == cs->n_children && c->n_children > 0, ARROYO_B200_INVALID_ARGUMENT,
                 "struct column: array/schema children mismatch");
      AB_REQUIRE(c->length >= a->length + a->offset, ARROYO_B200_INVALID_ARGUMENT, "child shorter than batch");
      AB_REQUIRE(c->null_count == 0 || c->n_buffers == 0 || c->buffers[0] == nullptr, ARROYO_B200_UNSUPPORTED,
                 std::string("column ") + (cs->name ? cs->name : "?") + " has nulls: NULLs are outside the supported subset");
      Nest n;
      n.first = (int)arrays.size();
      n.name = cs->name ? cs->name : "";
      for (int64_t j = 0; j < c->n_children; ++j) {
        AB_REQUIRE(c->children[j] && cs->children[j], ARROYO_B200_INVALID_ARGUMENT, "null child");
        AB_REQUIRE(!cs->children[j]->format || strcmp(cs->children[j]->format, "+s") != 0, ARROYO_B200_UNSUPPORTED,
                   "struct column nested in a struct column");
        arrays.push_back(c->children[j]);
        schemas.push_back(cs->children[j]);
        offsets.push_back(c->offset);
        n.names.push_back(cs->children[j]->name ? cs->children[j]->name : "");
        n.formats.push_back(cs->children[j]->format ? cs->children[j]->format : "");
      }
      nests->push_back(n);
    }
    // the flattened batch, as a view: children with the struct's offset folded into their own
    flat_storage.resize(arrays.size());
    std::vector<ArrowArray*> ap(arrays.size());
    std::vector<ArrowSchema*> sp(arrays.size());
    for (size_t i = 0; i < arrays.size(); ++i) {
      flat_storage[i] = *arrays[i];
      flat_storage[i].offset += offsets[i];
      flat_storage[i].length -= offsets[i];
      ap[i] = &flat_storage[i];
      sp[i] = const_cast<ArrowSchema*>(schemas[i]);
    }
    ArrowArray fa = *a;
    ArrowSchema fs = *s;
    fa.n_children = fs.n_children = (int64_t)arrays.size();
    fa.children = ap.data();
    fs.children = sp.data();
    return import_batch(&fa, &fs, n_rows, nullable_col);
  }
  std::vector<InColumn> cols;
  cols.reserve(a->n_children);
  for (int64_t i = 0; i < a->n_children; ++i) {
    const ArrowArray* c = a->children[i];
    const ArrowSchema* cs = s->children[i];
    AB_REQUIRE(c && cs, ARROYO_B200_INVALID_ARGUMENT, "null child");
    if (!format_is_64bit(cs->format)) {
      throw Error(ARROYO_B200_UNSUPPORTED, std::string("column ") + (cs->name ? cs->name : "?") +
                                               ": unsupported type '" + (cs->format ? cs->format : "") +
                                               "' (supported: l, L, g, tsn:)");
    }
    AB_REQUIRE(c->length >= a->length + a->offset, ARROYO_B200_INVALID_ARGUMENT, "child shorter than batch");
    AB_REQUIRE(c->n_buffers == 2, ARROYO_B200_INVALID_ARGUMENT, "primitive column must have 2 buffers");
    InColumn ic;
    if (i == nullable_col) {
      if (c->null_count != 0 && c->buffers[0] != nullptr) {
        ic.validity = (const uint8_t*)c->buffers[0];
        ic.validity_bit = c->offset + a->offset;
      }
    } else if (c->null_count != 0 && c->buffers[0] != nullptr) {
      // null_count may be -1 (unknown): count the zero validity bits of the logical range.
      int64_t nulls = c->null_count;
      if (nulls < 0) {
        const uint8_t* v = (const uint8_t*)c->buffers[0];
        nulls = 0;
        for (int64_t r = 0; r < a->length; ++r) {
          int64_t bit = c->offset + a->offset + r;
          if (!((v[bit >> 3] >> (bit & 7)) & 1)) ++nulls;
        }
      }
      if (nulls > 0)
        throw Error(ARROYO_B200_UNSUPPORTED, std::string("column ") + (cs->name ? cs->name : "?") +
                                                 " has nulls: NULL keys/values are outside the supported subset");
    }
    AB_REQUIRE(a->length == 0 || c->buffers[1] != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null data buffer");
    ic.data = (const uint64_t*)c->buffers[1] + c->offset + a->offset;
    ic.format = cs->format;
    cols.push_back(ic);
  }
  *n_rows = a->length;
  return cols;
}

// The aggregating operators compute sum / avg / min / max of Int64 columns grouped by an Int64, UInt64 or
// timestamp[ns] key (INTEGRATION.md §1).  Any other input type is refused, so the plan stays on the stock operator
// instead of being aggregated with signed-integer arithmetic over the wrong bits.  key_col < 0: unkeyed.
inline void require_aggregate_input_types(const std::vector<InColumn>& cols, int key_col, const int* val_cols,
                                          int n_vals) {
  if (key_col >= 0) {
    const std::string& f = cols[key_col].format;
    if (f != "l" && f != "L" && f.compare(0, 4, "tsn:") != 0)
      throw Error(ARROYO_B200_UNSUPPORTED, "group-by key of type '" + f + "' (supported: l, L, tsn:)");
  }
  for (int v = 0; v < n_vals; ++v) {
    const std::string& f = cols[val_cols[v]].format;
    if (f != "l")
      throw Error(ARROYO_B200_UNSUPPORTED, "aggregate input of type '" + f + "' (only Int64 'l' is supported)");
  }
}

// ---- export -------------------------------------------------------------------------------
struct OutColumn {
  std::string name;
  std::string format;               // "l", "g", "tsn:", or "+s" for a struct of children
  void* data = nullptr;             // pinned buffer from PinnedPool (ownership moves to the array)
  std::vector<OutColumn> children;  // struct only
  bool nullable = false;
  void* validity = nullptr;         // optional pinned validity bitmap
  int64_t null_count = 0;
};

namespace detail {
struct ArrayPriv {
  std::vector<const void*> buffers;
  std::vector<ArrowArray> child_storage;
  std::vector<ArrowArray*> child_ptrs;
  std::vector<void*> owned;  // pinned buffers to give back
};
struct SchemaPriv {
  std::string format, name;
  std::vector<ArrowSchema> child_storage;
  std::vector<ArrowSchema*> child_ptrs;
};

inline void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  auto* p = (ArrayPriv*)a->private_data;
  for (auto& c : p->child_storage)
    if (c.release) c.release(&c);
  for (void* b : p->owned) PinnedPool::get().free(b);
  delete p;
  a->release = nullptr;
}
inline void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  auto* p = (SchemaPriv*)s->private_data;
  for (auto& c : p->child_storage)
    if (c.release) c.release(&c);
  delete p;
  s->release = nullptr;
}

inline void fill_array(const OutColumn& col, int64_t n_rows, ArrowArray* out) {
  auto* p = new ArrayPriv();
  memset(out, 0, sizeof *out);
  out->length = n_rows;
  out->null_count = col.null_count;
  out->offset = 0;
  if (col.format == "+s") {
    p->buffers = {nullptr};
    p->child_storage.resize(col.children.size());
    for (size_t i = 0; i < col.children.size(); ++i) {
      fill_array(col.children[i], n_rows, &p->child_storage[i]);
    }
    for (auto& c : p->child_storage) p->child_ptrs.push_back(&c);
  } else {
    p->buffers = {col.validity, col.data};
    if (col.data) p->owned.push_back(col.data);
    if (col.validity) p->owned.push_back(col.validity);
  }
  out->n_buffers = (int64_t)p->buffers.size();
  out->buffers = p->buffers.data();
  out->n_children = (int64_t)p->child_ptrs.size();
  out->children = p->child_ptrs.empty() ? nullptr : p->child_ptrs.data();
  out->dictionary = nullptr;
  out->release = release_array;
  out->private_data = p;
}

inline void fill_schema(const OutColumn& col, ArrowSchema* out) {
  auto* p = new SchemaPriv();
  memset(out, 0, sizeof *out);
  p->format = col.format;
  p->name = col.name;
  p->child_storage.resize(col.children.size());
  for (size_t i = 0; i < col.children.size(); ++i) fill_schema(col.children[i], &p->child_storage[i]);
  for (auto& c : p->child_storage) p->child_ptrs.push_back(&c);
  out->format = p->format.c_str();
  out->name = p->name.c_str();
  out->metadata = nullptr;
  out->flags = col.nullable ? ARROW_FLAG_NULLABLE : 0;
  out->n_children = (int64_t)p->child_ptrs.size();
  out->children = p->child_ptrs.empty() ? nullptr : p->child_ptrs.data();
  out->dictionary = nullptr;
  out->release = release_schema;
  out->private_data = p;
}
}  // namespace detail

// Exports columns as one record batch (struct array + struct schema).
inline void export_batch(const std::vector<OutColumn>& cols, int64_t n_rows, ArrowArray* arr, ArrowSchema* sch) {
  OutColumn root;
  root.name = "";
  root.format = "+s";
  root.children = cols;
  detail::fill_array(root, n_rows, arr);
  detail::fill_schema(root, sch);
}

// Storage behind an ArroyoB200Batches value.
struct BatchesPriv {
  std::vector<ArrowArray> arrays;
  std::vector<ArrowSchema> schemas;
};

inline void batches_finish(BatchesPriv* p, ArroyoB200Batches* out) {
  out->n_batches = (int64_t)p->arrays.size();
  out->arrays = p->arrays.empty() ? nullptr : p->arrays.data();
  out->schemas = p->schemas.empty() ? nullptr : p->schemas.data();
  out->private_data = p;
}

// Device-to-host copy of `bytes` into a pooled pinned buffer (8 bytes at least, so an empty column still owns one),
// enqueued on `s`; `*d2h_bytes` counts the bytes copied.
inline void* d2h_pinned(const void* dev, size_t bytes, cudaStream_t s, uint64_t* d2h_bytes) {
  void* h = PinnedPool::get().alloc(std::max<size_t>(bytes, 8));
  if (bytes) AB_CUDA(cudaMemcpyAsync(h, dev, bytes, cudaMemcpyDeviceToHost, s));
  *d2h_bytes += bytes;
  return h;
}

// Appends the windowed output batch of the window and session aggregates to `out`: the columns `[key?, aggs...]`
// with the `window{start, end}` struct inserted at `window_pos` (no struct when `wstart` is null), then `_timestamp`
// (arroyo-planner extension/aggregate.rs:306-389).  `key` is null when the operator is unkeyed.  The columns are
// copied on `s`: nothing may read the batch before `s` has passed the copies.
inline void export_window_batch(BatchesPriv* out, int64_t n, cudaStream_t s, uint64_t* d2h_bytes, const void* key,
                                const std::string& key_format, const DevBuf* aggs,
                                const std::vector<std::string>& agg_formats, const void* wstart, const void* wend,
                                int window_pos, const void* ts) {
  auto column = [&](const std::string& name, const std::string& format, const void* dev) {
    OutColumn c;
    c.name = name;
    c.format = format;
    c.data = d2h_pinned(dev, (size_t)n * 8, s, d2h_bytes);
    return c;
  };
  std::vector<OutColumn> cols;
  if (key) cols.push_back(column("key", key_format, key));
  for (size_t g = 0; g < agg_formats.size(); ++g)
    cols.push_back(column("agg" + std::to_string(g), agg_formats[g], aggs[g].p));
  if (wstart) {
    OutColumn w;
    w.name = "window";
    w.format = "+s";
    w.children = {column("start", "tsn:", wstart), column("end", "tsn:", wend)};
    cols.insert(cols.begin() + window_pos, w);
  }
  cols.push_back(column("_timestamp", "tsn:", ts));
  out->arrays.emplace_back();
  out->schemas.emplace_back();
  export_batch(cols, n, &out->arrays.back(), &out->schemas.back());
}

// Releases every batch of `p`, and `p` itself: batches that never reach the caller.
inline void discard(BatchesPriv* p) {
  for (auto& a : p->arrays)
    if (a.release) a.release(&a);
  for (auto& s : p->schemas)
    if (s.release) s.release(&s);
  delete p;
}

inline void batches_release(ArroyoB200Batches* b) {
  if (!b || !b->private_data) return;
  discard((BatchesPriv*)b->private_data);
  b->n_batches = 0;
  b->arrays = nullptr;
  b->schemas = nullptr;
  b->private_data = nullptr;
}

// Host input batches the library has taken and holds until the stream has passed the copies that read them.  The
// owner drains its streams before this is destroyed, which releases whatever is still held.
class HeldInputs {
 public:
  HeldInputs() = default;
  HeldInputs(const HeldInputs&) = delete;
  HeldInputs& operator=(const HeldInputs&) = delete;
  ~HeldInputs() {
    for (auto& a : taken_)
      if (a.release) a.release(&a);
    for (auto& g : sealed_) {
      for (auto& a : g.batches)
        if (a.release) a.release(&a);
      cudaEventDestroy(g.ev);
    }
    for (cudaEvent_t e : pool_) cudaEventDestroy(e);
  }

  // Takes `batch` (its `release` is set to NULL).  It is held from the next seal() on.
  void take(ArrowArray* batch) {
    taken_.push_back(*batch);
    batch->release = nullptr;
  }
  size_t n_unsealed() const { return taken_.size(); }

  // Holds every batch taken since the last seal until `s` has passed the work enqueued on it so far: one event for
  // all of them, taken from a pool.
  void seal(cudaStream_t s) {
    if (taken_.empty()) return;
    if (pool_.empty()) {
      cudaEvent_t e;
      AB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      pool_.push_back(e);
    }
    AB_CUDA(cudaEventRecord(pool_.back(), s));
    sealed_.push_back({pool_.back(), std::move(taken_)});
    pool_.pop_back();
    taken_.clear();
  }

  // Takes `batch` until `s` has passed the work enqueued on it so far.
  void hold(ArrowArray* batch, cudaStream_t s) {
    take(batch);
    seal(s);
  }

  // Releases, in the order they were sealed, the batches whose copies have completed; with `wait`, every sealed one.
  void release(bool wait) {
    while (!sealed_.empty()) {
      Sealed& g = sealed_.front();
      if (wait) {
        AB_CUDA(cudaEventSynchronize(g.ev));
      } else {
        const cudaError_t e = cudaEventQuery(g.ev);
        if (e == cudaErrorNotReady) break;
        AB_CUDA(e);
      }
      for (auto& a : g.batches)
        if (a.release) a.release(&a);
      pool_.push_back(g.ev);
      sealed_.pop_front();
    }
  }

 private:
  struct Sealed {
    cudaEvent_t ev;
    std::vector<ArrowArray> batches;
  };
  std::vector<ArrowArray> taken_;  // taken since the last seal
  std::deque<Sealed> sealed_;
  std::vector<cudaEvent_t> pool_;  // recorded events whose batches have been released
};

}  // namespace ab
