/*
 * window_oracle.c -- CPU restatement (plain C) of the reference's tumbling / sliding window aggregate.
 * TEST INFRASTRUCTURE ONLY: used as the checker at sizes the numpy oracle cannot reach and as the timed
 * CPU baseline ("port") of bench.py.  Nothing under arroyo_b200/ links or calls this file.
 *
 * It follows the reference's algorithm step by step, not the GPU design:
 *   process_batch   bin = ts - ts % slide            (date_bin, planner builder.rs:201-224)
 *                   sort rows by bin, gather every column, partition into bin ranges
 *                                                    (sliding_aggregating_window.rs:604-625)
 *                   drop ranges with bin < bin(watermark)                         (:631-633)
 *                   feed each range to that pane's Partial hash aggregate         (:650-671)
 *   advance         close pane, insert its partial rows into the window store, take ALL panes in
 *                   [bin_end - width, bin_end), Final-merge them through a fresh hash aggregate,
 *                   project window.start/end and _timestamp = end - 1             (:115-222)
 *   tumbling        same with one pane per window (tumbling_aggregating_window.rs:250-392)
 * State machine (NoData / OnlyBufferedData / InMemoryData, state-table keys) as in :63-113, :176-187 and
 * arroyo-state/src/tables/expiring_time_key_map.rs:833-929.
 *
 * Accumulators (DataFusion 48 semantics, dep-knowledge): rows (COUNT(*) / AVG count), sum i64 wrapping,
 * sum f64 of inputs cast to f64 (AVG), min/max i64.
 *
 * The parallel driver mirrors the reference's dataflow: source-side subtasks hash-partition every
 * batch by key (ArrowCollector::repartition, arroyo-operator/src/context.rs:506-541) and `p` window
 * subtasks each own one partition; every subtask is single threaded, as a tokio task is.
 */
#define _GNU_SOURCE
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include <unistd.h>

#define NO_TIME INT64_MIN

static inline uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

static inline int64_t bin_start(int64_t ts, int64_t w) {  /* floor: a negative watermark bins below zero */
  if (w == 0) return ts;
  int64_t r = ts % w;
  return ts - (r < 0 ? r + w : r);
}

/* ---------------- group hash table (key -> accumulators) ---------------- */
typedef struct {
  int64_t key;
  int64_t rows; /* 0 = empty slot */
  int64_t sum;
  double fsum;
  int64_t mn, mx;
} Entry;

typedef struct {
  Entry* e;
  uint64_t cap, count;
} Table;

static void table_init(Table* t, uint64_t cap) {
  t->cap = cap;
  t->count = 0;
  t->e = (Entry*)calloc(cap, sizeof(Entry));
}
static void table_free(Table* t) {
  free(t->e);
  t->e = NULL;
  t->cap = t->count = 0;
}
static Entry* table_slot(Table* t, int64_t key);
static void table_grow(Table* t) {
  Table n;
  table_init(&n, t->cap * 2);
  for (uint64_t i = 0; i < t->cap; ++i)
    if (t->e[i].rows) {
      Entry* d = table_slot(&n, t->e[i].key);
      *d = t->e[i];
      n.count++;
    }
  free(t->e);
  *t = n;
}
/* returns the slot for key (either occupied by key or empty) */
static Entry* table_slot(Table* t, int64_t key) {
  uint64_t m = t->cap - 1, p = mix64((uint64_t)key) & m;
  while (t->e[p].rows && t->e[p].key != key) p = (p + 1) & m;
  return &t->e[p];
}
static inline Entry* table_upsert(Table* t, int64_t key) {
  if ((t->count + 1) * 2 > t->cap) table_grow(t);
  Entry* s = table_slot(t, key);
  if (!s->rows) {
    s->key = key;
    s->sum = 0;
    s->fsum = 0.0;
    s->mn = INT64_MAX;
    s->mx = INT64_MIN;
    t->count++;
  }
  return s;
}

/* ---------------- operator ---------------- */
typedef struct {
  int64_t bin;
  Table partial;
  int in_tier;   /* inserted into the window store (TieredRecordBatchHolder) */
  int active;    /* rows since last drain */
} Pane;

typedef struct {
  int64_t* v;
  size_t n, cap;
} I64Set; /* small sorted set */

static void set_insert(I64Set* s, int64_t x) {
  size_t i = 0;
  while (i < s->n && s->v[i] < x) ++i;
  if (i < s->n && s->v[i] == x) return;
  if (s->n == s->cap) {
    s->cap = s->cap ? s->cap * 2 : 16;
    s->v = (int64_t*)realloc(s->v, s->cap * sizeof(int64_t));
  }
  memmove(s->v + i + 1, s->v + i, (s->n - i) * sizeof(int64_t));
  s->v[i] = x;
  s->n++;
}
static int set_erase(I64Set* s, int64_t x) {
  for (size_t i = 0; i < s->n; ++i)
    if (s->v[i] == x) {
      memmove(s->v + i, s->v + i + 1, (s->n - i - 1) * sizeof(int64_t));
      s->n--;
      return 1;
    }
  return 0;
}
static void set_erase_below(I64Set* s, int64_t cutoff) {
  size_t i = 0;
  while (i < s->n && s->v[i] < cutoff) ++i;
  memmove(s->v, s->v + i, (s->n - i) * sizeof(int64_t));
  s->n -= i;
}

typedef struct {
  int64_t *key, *wstart, *wend, *rows, *sum, *mn, *mx, *ts;
  double* avg;
  int64_t n, cap;
} OracleOut;

static void out_reserve(OracleOut* o, int64_t extra) {
  if (o->n + extra <= o->cap) return;
  int64_t c = o->cap ? o->cap : 1024;
  while (c < o->n + extra) c *= 2;
#define GROW(f, T) o->f = (T*)realloc(o->f, (size_t)c * sizeof(T))
  GROW(key, int64_t); GROW(wstart, int64_t); GROW(wend, int64_t); GROW(rows, int64_t); GROW(sum, int64_t);
  GROW(mn, int64_t); GROW(mx, int64_t); GROW(ts, int64_t); GROW(avg, double);
#undef GROW
  o->cap = c;
}

enum { ST_NO_DATA = 0, ST_ONLY_BUFFERED = 1, ST_IN_MEMORY = 2 };

typedef struct OracleOp {
  int sliding, keyed, want_minmax, final_projection;
  int64_t width, slide;
  Pane* panes; /* unordered list of live panes (execs + window store) */
  size_t n_panes, cap_panes;
  int state;
  int64_t state_t;
  I64Set flushed, to_flush; /* keys of state table "t" */
  /* scratch for process_batch */
  int64_t *bins, *sk, *sv, *st;
  uint32_t* idx;
  int64_t scratch_cap;
  uint64_t late_rows;
} OracleOp;

OracleOp* oracle_window_create(int64_t width, int64_t slide, int keyed, int want_minmax, int final_projection) {
  OracleOp* op = (OracleOp*)calloc(1, sizeof(OracleOp));
  op->sliding = slide > 0;
  op->width = width;
  op->slide = slide > 0 ? slide : width;
  op->keyed = keyed;
  op->want_minmax = want_minmax;
  op->final_projection = final_projection;
  return op;
}

void oracle_window_destroy(OracleOp* op) {
  if (!op) return;
  for (size_t i = 0; i < op->n_panes; ++i) table_free(&op->panes[i].partial);
  free(op->panes);
  free(op->flushed.v);
  free(op->to_flush.v);
  free(op->bins); free(op->sk); free(op->sv); free(op->st); free(op->idx);
  free(op);
}

uint64_t oracle_window_late_rows(const OracleOp* op) { return op->late_rows; }

static Pane* find_pane(OracleOp* op, int64_t bin) {
  for (size_t i = 0; i < op->n_panes; ++i)
    if (op->panes[i].bin == bin) return &op->panes[i];
  return NULL;
}
static Pane* get_pane(OracleOp* op, int64_t bin) {
  Pane* p = find_pane(op, bin);
  if (p) return p;
  if (op->n_panes == op->cap_panes) {
    op->cap_panes = op->cap_panes ? op->cap_panes * 2 : 32;
    op->panes = (Pane*)realloc(op->panes, op->cap_panes * sizeof(Pane));
  }
  p = &op->panes[op->n_panes++];
  p->bin = bin;
  p->in_tier = 0;
  p->active = 0;
  table_init(&p->partial, 1024);
  return p;
}
static void drop_pane(OracleOp* op, Pane* p) {
  table_free(&p->partial);
  *p = op->panes[--op->n_panes];
}

static int cmp_bin_idx(const void* a, const void* b, void* ctx) {
  const int64_t* bins = (const int64_t*)ctx;
  uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
  if (bins[x] != bins[y]) return bins[x] < bins[y] ? -1 : 1;
  return x < y ? -1 : (x > y);
}

/* state-table (ExpiringTimeKeyView) keys */
static void tbl_flush(OracleOp* op, int has_wm, int64_t wm) {
  for (size_t i = 0; i < op->to_flush.n; ++i) {
    int64_t t = op->to_flush.v[i];
    if (has_wm && t < wm - op->width) continue;
    set_insert(&op->flushed, t);
  }
  op->to_flush.n = 0;
  if (has_wm) set_erase_below(&op->flushed, wm - op->width);
}
static int tbl_min(OracleOp* op, int64_t* out) {
  int any = 0;
  int64_t m = INT64_MAX;
  if (op->flushed.n) { m = op->flushed.v[0]; any = 1; }
  if (op->to_flush.n && (!any || op->to_flush.v[0] < m)) { m = op->to_flush.v[0]; any = 1; }
  *out = m;
  return any;
}

/* ArrowOperator::process_batch.  key may be NULL when !keyed; val may be NULL (COUNT only). */
void oracle_window_process_batch(OracleOp* op, const int64_t* key, const int64_t* val, const int64_t* ts, int64_t n,
                                 int has_wm, int64_t wm) {
  if (n <= 0) return;
  if (n > op->scratch_cap) {
    op->scratch_cap = n;
    op->bins = (int64_t*)realloc(op->bins, (size_t)n * 8);
    op->sk = (int64_t*)realloc(op->sk, (size_t)n * 8);
    op->sv = (int64_t*)realloc(op->sv, (size_t)n * 8);
    op->st = (int64_t*)realloc(op->st, (size_t)n * 8);
    op->idx = (uint32_t*)realloc(op->idx, (size_t)n * 4);
  }
  const int64_t w = op->slide;
  int64_t bmin = INT64_MAX, bmax = INT64_MIN;
  for (int64_t i = 0; i < n; ++i) {
    int64_t b = ts[i] - ts[i] % w; /* K1 date_bin */
    op->bins[i] = b;
    if (b < bmin) bmin = b;
    if (b > bmax) bmax = b;
  }
  /* K2 sort_to_indices: O(n) counting sort when the batch spans few panes (arrow-rs uses an unstable
   * comparison sort; this is at least as fast), comparison sort otherwise */
  int64_t span = (bmax - bmin) / w + 1;
  if (span <= 256) {
    uint32_t cnt[257];
    memset(cnt, 0, sizeof cnt);
    for (int64_t i = 0; i < n; ++i) cnt[(op->bins[i] - bmin) / w + 1]++;
    for (int s = 0; s < 256; ++s) cnt[s + 1] += cnt[s];
    for (int64_t i = 0; i < n; ++i) op->idx[cnt[(op->bins[i] - bmin) / w]++] = (uint32_t)i;
  } else {
    for (int64_t i = 0; i < n; ++i) op->idx[i] = (uint32_t)i;
    qsort_r(op->idx, (size_t)n, sizeof(uint32_t), cmp_bin_idx, op->bins);
  }
  /* take(): gather every column */
  for (int64_t i = 0; i < n; ++i) {
    uint32_t j = op->idx[i];
    if (op->keyed) op->sk[i] = key[j];
    if (val) op->sv[i] = val[j];
    op->st[i] = op->bins[j];
  }
  const int64_t late_bin = has_wm ? bin_start(wm, w) : INT64_MIN;
  /* partition() ranges */
  int64_t s = 0;
  while (s < n) {
    int64_t b = op->st[s], e = s + 1;
    while (e < n && op->st[e] == b) ++e;
    if (has_wm && b < late_bin) {
      op->late_rows += (uint64_t)(e - s);
      s = e;
      continue;
    }
    if (op->sliding) {
      if (op->state == ST_NO_DATA) { op->state = ST_ONLY_BUFFERED; op->state_t = b; }
      else if (op->state == ST_ONLY_BUFFERED && b < op->state_t) op->state_t = b;
    }
    Pane* p = get_pane(op, b);
    p->active = 1;
    /* K3 AggregateExec(Partial): group hash insert + accumulate */
    Table* t = &p->partial;
    for (int64_t i = s; i < e; ++i) {
      Entry* en = table_upsert(t, op->keyed ? op->sk[i] : 0);
      en->rows++;
      if (val) {
        int64_t v = op->sv[i];
        en->sum = (int64_t)((uint64_t)en->sum + (uint64_t)v);
        en->fsum += (double)v;
        if (op->want_minmax) {
          if (v < en->mn) en->mn = v;
          if (v > en->mx) en->mx = v;
        }
      }
    }
    s = e;
  }
}

/* K4 Final merge of the panes in [a, b) + K5 projection */
static void emit_window(OracleOp* op, int64_t a, int64_t b, OracleOut* out) {
  Table fin;
  int have = 0;
  /* ascending pane order, like batches_for_interval (:369-412) */
  for (int64_t cur = a; cur < b; cur += op->slide) {
    Pane* p = find_pane(op, cur);
    if (!p || !p->in_tier) continue;
    if (!have) {
      table_init(&fin, 1024);
      have = 1;
    }
    for (uint64_t i = 0; i < p->partial.cap; ++i) {
      Entry* s = &p->partial.e[i];
      if (!s->rows) continue;
      Entry* d = table_upsert(&fin, s->key);
      d->rows += s->rows;
      d->sum = (int64_t)((uint64_t)d->sum + (uint64_t)s->sum);
      d->fsum += s->fsum;
      if (s->mn < d->mn) d->mn = s->mn;
      if (s->mx > d->mx) d->mx = s->mx;
    }
  }
  if (!have) return;
  out_reserve(out, (int64_t)fin.count);
  const int64_t tstamp = op->final_projection ? b - 1 : a;
  for (uint64_t i = 0; i < fin.cap; ++i) {
    Entry* s = &fin.e[i];
    if (!s->rows) continue;
    int64_t o = out->n++;
    out->key[o] = s->key;
    out->wstart[o] = a;
    out->wend[o] = b;
    out->rows[o] = s->rows;
    out->sum[o] = s->sum;
    out->avg[o] = s->fsum / (double)(uint64_t)s->rows;
    out->mn[o] = s->mn;
    out->mx[o] = s->mx;
    out->ts[o] = tstamp;
  }
  table_free(&fin);
}

static int sliding_should_advance(OracleOp* op, int64_t wm) {
  if (op->state == ST_NO_DATA) return 0;
  return (__int128)op->state_t + op->slide <= (__int128)bin_start(wm, op->slide);
}

static void sliding_advance(OracleOp* op, OracleOut* out) {
  int64_t b = op->state_t, bin_end = b + op->slide;
  tbl_flush(op, 1, bin_end);
  Pane* p = find_pane(op, b);
  if (p && !p->in_tier) {
    if (p->active) set_insert(&op->to_flush, b);
    p->active = 0;
    p->in_tier = 1;
  }
  /* flush_timestamp(bin_end) */
  if (set_erase(&op->to_flush, bin_end)) set_insert(&op->flushed, bin_end);
  /* expire_timestamp: the pane that has just left (the reference expires bin_end - width + slide, the oldest pane of the
     NEXT window, which its tier still holds; see oracle/arroyo_oracle.py) */
  set_erase(&op->flushed, bin_end - op->width);
  set_erase(&op->to_flush, bin_end - op->width);
  emit_window(op, bin_end - op->width, bin_end, out);
  /* delete_before(bin_end + slide - width) */
  int64_t cutoff = bin_start(bin_end + op->slide - op->width, op->slide);
  int tier_empty = 1;
  for (size_t i = 0; i < op->n_panes;) {
    Pane* q = &op->panes[i];
    if (q->in_tier && q->bin < cutoff) {
      drop_pane(op, q);
      continue;
    }
    if (q->in_tier) tier_empty = 0;
    ++i;
  }
  if (tier_empty) {
    /* panes still pending (not in the tier) are candidates as well as the table: the reference looks only at the
       table and would never emit rows that arrived while the store was non-empty and were not checkpointed */
    int64_t mt;
    int has = tbl_min(op, &mt);
    for (size_t i = 0; i < op->n_panes; ++i) {
      const Pane* q = &op->panes[i];
      if (!q->in_tier && (!has || q->bin < mt)) { mt = q->bin; has = 1; }
    }
    if (has) { op->state = ST_ONLY_BUFFERED; op->state_t = bin_start(mt, op->slide); }
    else op->state = ST_NO_DATA;
  } else {
    op->state = ST_IN_MEMORY;
    op->state_t = bin_end;
  }
}

/* ArrowOperator::handle_watermark; appends emitted rows to `out`. */
void oracle_window_handle_watermark(OracleOp* op, int64_t wm, OracleOut* out) {
  if (op->sliding) {
    while (sliding_should_advance(op, wm)) sliding_advance(op, out);
    return;
  }
  int64_t wbin = bin_start(wm, op->width);
  for (;;) {
    Pane* first = NULL;
    for (size_t i = 0; i < op->n_panes; ++i)
      if (!first || op->panes[i].bin < first->bin) first = &op->panes[i];
    if (!first || !(first->bin < wbin)) break;
    first->in_tier = 1;
    emit_window(op, first->bin, first->bin + op->width, out);
    drop_pane(op, find_pane(op, first->bin));
  }
}

/* ArrowOperator::handle_checkpoint: control-flow effect only (state-table keys). */
void oracle_window_handle_checkpoint(OracleOp* op, int has_wm, int64_t wm) {
  if (!op->sliding) return;
  for (size_t i = 0; i < op->n_panes; ++i) {
    Pane* p = &op->panes[i];
    if (p->in_tier || !p->active) continue;
    p->active = 0;
    set_insert(&op->to_flush, p->bin);
  }
  tbl_flush(op, has_wm, wm);
}

OracleOut* oracle_out_create(void) { return (OracleOut*)calloc(1, sizeof(OracleOut)); }
void oracle_out_clear(OracleOut* o) { o->n = 0; }
void oracle_out_destroy(OracleOut* o) {
  if (!o) return;
  free(o->key); free(o->wstart); free(o->wend); free(o->rows); free(o->sum); free(o->mn); free(o->mx); free(o->ts);
  free(o->avg);
  free(o);
}

/* ---------------- parallel driver (CPU baseline) ---------------- */
static double now_s(void) {
  struct timespec t;
  clock_gettime(CLOCK_MONOTONIC, &t);
  return (double)t.tv_sec + 1e-9 * (double)t.tv_nsec;
}

typedef struct {
  double seconds;
  uint64_t rows_in, rows_out, windows_out, late_rows;
  uint64_t sum_of_sums;  /* wrapping checksum over emitted rows */
  uint64_t sum_of_rows;
  double sum_of_avgs;
  int threads;
} OracleRunResult;

int oracle_max_threads(void) {
  long n = sysconf(_SC_NPROCESSORS_ONLN);
  return n > 0 ? (int)n : 1;
}

/* fork-join over a persistent pool: the workers are created once per process and parked on a condition
 * variable between calls (a thread per call and worker cost ~1 000 pthread_create per pane and made the CPU
 * figure pessimistic).  Items are claimed from a shared counter. */
typedef struct {
  void (*fn)(int64_t item, void* ctx);
  void* ctx;
  int64_t n;
  int64_t next;
} ParFor;

#define POOL_MAX 1024
static struct {
  pthread_mutex_t mu;
  pthread_cond_t go, done;
  pthread_t th[POOL_MAX];
  int n_threads;      /* workers created so far */
  int want;           /* workers that take part in the current job */
  uint64_t gen;       /* job generation */
  int running;        /* workers still inside the current job */
  ParFor* job;
} g_pool = {PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, PTHREAD_COND_INITIALIZER, {0}, 0, 0, 0, 0, NULL};

static void parfor_drain(ParFor* pf) {
  for (;;) {
    int64_t i = __atomic_fetch_add(&pf->next, 1, __ATOMIC_RELAXED);
    if (i >= pf->n) break;
    pf->fn(i, pf->ctx);
  }
}

static void* pool_worker(void* arg) {
  const int me = (int)(intptr_t)arg;
  uint64_t seen = 0;
  pthread_mutex_lock(&g_pool.mu);
  for (;;) {
    while (g_pool.gen == seen) pthread_cond_wait(&g_pool.go, &g_pool.mu);
    seen = g_pool.gen;
    if (me >= g_pool.want) continue;
    ParFor* pf = g_pool.job;
    pthread_mutex_unlock(&g_pool.mu);
    parfor_drain(pf);
    pthread_mutex_lock(&g_pool.mu);
    if (--g_pool.running == 0) pthread_cond_signal(&g_pool.done);
  }
  return NULL;
}

static void parallel_for(int64_t n, int threads, void (*fn)(int64_t, void*), void* ctx) {
  ParFor pf = {fn, ctx, n, 0};
  if (threads > n) threads = (int)n;
  if (threads > POOL_MAX) threads = POOL_MAX;
  if (threads <= 1) {
    parfor_drain(&pf);
    return;
  }
  const int helpers = threads - 1;  /* the caller works too */
  pthread_mutex_lock(&g_pool.mu);
  while (g_pool.n_threads < helpers) {
    pthread_create(&g_pool.th[g_pool.n_threads], NULL, pool_worker, (void*)(intptr_t)g_pool.n_threads);
    pthread_detach(g_pool.th[g_pool.n_threads]);
    ++g_pool.n_threads;
  }
  g_pool.job = &pf;
  g_pool.want = helpers;
  g_pool.running = helpers;
  ++g_pool.gen;
  pthread_cond_broadcast(&g_pool.go);
  pthread_mutex_unlock(&g_pool.mu);
  parfor_drain(&pf);
  pthread_mutex_lock(&g_pool.mu);
  while (g_pool.running > 0) pthread_cond_wait(&g_pool.done, &g_pool.mu);
  pthread_mutex_unlock(&g_pool.mu);
}

typedef struct {
  const int64_t *key, *val, *ts;
  int64_t n_rows, batch_rows, b0, nb;
  int p;
  uint64_t range;
  int64_t *pk, *pv, *pt, *off, *wm_of;
  OracleOp** ops;
  OracleOut** outs;
  int has_wm;
  int64_t cur_wm;
} RunCtx;

/* repartition (context.rs:506-541): hash -> dest -> bucket the rows of one batch */
static void partition_batch(int64_t r, void* vctx) {
  RunCtx* c = (RunCtx*)vctx;
  const int p = c->p;
  int64_t s = (c->b0 + r) * c->batch_rows, e = s + c->batch_rows < c->n_rows ? s + c->batch_rows : c->n_rows;
  int64_t* o = c->off + r * (p + 1);
  int64_t cnt[1025];
  memset(cnt, 0, sizeof(int64_t) * (size_t)(p + 1));
  for (int64_t i = s; i < e; ++i) cnt[(mix64((uint64_t)c->key[i]) / c->range) % (uint64_t)p + 1]++;
  for (int d = 0; d < p; ++d) cnt[d + 1] += cnt[d];
  memcpy(o, cnt, sizeof(int64_t) * (size_t)(p + 1));
  int64_t base = r * c->batch_rows;
  for (int64_t i = s; i < e; ++i) {
    int d = (int)((mix64((uint64_t)c->key[i]) / c->range) % (uint64_t)p);
    int64_t q = base + cnt[d]++;
    c->pk[q] = c->key[i];
    c->pv[q] = c->val[i];
    c->pt[q] = c->ts[i];
  }
}

/* one window subtask consumes its slice of every batch of the round, in order */
static void run_subtask(int64_t d, void* vctx) {
  RunCtx* c = (RunCtx*)vctx;
  int sub_has_wm = c->has_wm;
  int64_t sub_wm = c->cur_wm;
  for (int64_t r = 0; r < c->nb; ++r) {
    int64_t* o = c->off + r * (c->p + 1);
    int64_t base = r * c->batch_rows;
    oracle_window_process_batch(c->ops[d], c->pk + base + o[d], c->pv + base + o[d], c->pt + base + o[d],
                                o[d + 1] - o[d], sub_has_wm, sub_wm);
    if (c->wm_of[r] != NO_TIME) {
      sub_has_wm = 1;
      sub_wm = c->wm_of[r];
      oracle_window_handle_watermark(c->ops[d], sub_wm, c->outs[d]);
    }
  }
}

static void final_flush(int64_t d, void* vctx) {
  RunCtx* c = (RunCtx*)vctx;
  oracle_window_handle_watermark(c->ops[d], INT64_MAX, c->outs[d]);
}

/* A resumable run: p key-partitioned window subtasks on p threads, fed any number of row chunks.
 * Watermarks: WatermarkGenerator rule (watermark_generator.rs:150-197) with delay `wm_delay`, interval 1 s.
 * slide == 0 => tumbling. */
/* checksums of one emitted window (all subtasks): what a GPU run of the same input is compared with */
typedef struct {
  int64_t wstart, wend;
  uint64_t rows_out;
  uint64_t sum_of_rows;  /* sum of COUNT(*) */
  uint64_t sum_of_sums;  /* wrapping sum of SUM(value) */
  double sum_of_avgs;
} OracleWindowSum;

typedef struct OracleRunner {
  RunCtx c;
  int64_t R;
  int64_t last_emitted_at;
  int64_t wm_delay;
  OracleRunResult acc;
  OracleWindowSum* wins;
  int64_t n_wins, cap_wins;
} OracleRunner;

static OracleWindowSum* runner_window(OracleRunner* r, int64_t wstart, int64_t wend) {
  for (int64_t i = r->n_wins - 1; i >= 0; --i)
    if (r->wins[i].wstart == wstart) return &r->wins[i];
  if (r->n_wins == r->cap_wins) {
    r->cap_wins = r->cap_wins ? r->cap_wins * 2 : 64;
    r->wins = (OracleWindowSum*)realloc(r->wins, (size_t)r->cap_wins * sizeof(OracleWindowSum));
  }
  OracleWindowSum* w = &r->wins[r->n_wins++];
  memset(w, 0, sizeof *w);
  w->wstart = wstart;
  w->wend = wend;
  return w;
}

OracleRunner* oracle_runner_create(int p, int64_t width, int64_t slide, int64_t wm_delay, int64_t batch_rows) {
  if (p < 1 || p > 1024 || batch_rows < 1) return NULL;
  OracleRunner* r = (OracleRunner*)calloc(1, sizeof(OracleRunner));
  RunCtx* c = &r->c;
  r->R = 64;
  c->p = p;
  c->batch_rows = batch_rows;
  c->range = UINT64_MAX / (uint64_t)p;
  c->ops = (OracleOp**)calloc((size_t)p, sizeof(OracleOp*));
  c->outs = (OracleOut**)calloc((size_t)p, sizeof(OracleOut*));
  for (int i = 0; i < p; ++i) {
    c->ops[i] = oracle_window_create(width, slide, 1, 0, 1);
    c->outs[i] = oracle_out_create();
  }
  c->pk = (int64_t*)malloc((size_t)(r->R * batch_rows) * 8);
  c->pv = (int64_t*)malloc((size_t)(r->R * batch_rows) * 8);
  c->pt = (int64_t*)malloc((size_t)(r->R * batch_rows) * 8);
  c->off = (int64_t*)malloc((size_t)(r->R * (p + 1)) * 8);
  c->wm_of = (int64_t*)malloc((size_t)r->R * 8);
  r->acc.threads = p;
  r->last_emitted_at = 0;
  r->wm_delay = wm_delay;
  return r;
}

static void runner_sink(OracleRunner* r) {
  RunCtx* c = &r->c;
  for (int d = 0; d < c->p; ++d) {
    OracleOut* o = c->outs[d];
    int64_t last_w = NO_TIME;
    OracleWindowSum* ws = NULL;
    for (int64_t i = 0; i < o->n; ++i) {
      r->acc.sum_of_sums += (uint64_t)o->sum[i];
      r->acc.sum_of_rows += (uint64_t)o->rows[i];
      r->acc.sum_of_avgs += o->avg[i];
      if (!ws || ws->wstart != o->wstart[i]) ws = runner_window(r, o->wstart[i], o->wend[i]);
      ws->rows_out += 1;
      ws->sum_of_rows += (uint64_t)o->rows[i];
      ws->sum_of_sums += (uint64_t)o->sum[i];
      ws->sum_of_avgs += o->avg[i];
      if (d == 0 && o->wstart[i] != last_w) { ++r->acc.windows_out; last_w = o->wstart[i]; }
    }
    r->acc.rows_out += (uint64_t)o->n;
    o->n = 0;
  }
}

/* Feeds n_rows rows (cut into batches of batch_rows); returns the seconds this call took. */
double oracle_runner_feed(OracleRunner* r, const int64_t* key, const int64_t* val, const int64_t* ts, int64_t n_rows) {
  RunCtx* c = &r->c;
  const int64_t wm_delay = r->wm_delay;
  const int64_t batch_rows = c->batch_rows;
  const int64_t n_batches = (n_rows + batch_rows - 1) / batch_rows;
  c->key = key; c->val = val; c->ts = ts; c->n_rows = n_rows;
  const double t0 = now_s();
  for (int64_t b0 = 0; b0 < n_batches; b0 += r->R) {
    const int64_t nb = (n_batches - b0) < r->R ? (n_batches - b0) : r->R;
    c->b0 = b0; c->nb = nb;
    /* watermark generator (source subtask): min/max per batch */
    for (int64_t q = 0; q < nb; ++q) {
      int64_t s = (b0 + q) * batch_rows, e = s + batch_rows < n_rows ? s + batch_rows : n_rows;
      int64_t mn = INT64_MAX, mx = INT64_MIN;
      for (int64_t i = s; i < e; ++i) {
        if (ts[i] < mn) mn = ts[i];
        if (ts[i] > mx) mx = ts[i];
      }
      int64_t d = mx - r->last_emitted_at;
      if (d < 0) d = 0;
      if (d > 1000000000ll) {
        r->last_emitted_at = mx;
        c->wm_of[q] = mn - wm_delay;
      } else {
        c->wm_of[q] = NO_TIME;
      }
    }
    parallel_for(nb, c->p, partition_batch, c);
    parallel_for(c->p, c->p, run_subtask, c);
    for (int64_t q = 0; q < nb; ++q)
      if (c->wm_of[q] != NO_TIME) {
        c->has_wm = 1;
        c->cur_wm = c->wm_of[q];
      }
    runner_sink(r);
  }
  const double dt = now_s() - t0;
  r->acc.seconds += dt;
  r->acc.rows_in += (uint64_t)n_rows;
  return dt;
}

/* end of data: final watermark flushes every window */
double oracle_runner_finish(OracleRunner* r) {
  const double t0 = now_s();
  parallel_for(r->c.p, r->c.p, final_flush, &r->c);
  runner_sink(r);
  const double dt = now_s() - t0;
  r->acc.seconds += dt;
  return dt;
}

void oracle_runner_result(OracleRunner* r, OracleRunResult* res) {
  *res = r->acc;
  uint64_t late = 0;
  for (int i = 0; i < r->c.p; ++i) late += r->c.ops[i]->late_rows;
  res->late_rows = late;
}

/* per-window checksums, in emission order; returns how many exist (copies at most `cap`) */
int64_t oracle_runner_windows(OracleRunner* r, OracleWindowSum* out, int64_t cap) {
  for (int64_t i = 0; i < r->n_wins && i < cap; ++i) out[i] = r->wins[i];
  return r->n_wins;
}

void oracle_runner_destroy(OracleRunner* r) {
  if (!r) return;
  free(r->wins);
  RunCtx* c = &r->c;
  for (int i = 0; i < c->p; ++i) {
    oracle_window_destroy(c->ops[i]);
    oracle_out_destroy(c->outs[i]);
  }
  free(c->ops); free(c->outs); free(c->pk); free(c->pv); free(c->pt); free(c->off); free(c->wm_of);
  free(r);
}

/* One-shot convenience wrapper. */
int oracle_run_windows(const int64_t* key, const int64_t* val, const int64_t* ts, int64_t n_rows, int64_t batch_rows,
                       int64_t width, int64_t slide, int64_t wm_delay, int p, int flush_at_end,
                       OracleRunResult* res) {
  OracleRunner* r = oracle_runner_create(p, width, slide, wm_delay, batch_rows);
  if (!r) return -1;
  oracle_runner_feed(r, key, val, ts, n_rows);
  if (flush_at_end) oracle_runner_finish(r);
  oracle_runner_result(r, res);
  oracle_runner_destroy(r);
  return 0;
}
