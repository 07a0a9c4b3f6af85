/*
 * dt_oracle.c -- CPU restatement of h2oai/datatable's DT[i, j, by(), sort()] hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (datatable_b200/) may
 * link, import or call this file; it is used by tests/, by
 * __graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference
 * legs as the *checker*, never as the thing measured or shipped.
 *
 * Parity status: PINNED.  tests/test_oracle_golden.py checks every function
 * here against fixtures under tests/golden/ that were produced by importing
 * the reference itself (built from its source tree, commit 3611640) with
 * tests/golden/make_golden.py, which also restates the reference's own
 * known-answer vectors (tests/ijby/test-sort.py, tests/test-groups.py,
 * tests/test-reduce.py).
 *
 * Each function cites the reference file:line it restates
 * (paths relative to the reference's src/core/).
 *
 * Plain C99 + pthreads.  Single-threaded by default (the parity tests); orc_set_threads(T)
 * lets bench.py's CPU legs use the host's cores the way the reference does (its radix sort
 * histograms and reorders chunk-parallel, sort.cc:904-1012, and its reducers are materialised
 * group-parallel, column/column_impl.cc:78-103).  Results do not depend on T: every parallel
 * region below is a static partition of the rows (or groups) with a deterministic combine.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <pthread.h>

/* ---- fork-join over T static parts ------------------------------------------------------- */
#define ORC_MAX_THREADS 256
static int g_threads = 1;
void orc_set_threads(int t) { g_threads = t < 1 ? 1 : (t > ORC_MAX_THREADS ? ORC_MAX_THREADS : t); }
int orc_get_threads(void) { return g_threads; }

typedef void (*part_fn)(int t, int T, void* ctx);
typedef struct { part_fn fn; void* ctx; int t, T; } part_arg;
static void* part_tramp(void* p) { part_arg* a = (part_arg*)p; a->fn(a->t, a->T, a->ctx); return NULL; }
static void par_run(int T, part_fn fn, void* ctx) {
  if (T <= 1) { fn(0, 1, ctx); return; }
  pthread_t th[ORC_MAX_THREADS]; part_arg arg[ORC_MAX_THREADS]; int started[ORC_MAX_THREADS];
  for (int t = 1; t < T; t++) {
    arg[t].fn = fn; arg[t].ctx = ctx; arg[t].t = t; arg[t].T = T;
    started[t] = (pthread_create(&th[t], NULL, part_tramp, &arg[t]) == 0);
  }
  fn(0, T, ctx);
  for (int t = 1; t < T; t++) {
    if (started[t]) pthread_join(th[t], NULL);
    else fn(t, T, ctx);                                  /* could not start a thread: do its part here */
  }
}
/* rows [lo, hi) of part t out of T */
static void part(int64_t n, int t, int T, int64_t* lo, int64_t* hi) {
  *lo = n / T * t + (n % T) * t / T; *hi = n / T * (t + 1) + (n % T) * (t + 1) / T;
}
static int threads_for(int64_t n) { return n < 65536 ? 1 : g_threads; }

/* stype codes: src/datatable/include/datatable.h:32-42 */
enum {
  ST_BOOL = 1, ST_INT8 = 2, ST_INT16 = 3, ST_INT32 = 4, ST_INT64 = 5,
  ST_FLOAT32 = 6, ST_FLOAT64 = 7, ST_DATE32 = 17, ST_TIME64 = 18
};
/* sort flags / NA position: sort.h:36-48 */
enum { FLAG_DESCENDING = 2, FLAG_SORT_ONLY = 4 };
enum { NA_FIRST = 1, NA_LAST = 2, NA_REMOVE = 3 };
/* reducer codes (ours; one per reference ColumnImpl) */
enum { OP_SUM = 1, OP_MEAN = 2, OP_MIN = 3, OP_MAX = 4, OP_COUNT = 5,
       OP_COUNTNA = 6, OP_NROWS = 7,
       /* within-group ordered reducers, expr/head_reduce_unary.cc */
       OP_FIRST = 8, OP_LAST = 9, OP_SD = 10, OP_MEDIAN = 11, OP_NUNIQUE = 12 };

static int stype_size(int st) {
  switch (st) {
    case ST_BOOL: case ST_INT8: return 1;
    case ST_INT16: return 2;
    case ST_INT32: case ST_FLOAT32: case ST_DATE32: return 4;
    case ST_INT64: case ST_FLOAT64: case ST_TIME64: return 8;
    default: return 0;
  }
}

/* Read element i of an integer-like column as int64; *na set when it is the
 * type's NA sentinel (stype.h:186-189: INT*_MIN; bool NA is int8 -128). */
static int64_t read_int(const void* p, int st, int64_t i, int* na) {
  switch (st) {
    case ST_BOOL: case ST_INT8: {
      int8_t v = ((const int8_t*)p)[i]; *na = (v == INT8_MIN); return v; }
    case ST_INT16: {
      int16_t v = ((const int16_t*)p)[i]; *na = (v == INT16_MIN); return v; }
    case ST_INT32: case ST_DATE32: {
      int32_t v = ((const int32_t*)p)[i]; *na = (v == INT32_MIN); return v; }
    default: {
      int64_t v = ((const int64_t*)p)[i]; *na = (v == INT64_MIN); return v; }
  }
}

/*---------------------------------------------------------------------------
 * Key normalisation: every key column becomes an array of uint64 radix keys
 * whose unsigned order is the requested row order.
 *   bool   : sort.cc:690-720  (_initB)
 *   int*   : sort.cc:729-776  (_initI/_initI_impl): NA->0, x = t-min+1 (ASC),
 *            max-t+1 (DESC); NA last: NA -> max-min+1 and the increment is 0.
 *            min/max are the column's non-NA stats (stats.cc:601-634).
 *   float* : sort.cc:809-845  (_initF): NaN -> 0 (all ones when NA last);
 *            ASC  t ^ (SBT | -(t>>63)), DESC t ^ (~SBT & ((t>>63) - 1)).
 * Returns the number of significant bits (sort.cc:735-736), or -1 for an
 * unsupported stype (NotImplError at sort.cc:673).
 *--------------------------------------------------------------------------*/
typedef struct {
  const void* col; int st, desc, na_pos; int64_t n; uint64_t* x;
  int phase;                       /* ints: 0 = stats, 1 = fill */
  int64_t mn, mx;                  /* ints, phase 1 */
  int64_t nna[ORC_MAX_THREADS], pmn[ORC_MAX_THREADS], pmx[ORC_MAX_THREADS];
} norm_ctx;

static void normalise_part(int t, int T, void* vc)
{
  norm_ctx* c = (norm_ctx*)vc;
  int64_t lo, hi; part(c->n, t, T, &lo, &hi);
  const void* col = c->col; const int st = c->st, desc = c->desc, na_pos = c->na_pos;
  uint64_t* x = c->x;
  int64_t nna = 0;
  if (st == ST_BOOL) {
    const uint8_t* xi = (const uint8_t*)col;
    uint8_t rep = (na_pos == NA_LAST) ? 3 : 0;
    for (int64_t j = lo; j < hi; j++) {
      uint8_t t8 = xi[j];
      if (t8 == 128) { x[j] = rep; nna++; }
      else x[j] = desc ? (uint8_t)((uint8_t)(128 - t8) >> 6) : (uint8_t)(t8 + 1);
    }
  } else if (st == ST_FLOAT32) {
    const uint32_t* xi = (const uint32_t*)col;
    const uint32_t EXP = 0x7F800000u, SIG = 0x007FFFFFu, SBT = 0x80000000u;
    uint32_t rep = (na_pos == NA_LAST) ? 0xFFFFFFFFu : 0;
    for (int64_t j = lo; j < hi; j++) {
      uint32_t u = xi[j];
      if ((u & EXP) == EXP && (u & SIG) != 0) { x[j] = rep; nna++; }
      else x[j] = desc ? (uint32_t)(u ^ (~SBT & ((u >> 31) - 1)))
                       : (uint32_t)(u ^ (SBT | (0u - (u >> 31))));
    }
  } else if (st == ST_FLOAT64) {
    const uint64_t* xi = (const uint64_t*)col;
    const uint64_t EXP = 0x7FF0000000000000ull, SIG = 0x000FFFFFFFFFFFFFull,
                   SBT = 0x8000000000000000ull;
    uint64_t rep = (na_pos == NA_LAST) ? ~0ull : 0;
    for (int64_t j = lo; j < hi; j++) {
      uint64_t u = xi[j];
      if ((u & EXP) == EXP && (u & SIG) != 0) { x[j] = rep; nna++; }
      else x[j] = desc ? (u ^ (~SBT & ((u >> 63) - 1)))
                       : (u ^ (SBT | (0ull - (u >> 63))));
    }
  } else if (c->phase == 0) {
    /* integer family, pass 1: the column's non-NA min / max (stats.cc:601-634) */
    int64_t mn = 0, mx = 0; int have = 0;
    for (int64_t j = lo; j < hi; j++) {
      int na; int64_t v = read_int(col, st, j, &na);
      if (na) { nna++; continue; }
      if (!have) { mn = mx = v; have = 1; }
      else { if (v < mn) mn = v; if (v > mx) mx = v; }
    }
    c->pmn[t] = have ? mn : INT64_MAX;
    c->pmx[t] = have ? mx : INT64_MIN;
  } else {
    /* integer family, pass 2 */
    const int sz = stype_size(st);
    const uint64_t tmask = (sz == 8) ? ~0ull : ((1ull << (8 * sz)) - 1);
    const uint64_t range1 = ((uint64_t)c->mx - (uint64_t)c->mn + 1) & tmask;
    const uint64_t rep = (na_pos == NA_LAST) ? range1 : 0;
    const uint64_t inc = (na_pos == NA_LAST) ? 0 : 1;
    for (int64_t j = lo; j < hi; j++) {
      int na; int64_t v = read_int(col, st, j, &na);
      if (na) x[j] = rep;
      else x[j] = (desc ? ((uint64_t)c->mx - (uint64_t)v + inc)
                        : ((uint64_t)v - (uint64_t)c->mn + inc)) & tmask;
    }
    return;
  }
  c->nna[t] = nna;
}

static int normalise(const void* col, int st, int desc, int na_pos,
                     int64_t n, uint64_t* x, int64_t* nacount)
{
  const int sz = stype_size(st);
  if (sz == 0) return -1;
  const int T = threads_for(n);
  norm_ctx* c = (norm_ctx*)calloc(1, sizeof(norm_ctx));
  c->col = col; c->st = st; c->desc = desc; c->na_pos = na_pos; c->n = n; c->x = x; c->phase = 0;
  par_run(T, normalise_part, c);
  int64_t nna = 0;
  for (int t = 0; t < T; t++) nna += c->nna[t];
  *nacount = nna;
  int nsig;
  if (st == ST_BOOL) nsig = 2;
  else if (st == ST_FLOAT32) nsig = 32;
  else if (st == ST_FLOAT64) nsig = 64;
  else {
    int64_t mn = INT64_MAX, mx = INT64_MIN;
    for (int t = 0; t < T; t++) { if (c->pmn[t] < mn) mn = c->pmn[t]; if (c->pmx[t] > mx) mx = c->pmx[t]; }
    if (mn > mx) { mn = 0; mx = 0; }                     /* no valid value */
    uint64_t range1 = (uint64_t)mx - (uint64_t)mn + 1;   /* max - min + 1 */
    uint64_t tmask = (sz == 8) ? ~0ull : ((1ull << (8 * sz)) - 1);
    range1 &= tmask;
    nsig = 0; { uint64_t r = range1; while (r) { nsig++; r >>= 1; } }
    c->phase = 1; c->mn = mn; c->mx = mx;
    par_run(T, normalise_part, c);
  }
  free(c);
  return nsig;
}

/* Stable LSD counting sort of (key, row) pairs on `nbits` low bits of key.
 * The reference sorts MSD-first with insertion-sort leaves
 * (sort.cc:1129-1353, sort_insert.cc:96-144); its contract is only
 * "stable ascending order of the normalised key" (sort.cc:27-33), which an
 * LSD pass sequence satisfies identically. */
typedef struct {
  uint64_t* k; int32_t* o; uint64_t* k2; int32_t* o2; int64_t n; int shift; int64_t* hist; int phase;
} lsd_ctx;

static void lsd_part(int t, int T, void* vc)
{
  lsd_ctx* c = (lsd_ctx*)vc;
  int64_t lo, hi; part(c->n, t, T, &lo, &hi);
  int64_t* h = c->hist + (size_t)t * 256;
  const uint64_t* k = c->k; const int shift = c->shift;
  if (c->phase == 0) {
    for (int64_t i = lo; i < hi; i++) h[(k[i] >> shift) & 255]++;
  } else if (c->phase == 1) {
    for (int64_t i = lo; i < hi; i++) {
      int64_t d = h[(k[i] >> shift) & 255]++;
      c->k2[d] = k[i]; c->o2[d] = c->o[i];
    }
  } else {
    memcpy(c->k + lo, c->k2 + lo, (size_t)(hi - lo) * sizeof(uint64_t));
    memcpy(c->o + lo, c->o2 + lo, (size_t)(hi - lo) * sizeof(int32_t));
  }
}

static void lsd_pairs(uint64_t* k, int32_t* o, uint64_t* k2, int32_t* o2,
                      int64_t n, int nbits)
{
  /* chunk-parallel like the reference (build_histogram / reorder_data, sort.cc:904-1012): every
   * part counts its contiguous chunk, the (digit, chunk) prefix gives each chunk its output slots,
   * every part scatters its chunk -- stable because chunks keep their order inside a digit */
  const int T = threads_for(n);
  int64_t* hist = (int64_t*)malloc((size_t)T * 256 * sizeof(int64_t));
  lsd_ctx c; c.k = k; c.o = o; c.k2 = k2; c.o2 = o2; c.n = n; c.hist = hist;
  for (int shift = 0; shift < nbits; shift += 8) {
    memset(hist, 0, (size_t)T * 256 * sizeof(int64_t));
    c.shift = shift; c.phase = 0;
    par_run(T, lsd_part, &c);
    int constant = 0;
    for (int b = 0; b < 256; b++) {
      int64_t tot = 0;
      for (int t = 0; t < T; t++) tot += hist[(size_t)t * 256 + b];
      if (tot == n) constant = 1;
    }
    if (constant) continue;
    int64_t run = 0;
    for (int b = 0; b < 256; b++)
      for (int t = 0; t < T; t++) {
        int64_t cnt = hist[(size_t)t * 256 + b]; hist[(size_t)t * 256 + b] = run; run += cnt;
      }
    c.phase = 1; par_run(T, lsd_part, &c);
    c.phase = 2; par_run(T, lsd_part, &c);
  }
  free(hist);
}

typedef struct {
  int64_t n; int32_t* order; const uint64_t* x; uint64_t* k; uint8_t* head; int32_t* offsets; int phase;
  int64_t pc[ORC_MAX_THREADS];
} grp_ctx;

static void grp_part(int t, int T, void* vc)
{
  grp_ctx* c = (grp_ctx*)vc;
  int64_t lo, hi; part(c->n, t, T, &lo, &hi);
  switch (c->phase) {
    case 0: for (int64_t i = lo; i < hi; i++) c->order[i] = (int32_t)i; break;
    case 1: for (int64_t i = lo; i < hi; i++) c->k[i] = c->x[c->order[i]]; break;
    case 2: for (int64_t i = (lo > 1 ? lo : 1); i < hi; i++)
              if (c->x[c->order[i]] != c->x[c->order[i - 1]]) c->head[i] = 1;
            break;
    case 3: { int64_t cnt = 0; for (int64_t i = lo; i < hi; i++) cnt += c->head[i]; c->pc[t] = cnt; break; }
    case 4: { int64_t g = c->pc[t]; for (int64_t i = lo; i < hi; i++) if (c->head[i]) c->offsets[g++] = (int32_t)i; break; }
  }
}

/*---------------------------------------------------------------------------
 * orc_group: restates group() (sort.cc:1411-1495).
 *   cols/stypes/flags : ncols key columns (flag bits: 2 = DESCENDING,
 *                       4 = SORT_ONLY, sort.h:36-41)
 *   order   [n]   : the RowIndex ARR32 payload (sort.cc:598-608)
 *   offsets [n+1] : Groupby offsets, offsets[0]=0 .. offsets[ng]=n
 *                   (groupby.h:41-47); written only when groups are produced
 *   *ngroups      : number of groups, or -1 when the reference returns an
 *                   empty Groupby (first flag SORT_ONLY, sort.cc:1491)
 *   *nskip        : rows to drop from the front of `order` when
 *                   na_pos == REMOVE (= NA count of the LAST key column,
 *                   sort.cc:598-605 -- quirk of the reference kept as is)
 * Returns 0, or -1 for an unsupported stype.
 *--------------------------------------------------------------------------*/
int orc_group(const void** cols, const int* stypes, const int* flags,
              int ncols, int na_pos, int64_t n,
              int32_t* order, int32_t* offsets,
              int64_t* ngroups, int64_t* nskip)
{
  *nskip = 0;
  if (n == 0) {                         /* sort.cc:1431-1434 */
    offsets[0] = 0; *ngroups = 0; return 0;
  }
  if (n == 1) {                         /* sort.cc:1435-1439 */
    order[0] = 0; offsets[0] = 0; offsets[1] = 1; *ngroups = 1; return 0;
  }
  uint64_t* x  = (uint64_t*)malloc((size_t)n * 8);
  uint64_t* k  = (uint64_t*)malloc((size_t)n * 8);
  uint64_t* k2 = (uint64_t*)malloc((size_t)n * 8);
  int32_t*  o2 = (int32_t*) malloc((size_t)n * 4);
  uint8_t* head = (uint8_t*)calloc((size_t)n, 1);
  grp_ctx gc; gc.n = n; gc.order = order; gc.x = x; gc.k = k; gc.head = head; gc.offsets = offsets;
  const int T = threads_for(n);
  gc.phase = 0; par_run(T, grp_part, &gc);              /* order[i] = i */

  /* number of leading "by" columns whose values define the groups
   * (sort.cc:1471-1482: groups are frozen at the by -> sort transition) */
  int nby = 0;
  while (nby < ncols && !(flags[nby] & FLAG_SORT_ONLY)) nby++;

  int rc = 0;
  int64_t nacount_last = 0;
  /* least-significant key first; each pass is stable */
  for (int c = ncols - 1; c >= 0; c--) {
    int64_t nna;
    int nsig = normalise(cols[c], stypes[c], (flags[c] & FLAG_DESCENDING) != 0,
                         na_pos, n, x, &nna);
    if (nsig < 0) { rc = -1; break; }
    if (c == ncols - 1) nacount_last = nna;
    gc.phase = 1; par_run(T, grp_part, &gc);            /* k[i] = x[order[i]] */
    lsd_pairs(k, order, k2, o2, n, nsig);
  }
  if (rc == 0) {
    if (nby > 0) {
      /* adjacent-compare group detection (sort_groups.cc:48-62 from_data) */
      head[0] = 1;
      for (int c = 0; c < nby; c++) {
        int64_t nna;
        normalise(cols[c], stypes[c], (flags[c] & FLAG_DESCENDING) != 0,
                  na_pos, n, x, &nna);
        gc.phase = 2; par_run(T, grp_part, &gc);        /* head[i] |= x[order[i]] != x[order[i-1]] */
      }
      /* heads -> offsets: per-part counts, prefix, fill */
      gc.phase = 3; par_run(T, grp_part, &gc);
      int64_t ng = 0;
      for (int t = 0; t < T; t++) { int64_t cnt = gc.pc[t]; gc.pc[t] = ng; ng += cnt; }
      gc.phase = 4; par_run(T, grp_part, &gc);
      offsets[ng] = (int32_t)n;
      *ngroups = ng;
    } else {
      *ngroups = -1;
    }
    if (na_pos == NA_REMOVE) *nskip = nacount_last;
  }
  free(x); free(k); free(k2); free(o2); free(head);
  return rc;
}

/*---------------------------------------------------------------------------
 * orc_gather: restates ArrayView_ColumnImpl<int32_t>::get_element
 * (column/view.cc:138-155) materialised by _materialize_fw
 * (column/column_impl.cc:78-103): out[i] = idx[i] < 0 ? NA : src[idx[i]].
 *--------------------------------------------------------------------------*/
int orc_gather(const void* src, int st, const int32_t* idx, int64_t n, void* out)
{
  int sz = stype_size(st);
  if (!sz) return -1;
  for (int64_t i = 0; i < n; i++) {
    int32_t j = idx[i];
    char* dst = (char*)out + i * sz;
    if (j >= 0) { memcpy(dst, (const char*)src + (int64_t)j * sz, (size_t)sz); continue; }
    switch (st) {
      case ST_BOOL: case ST_INT8: *(int8_t*)dst = INT8_MIN; break;
      case ST_INT16: *(int16_t*)dst = INT16_MIN; break;
      case ST_INT32: case ST_DATE32: *(int32_t*)dst = INT32_MIN; break;
      case ST_INT64: case ST_TIME64: *(int64_t*)dst = INT64_MIN; break;
      case ST_FLOAT32: *(float*)dst = NAN; break;
      case ST_FLOAT64: *(double*)dst = NAN; break;
    }
  }
  return 0;
}

/*---------------------------------------------------------------------------
 * orc_reduce: restates the per-group reducers.  `order` may be NULL
 * (identity RowIndex).  Output stypes and NA rules:
 *   SUM   column/sumprod.h:34-59, expr/fexpr_sumprod.cc:47-66
 *         bool/int* -> int64 (wraps), float32 -> float32 accumulated in
 *         float32, float64 -> float64; sequential in sorted order; NA skipped;
 *         never NA (empty -> 0).
 *   MEAN  column/mean.h:33-51, expr/fexpr_mean.cc:45-78
 *         double accumulator; ints/bool/float64 -> float64, float32 ->
 *         float32; no valid rows -> NA (NaN).
 *   MIN/MAX column/minmax.h:33-60, expr/fexpr_minmax.cc:47-72
 *         same stype as input (bool -> int8); first strictly-better valid
 *         value wins; no valid rows -> NA.
 *   COUNT/COUNTNA column/count.h:35-56; NROWS column/count.h:82-87 -> int64.
 *   FIRST/LAST expr/head_reduce_unary.cc:160-167: the element at the group's first / last
 *         position (NA stays NA), input stype.
 *   SD    expr/head_reduce_unary.cc:197-219: Welford recurrence over the valid rows in sorted
 *         order; count <= 1 or NaN m2 -> NA; float32 -> float32, everything else -> float64.
 *   MEDIAN expr/head_reduce_unary.cc:440-468: `order` must be sorted inside every group by the
 *         value, NA first (Column::sort_grouped, sort.cc:1499-1530; oracle.sort_grouped);
 *         skips the leading NAs, middle element or the mean of the two middle ones.
 *   NUNIQUE expr/head_reduce_unary.cc:383-394: size of a std::set<T> of the valid values
 *         (floats compare by value: -0.0 and +0.0 are one value) -> int64.
 *--------------------------------------------------------------------------*/
static int cmp_i64(const void* a, const void* b) { int64_t x = *(const int64_t*)a, y = *(const int64_t*)b; return (x > y) - (x < y); }
static int cmp_f64(const void* a, const void* b) { double x = *(const double*)a, y = *(const double*)b; return (x > y) - (x < y); }

static double elem_as_double(const void* v, int st, int64_t j, int* na) {
  if (st == ST_FLOAT32) { float f = ((const float*)v)[j]; *na = isnan(f); return (double)f; }
  if (st == ST_FLOAT64) { double d = ((const double*)v)[j]; *na = isnan(d); return d; }
  return (double)read_int(v, st, j, na);
}

static void ordered_groups(int op, const void* v, int st, const int32_t* order,
                           const int32_t* offsets, int64_t g_lo, int64_t g_hi, void* out)
{
  int sz = stype_size(st);
  int isf = (st == ST_FLOAT32 || st == ST_FLOAT64);
  for (int64_t g = g_lo; g < g_hi; g++) {
    int64_t i0 = offsets[g], i1 = offsets[g + 1];
    if (op == OP_FIRST || op == OP_LAST) {
      int64_t p = (op == OP_FIRST) ? i0 : i1 - 1;
      int64_t j = order ? order[p] : p;
      memcpy((char*)out + g * sz, (const char*)v + j * sz, (size_t)sz);
    } else if (op == OP_SD) {
      double mean = 0, m2 = 0; int64_t count = 0;
      for (int64_t gi = i0; gi < i1; gi++) {
        int64_t j = order ? order[gi] : gi;
        int na; double value = elem_as_double(v, st, j, &na);
        if (na) continue;
        count++;
        double tmp1 = value - mean;
        mean += tmp1 / (double)count;
        double tmp2 = value - mean;
        m2 += tmp1 * tmp2;
      }
      int valid = !(count <= 1 || isnan(m2));
      double sd = m2 >= 0 ? sqrt(m2 / (double)(count - 1)) : 0.0;
      if (st == ST_FLOAT32) ((float*)out)[g] = valid ? (float)sd : NAN;
      else ((double*)out)[g] = valid ? sd : NAN;
    } else if (op == OP_MEDIAN) {
      int na = 1;
      while (i0 < i1) { int64_t j = order ? order[i0] : i0; (void)elem_as_double(v, st, j, &na); if (!na) break; i0++; }
      if (i0 == i1) { if (st == ST_FLOAT32) ((float*)out)[g] = NAN; else ((double*)out)[g] = NAN; continue; }
      int64_t jm = (i0 + i1) / 2;
      int64_t r1 = order ? order[jm] : jm;
      double v1 = elem_as_double(v, st, r1, &na);
      if ((i1 - i0) & 1) {
        if (st == ST_FLOAT32) ((float*)out)[g] = (float)v1; else ((double*)out)[g] = v1;
      } else {
        int64_t r2 = order ? order[jm - 1] : jm - 1;
        double v2 = elem_as_double(v, st, r2, &na);
        if (st == ST_FLOAT32) ((float*)out)[g] = ((float)v1 + (float)v2) / 2;
        else ((double*)out)[g] = (v1 + v2) / 2;
      }
    } else if (op == OP_NUNIQUE) {
      int64_t m = i1 - i0, k = 0, distinct = 0;
      void* tmp = malloc((size_t)(m > 0 ? m : 1) * 8);
      for (int64_t gi = i0; gi < i1; gi++) {
        int64_t j = order ? order[gi] : gi;
        int na;
        if (isf) { double d = elem_as_double(v, st, j, &na); if (!na) ((double*)tmp)[k++] = d; }
        else { int64_t t = read_int(v, st, j, &na); if (!na) ((int64_t*)tmp)[k++] = t; }
      }
      qsort(tmp, (size_t)k, 8, isf ? cmp_f64 : cmp_i64);
      for (int64_t i = 0; i < k; i++)
        if (i == 0 || (isf ? ((double*)tmp)[i] != ((double*)tmp)[i - 1] : ((int64_t*)tmp)[i] != ((int64_t*)tmp)[i - 1])) distinct++;
      free(tmp);
      ((int64_t*)out)[g] = distinct;
    }
  }
}

typedef struct {
  int op; const void* v; int st; const int32_t* order; const int32_t* offsets; int64_t ng; void* out;
} red_ctx;

static void reduce_groups(int op, const void* v, int st, const int32_t* order,
                          const int32_t* offsets, int64_t g_lo, int64_t g_hi, void* out);

static void red_part(int t, int T, void* vc)
{
  /* groups are dealt out in blocks of 1024 round-robin, so that a few huge groups do not all land
   * in one part (the reference's parallel_for_static over groups, column_impl.h:106) */
  red_ctx* c = (red_ctx*)vc;
  for (int64_t g0 = (int64_t)t * 1024; g0 < c->ng; g0 += (int64_t)T * 1024) {
    int64_t g1 = g0 + 1024 < c->ng ? g0 + 1024 : c->ng;
    if (c->op >= OP_FIRST) ordered_groups(c->op, c->v, c->st, c->order, c->offsets, g0, g1, c->out);
    else reduce_groups(c->op, c->v, c->st, c->order, c->offsets, g0, g1, c->out);
  }
}

int orc_reduce(int op, const void* v, int st, const int32_t* order,
               const int32_t* offsets, int64_t ng, void* out)
{
  if (op < OP_SUM || op > OP_NUNIQUE) return -1;
  if (op != OP_NROWS && !stype_size(st)) return -1;
  red_ctx c; c.op = op; c.v = v; c.st = st; c.order = order; c.offsets = offsets; c.ng = ng; c.out = out;
  par_run(ng < 4096 ? 1 : g_threads, red_part, &c);
  return 0;
}

static void reduce_groups(int op, const void* v, int st, const int32_t* order,
                          const int32_t* offsets, int64_t g_lo, int64_t g_hi, void* out)
{
  int isf = (st == ST_FLOAT32 || st == ST_FLOAT64);
  for (int64_t g = g_lo; g < g_hi; g++) {
    int64_t i0 = offsets[g], i1 = offsets[g + 1];
    if (op == OP_NROWS) { ((int64_t*)out)[g] = i1 - i0; continue; }
    int64_t isum = 0; float fsum = 0.0f; double dsum = 0.0;
    int64_t cnt = 0;
    int have = 0; int64_t ibest = 0; double dbest = 0;
    for (int64_t gi = i0; gi < i1; gi++) {
      int64_t j = order ? order[gi] : gi;
      if (isf) {
        double d = (st == ST_FLOAT32) ? (double)((const float*)v)[j]
                                      : ((const double*)v)[j];
        if (isnan(d)) continue;
        cnt++;
        if (op == OP_SUM) {
          if (st == ST_FLOAT32) fsum = fsum + ((const float*)v)[j];
          else dsum = dsum + d;
        } else if (op == OP_MEAN) dsum += d;
        else if (op == OP_MIN) { if (!have || d < dbest) { dbest = d; have = 1; } }
        else if (op == OP_MAX) { if (!have || d > dbest) { dbest = d; have = 1; } }
      } else {
        int na; int64_t t = read_int(v, st, j, &na);
        if (na) continue;
        cnt++;
        if (op == OP_SUM) isum = (int64_t)((uint64_t)isum + (uint64_t)t);
        else if (op == OP_MEAN) dsum += (double)t;
        else if (op == OP_MIN) { if (!have || t < ibest) { ibest = t; have = 1; } }
        else if (op == OP_MAX) { if (!have || t > ibest) { ibest = t; have = 1; } }
      }
    }
    switch (op) {
      case OP_SUM:
        if (st == ST_FLOAT32) ((float*)out)[g] = fsum;
        else if (st == ST_FLOAT64) ((double*)out)[g] = dsum;
        else ((int64_t*)out)[g] = isum;
        break;
      case OP_MEAN:
        if (st == ST_FLOAT32) ((float*)out)[g] = cnt ? (float)(dsum / (double)cnt) : NAN;
        else ((double*)out)[g] = cnt ? dsum / (double)cnt : NAN;
        break;
      case OP_MIN: case OP_MAX:
        switch (st) {
          case ST_BOOL: case ST_INT8: ((int8_t*)out)[g] = have ? (int8_t)ibest : INT8_MIN; break;
          case ST_INT16: ((int16_t*)out)[g] = have ? (int16_t)ibest : INT16_MIN; break;
          case ST_INT32: case ST_DATE32: ((int32_t*)out)[g] = have ? (int32_t)ibest : INT32_MIN; break;
          case ST_INT64: case ST_TIME64: ((int64_t*)out)[g] = have ? ibest : INT64_MIN; break;
          case ST_FLOAT32: ((float*)out)[g] = have ? (float)dbest : NAN; break;
          case ST_FLOAT64: ((double*)out)[g] = have ? dbest : NAN; break;
        }
        break;
      case OP_COUNT:   ((int64_t*)out)[g] = cnt; break;
      case OP_COUNTNA: ((int64_t*)out)[g] = (i1 - i0) - cnt; break;
      default: break;
    }
  }
}
