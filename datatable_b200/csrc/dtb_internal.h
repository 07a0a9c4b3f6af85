// dtb_internal.h -- declarations shared by the engine's translation units.
// Host-side launch wrappers live next to their kernels; dtb_api.cu plans a
// call and strings them together on one stream.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include "../../include/dtb200.h"

namespace dtb {

constexpr int MAX_KEYS = 8;
constexpr int MAX_PASSES = 16;

// Thread-local error slot + launch counter (dtb_api.cu)
void set_error(const std::string& msg);
void count_launch(int n = 1);
// Optional CUDA-event timing of a kernel family (option "profile"; a no-op otherwise): the work enqueued on `s`
// while the scope lives, recorded on every way out of it.
struct ProfScope {
  ProfScope(const char* name, cudaStream_t s);
  ~ProfScope();
  bool on; cudaStream_t s; const char* name; cudaEvent_t a, b;
};

#define DTB_CUDA_CHECK(expr)                                                     \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) {                                                     \
      ::dtb::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));      \
      return DTB_ECUDA;                                                          \
    }                                                                            \
  } while (0)

#define DTB_TRY(expr)                                                            \
  do { int _rc = (expr); if (_rc != DTB_OK) return _rc; } while (0)

// ---------------------------------------------------------------------------
// Column statistics (replaces NumericStats<T>::compute_minmax, stats.cc:601-634)
// ---------------------------------------------------------------------------
// For integer stypes lo/hi are the signed min/max of the non-NA values; for
// float stypes they are the min/max of the order-preserving unsigned image
// (sort.cc:809-845 ASC transform).  bits_or / bits_and are OR / AND of that
// same image over the non-NA rows: bits that never vary need not be sorted.
struct ColStats {
  unsigned long long lo;       // int: (uint64)(int64 min); float: min image
  unsigned long long hi;
  unsigned long long bits_or;
  unsigned long long bits_and;
  unsigned long long nacount;
  unsigned long long nvalid;
};

int launch_col_stats(const void* data, int stype, int64_t n, ColStats* d_stats,
                     cudaStream_t s);
// The same statistics AND, from the same read of the column, the histogram of the low 8 bits of u (the
// sign-extended integer / float image) of every 4096-row tile: tile_hist u16[ntiles][256], NA rows apart in
// tile_na u16[ntiles].  Once edge / inc are known, the first radix pass folds it into its digit counts
// (PassIO::raw_hist) instead of reading the column a second time.
size_t stats_hist_bytes(int64_t n);          // bytes of tile_hist (tile_na follows, stats_na_bytes)
size_t stats_na_bytes(int64_t n);
int launch_col_stats_hist(const void* data, int stype, int64_t n, ColStats* d_stats, unsigned short* tile_hist,
                          unsigned short* tile_na, cudaStream_t s);
// The same statistics (bits_or / bits_and included) over the n positions of a RowIndex: position p reads
// data[order[p]] (int32 or int64 row ids), and an index outside [0, nrows) counts as an NA row.
int launch_col_stats_gather(const void* data, int stype, int64_t nrows, const void* order, int order_is64, int64_t n,
                            ColStats* d_stats, cudaStream_t s);

// ---------------------------------------------------------------------------
// Key normalisation parameters for one key column (restates _initB/_initI/_initF,
// sort.cc:690-845, as a function evaluated on the fly inside the kernels).
//   x = NA ? na_value : (((desc ? edge - u : u - edge) >> cshift) + inc)
// where u is the raw integer (sign-extended) or the float's ordered image.
// ---------------------------------------------------------------------------
struct KeyNorm {
  const void* data;
  int32_t  stype;
  int32_t  desc;
  unsigned long long edge;      // min (ASC) or max (DESC)
  unsigned long long na_value;  // 0 (NA first) or range+1 (NA last)
  unsigned long long inc;       // 1 (NA first) or 0 (NA last)
  int32_t  cshift;              // constant low bits dropped
  int32_t  bits;                // significant bits of x
  int32_t  lshift;              // position of x inside the composite key
  int32_t  pad;
};

struct KeyPlan {
  int      nkeys;
  int      total_bits;          // bits of the composite key
  int      group_shift;         // composite >> group_shift = group key (by-columns only)
  KeyNorm  k[MAX_KEYS];
};

// ---------------------------------------------------------------------------
// Radix sort (replaces SortContext::radix_psort / _radix_recurse,
// sort.cc:1129-1353, with stable LSD single-sweep passes)
// ---------------------------------------------------------------------------
struct PassPlan {
  int npasses;
  int shift[MAX_PASSES];
  int bits[MAX_PASSES];
};

// Composite key materialisation for multi-column keys: out[i] = X(row idx[i]) >> out_shift (idx NULL = identity).
// 4-byte keys must hold all total_bits - out_shift bits (DTB_EINVAL otherwise: never truncated).
int launch_compose_keys(const KeyPlan& kp, int64_t n, const int32_t* idx, void* keys_out,
                        int key_bytes, cudaStream_t s, int out_shift = 0);

struct PassIO {
  int         src_kind;     // 0 packed keys + idx_in (idx_in NULL = identity), 1 raw column (identity idx)
  const void* keys_in;      // packed keys (src_kind 0)
  const int32_t* idx_in;
  void*       keys_out;     // may be NULL on the last pass of a sort-only call
  int32_t*    idx_out;
  // first pass over a raw column whose normalisation keeps the low bits (cshift == 0): per-tile histogram of
  // the low 8 bits of u from launch_col_stats_hist; the pass folds it (x = +-(u - edge) + inc, NA -> na_value)
  // into its digit counts and does not run its count kernel
  const unsigned short* raw_hist = nullptr;
  const unsigned short* raw_na = nullptr;
  // keys_out receives (key >> out_shift) in words of out_bytes (1, 2, 4 or 8): only the bits later passes read
  int         out_shift = 0;
  int         out_bytes = 0;
  // Recovering the low bits of the keys in the last pass of a count-table round (the passes before it dropped them;
  // a row's consumed low bits v follow from its slot, the rows of v sit in slots [low_base[v], low_base[v+1])):
  //   bases_out   : receives the pass's 256 digit bases (the 2-pass low_base, or the next pass's regions)
  //   regions     : the previous pass's digit bases; the count kernel adds every row to low_hist[digit << region_bits
  //                 | region of its slot], and the pass turns low_hist into its exclusive scan (the 3-pass low_base)
  //   low_base    : last pass: key = (keys_in << low_bits) | v, v found from the row's slot
  uint32_t*       bases_out = nullptr;
  const uint32_t* regions = nullptr;
  int             region_bits = 0;
  uint32_t*       low_hist = nullptr;
  const uint32_t* low_base = nullptr;
  int             low_bits = 0;
  // First pass over a raw column with 32-bit keys (row id = position) of a region sum (launch_region_sum): the value
  // column `vals` (vbytes = 1, 2, 4 or 8 per row) travels with the rows, vperm[slot] = vals[row of the slot]
  const void*     vals = nullptr;
  void*           vperm = nullptr;
  int             vbytes = 0;
};

// One stable pass = count + scan + scatter kernels.  work: radix_pass_work_bytes(n) of scratch.
size_t radix_pass_work_bytes(int64_t n);
// group_count (optional, last pass only): uint32 table indexed by (key >> group_shift), zeroed by the
// caller; receives the number of rows of every group key (see launch_offsets_from_counts).
// key_bytes: width of the packed keys_in words (1, 2, 4 or 8), or of the composite for a raw column (4 or 8).
int launch_radix_pass(const PassIO& io, const KeyPlan& kp, int key_bytes, int64_t n,
                      int shift, int bits, uint32_t* work, cudaStream_t s,
                      uint32_t* group_count = nullptr, int group_shift = 0);

// Groupby offsets from a per-group-key row count table (small key domains): offsets[] = exclusive
// scan of the non-zero counts, gkeys[g] = key of group g, *d_ngroups = number of groups.
// table must be a multiple of 1024 entries and at most 2^22; scratch: uint64[2 * table / 1024 + 2].
int launch_offsets_from_counts(const uint32_t* count, int64_t table, int64_t n, int32_t* offsets,
                               uint32_t* gkeys, unsigned long long* d_ngroups, unsigned long long* scratch,
                               cudaStream_t s);

// Dense per-key tables for the multi-GPU merge of per-group partials (dtb_dense_scatter / dtb_dense_compact).
int launch_dense_scatter(const void* keys, int key_bytes, const void* vals, int64_t n, int64_t kmin, int64_t size,
                         void* table, uint32_t* present, cudaStream_t s);
int launch_dense_emit(const uint32_t* gidx, const void* table, int64_t ng, int64_t kmin, int key_bytes,
                      void* out_keys, void* out_vals, cudaStream_t s);

// ---------------------------------------------------------------------------
// Group offsets (replaces GroupGatherer, sort_groups.cc:34-117): heads where
// (key >> group_shift) changes, compacted into offsets[] by a single-pass scan.
// ---------------------------------------------------------------------------
// scratch: uint64[ntiles + 2] zeroed by the caller.  ngroups_out: device int64.
int64_t offsets_num_tiles(int64_t n);
// key_bytes 4/8: heads from adjacent sorted keys; key_bytes 1: `sorted_keys` is a uint8 head-flag
// array (multi-round composites wider than 64 bits, see launch_mark_heads).
int launch_group_offsets(const void* sorted_keys, int key_bytes, int group_shift, int64_t n,
                         int32_t* offsets_out, unsigned long long* d_ngroups,
                         unsigned long long* scratch, cudaStream_t s);
// flags[i] |= (keys[i] >> shift) != (keys[i-1] >> shift)
int launch_mark_heads(const void* sorted_keys, int key_bytes, int group_shift, int64_t n,
                      uint8_t* flags, cudaStream_t s);

// ---------------------------------------------------------------------------
// Reducers / gather
// ---------------------------------------------------------------------------
// Float min / max whose result is a zero: the reference keeps the first value that is strictly better
// (column/minmax.h:40-53), so the sign is that of the group's first valid zero in RowIndex order.  The
// order-preserving images rank -0.0 below +0.0, so the finalize looks that zero up, in one of two ways:
//   zpos (zero_fix_bytes(ngroups) of device scratch): the finalize marks the groups whose result is a zero, and one
//        row-parallel pass over the value column seen through order[0 .. n) (order NULL = identity; it returns at
//        once when no group was marked) finds each marked group's first valid zero;
//   first_zero (reducers fed piecewise): first_zero[g] = (RowIndex position << 1 | sign bit) of that zero, ~0: none.
// Neither set: the finalize keeps the zero it has.
struct GroupRows {
  const void* v = nullptr;
  int64_t nv = 0;
  const void* order = nullptr;
  int order_is64 = 0;
  const int32_t* offsets = nullptr;
  int64_t n = 0;                                   // positions under the groups: offsets[ngroups]
  unsigned long long* zpos = nullptr;
  const unsigned long long* first_zero = nullptr;
};
size_t zero_fix_bytes(int64_t ngroups);
// The reducer is a float min / max: the sign of a zero result needs the lookup above.
bool minmax_zero_sign(int op, int stype);

// pos[g] = min(pos[g], first position p in group g whose row order[p] (order NULL = identity) holds a zero of the
// float32 / float64 column v).  Row-parallel: one read of the positions and the values, one atomic per thread and
// group.  gate != NULL: nothing happens unless *gate != 0.  pos: the caller sets the groups it wants to ~0.
int launch_first_zero_pos(const void* v, int stype, int64_t nv, const void* order, int order_is64, const int32_t* offsets,
                          int64_t ngroups, int64_t n, const unsigned long long* gate, unsigned long long* pos,
                          cudaStream_t s);

// acc0/acc1: device scratch, ngroups uint64 each.  n = offsets[ngroups] (rows under the groups).
int launch_reduce_impl(int op, const void* value, int stype, int64_t nrows_value,
                       const void* order, int order_is64, const int32_t* offsets, int64_t ngroups,
                       int64_t n, unsigned long long* acc0, unsigned long long* acc1,
                       void* out, cudaStream_t s, void* extra = nullptr);
// device scratch `extra` that launch_reduce_impl needs for `op` (sd: sq[ng] and pivot[ng]; nunique: one flag byte per
// row; float min / max: the zero lookup's marks, see GroupRows)
size_t reduce_extra_bytes(int op, int stype, int64_t ng, int64_t n);
int reduce_out_stype_host(int op, int stype);
// *d_bad (device int, zeroed by the caller) = 1 + index of a group with offsets[g] >= offsets[g+1] (or offsets[0] != 0).
int launch_offsets_check(const int32_t* offsets, int64_t ng, int* d_bad, cudaStream_t s);

// Direct-address reducers over a small normalised key domain (see dtb_reduce.cu).
// Few distinct group keys (<= SMALL_TABLE) fold in per-CTA shared-memory tables (DIRECT_SMALL).
constexpr int SMALL_TABLE = 2048;
enum { DIRECT_PLAIN = 0,        // one L2 atomic per row into acc[x]
       DIRECT_SMALL = 1,        // <= 2048 accumulators: per-CTA shared-memory tables (map: uint16 x -> group, or NULL)
       DIRECT_HOT = 2 };        // skewed group sizes: rows of hot keys (map: uint8 hot[x]) fold in shared memory
struct DirectPlan {
  int kind;
  const void* map;
  int64_t nslots;               // accumulators in use: table, or ngroups for a dense-mapped small table
};
size_t direct_map_bytes(int64_t table);
// Chooses the streaming mode from the group structure (gmax = rows of the largest group) and builds the
// map it needs in map_scratch (direct_map_bytes(table) bytes, device).
int plan_direct(int64_t table, const uint32_t* gkeys, const int32_t* offsets, int64_t ngroups, int64_t n,
                int64_t gmax, void* map_scratch, cudaStream_t s, DirectPlan& dp);
// The accumulator tables' identities (once per reducer; the rows may then arrive in pieces), then the rows.
int launch_direct_init(int op, const DirectPlan& dp, int64_t table, unsigned long long* acc0, unsigned long long* acc1, cudaStream_t s);
int launch_direct_accumulate_rows(int op, const KeyPlan& kp, const DirectPlan& dp, const void* value, int stype, int64_t n,
                                  unsigned long long* acc0, unsigned long long* acc1, cudaStream_t s);
// A sum over the rows as the first radix pass left them (GroupPlan::region_sum): the pass put every row in the region of
// its low rbits key bits (region d = slots [bases[d], bases[d + 1]), bases: the pass's 256 digit bases), and wrote the
// rest of its group key (lbits <= 13 bits, in words of key_bytes = 1 or 2) to lkey[slot] and its value to vperm[slot].
// Every row adds its value to acc0[lkey << rbits | d].  hot: the hot-key map of a DIRECT_HOT plan, or NULL.
constexpr int REGION_MAX_LBITS = 13;
int launch_region_sum(const void* lkey, int key_bytes, int rbits, int lbits, const uint32_t* bases, const void* vperm,
                      int stype, int64_t n, const uint8_t* hot, unsigned long long* acc0, cudaStream_t s);
// out[g] from the accumulators of group key gkeys[g], or of group g when dp is a dense-mapped small table.
int launch_direct_finalize(int op, int stype, const unsigned long long* acc0, const unsigned long long* acc1,
                           const DirectPlan& dp, const uint32_t* gkeys, int64_t ngroups, void* out, const GroupRows& rows,
                           cudaStream_t s);
// Reducers fed piecewise, float min / max: inv[order[p]] = p over the handle's RowIndex (n int32), then for every
// piece the RowIndex position and sign of each group's first valid zero (GroupRows::first_zero, ngroups u64
// set to ~0 by the caller).
int launch_inverse_order(const int32_t* order, int64_t n, int32_t* inv, cudaStream_t s);
int launch_first_zero_rows(const void* value_rows, int stype, int64_t row0, int64_t nrows, const int32_t* inv,
                           const int32_t* offsets, int64_t ngroups, unsigned long long* first_zero, cudaStream_t s);
int launch_nrows(const int32_t* offsets, int64_t ngroups, void* out, cudaStream_t s);
int launch_group_keys(const void* sorted_keys, int key_bytes, const int32_t* offsets, int group_shift,
                      int64_t ngroups, uint32_t* gkeys, cudaStream_t s);

// Bucketed multi-reducer (dtb_bucket.cu): all reducers of one value column in one sweep over rows partitioned
// by group-key bucket, shared-memory accumulators.  Words a column can ask for:
enum { BK_SUMI = 0, BK_SUMF = 1, BK_CNT = 2, BK_MIN = 3, BK_MAX = 4, BK_CNTNA = 5, BK_NWORDS = 6 };
constexpr int BK_MAX_DBITS = 20, BK_MIN_DBITS = 12;
// rows per (slab of tiles, bucket) of the group keys xkeys[i] >> gshift: slab_starts u32[bucket_starts_bytes(n)/4]
// (first output slot of every slab inside every bucket), bstart u32[nb+1] (bucket boundaries)
size_t bucket_starts_bytes(int64_t n);
int launch_bucket_starts(const uint32_t* xkeys, int gshift, int64_t n, int nb, uint32_t* slab_starts, uint32_t* bstart, cudaStream_t s);
constexpr int BK_MAXCOLS = 4;                 // value columns partitioned in one sweep
size_t bucket_scratch_bytes(int64_t n, int sum_value_bytes, int ncols);
int launch_bucketed_reduce(const uint32_t* xkeys, int gshift, int dbits, int ncols, const void* const* values,
                           const int* stypes, int64_t n, const uint32_t* slab_starts, const uint32_t* start,
                           unsigned long long* const (*acc_w)[BK_NWORDS], void* scratch, cudaStream_t s);
void fill_u64(unsigned long long* p, int64_t n, unsigned long long v, cudaStream_t s);

int launch_gather(const void* src, int stype, int64_t nrows_src, const void* order,
                  int order_is64, int64_t n, void* out, cudaStream_t s);

int launch_iota32(int32_t* out, int64_t n, cudaStream_t s);
int launch_widen_u32(const uint32_t* in, int64_t n, int64_t* out, cudaStream_t s);   // ARR32 bit patterns -> ARR64

// ---------------------------------------------------------------------------
// SURVEY.md 8(f) rows (dtb_next.cu): ordered reducers, set operations, mode, join
// ---------------------------------------------------------------------------
int launch_firstlast(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                     int64_t ng, int last, void* out, cudaStream_t s);
int launch_expand_gid(const int32_t* offsets, int64_t ng, int64_t n, int32_t* gid, cudaStream_t s);
// integer slice applied inside every group (dtb_slice_groups)
struct SliceParams { long long start, stop, step, nrows; int has_start, has_stop; };
size_t slice_scratch_bytes(int64_t ng);
int launch_slice_groups_plan(const int32_t* offsets, int64_t ng, const SliceParams& p, void* scratch, int32_t* offsets_out,
                             int32_t* gsel, unsigned long long* totals, cudaStream_t s);
int launch_slice_groups_emit(const int32_t* offsets, const SliceParams& p, const int32_t* offsets_out, const int32_t* gsel,
                             int64_t ng_out, int64_t nout, int32_t* gid, int32_t* rows_out, cudaStream_t s);
// rows selected by a bool8 column (dtb_mask_rows): launch_mask_count writes the selected rows of every tile and turns
// them into each tile's first output position in tile_count (u64[mask_num_tiles(n)]), and their sum to *total
// (device u64); launch_mask_emit then writes the ascending positions, *total of them, to rows_out
int64_t mask_num_tiles(int64_t n);
int launch_mask_count(const int8_t* mask, int64_t n, unsigned long long* tile_count, unsigned long long* total,
                      cudaStream_t s);
int launch_mask_emit(const int8_t* mask, int64_t n, const unsigned long long* tile_start, int32_t* rows_out,
                     cudaStream_t s);
// an int8 / int16 / int64 selector as an int32 RowIndex, NA -> INT32_MIN (dtb_int_rows)
int launch_narrow_rows(const void* sel, int stype, int64_t n, int32_t* out, cudaStream_t s);
// sd, cov and corr per group: two passes over the values shifted by a pivot, the value at the group's first valid
// row.  The words of every group (device, ng each; the kernels set them): sum[k] = Σ (x_k - pivot_k) and cnt (the first
// pass), sq[k] = Σ dx_k² and sxy = Σ dx_0 dx_1 (the second), pivot[k].  sd uses sum[0], cnt, sq[0] and pivot[0]; cov
// sum, cnt, sxy and pivot; corr every word.
struct MomentWords { double* sum[2]; unsigned long long* cnt; double* sq[2]; double* sxy; double* pivot[2]; };
// op = DTB_OP_SD: sd of column x (y unused) through an int32 RowIndex; DTB_OP_COV / DTB_OP_CORR: over the pairs (x, y)
// where both are valid, through int32 or int64 row ids.  out: out_stype, float32 or float64.
int launch_moments(int op, const void* x, int sx, const void* y, int sy, int64_t nv, const void* order, int order_is64,
                   const int32_t* offsets, int64_t ng, int64_t n, const MomentWords& w, int out_stype, void* out,
                   cudaStream_t s);
// cov / corr over the pairs (x, y) seen through `order` (int32 or int64 row ids), segmented by offsets.  scratch:
// reduce2_scratch_bytes(ng) of device memory.  out: float32 when out_f32, else float64 (reduce2_out_stype_host).
int reduce2_out_stype_host(int op, int stype_x, int stype_y);
size_t reduce2_scratch_bytes(int64_t ng);
int launch_reduce2(int op, const void* x, int sx, const void* y, int sy, int64_t nv, const void* order, int order_is64,
                   const int32_t* offsets, int64_t ng, int64_t n, unsigned long long* scratch, int out_f32, void* out,
                   cudaStream_t s);
int launch_median(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                  int64_t ng, void* out, cudaStream_t s);
int launch_distinct_flags(const void* v, int stype, int64_t nv, const int32_t* order, const int32_t* offsets,
                          int64_t ng, int64_t n, int8_t* flag, cudaStream_t s);
// qcut inside every group (dtb_qcut): cord / coff / nc are group() of the composite key (gid, vg), with gid / vg the
// outer group id and the value at every RowIndex position (n of them, ng outer groups); out[pos]: int32 bins in the
// outer RowIndex's layout.  scratch: qcut_scratch_bytes(nc, ng) of device memory.
size_t qcut_scratch_bytes(int64_t nc, int64_t ng);
int launch_qcut(const void* vg, int stype, const int32_t* cord, const int32_t* coff, int64_t nc, const int32_t* gid,
                int64_t ng, int64_t n, int q, void* scratch, int32_t* out, cudaStream_t s);
// cut over the n positions of a RowIndex (dtb_cut, dtb_cut.cu); order NULL = identity.  out: int32[n].
//   nbins mode: launch_cut_coef turns the statistics of the column seen through the RowIndex into the coefficients
//               (device, one CutCoef), then launch_cut_emit writes the bins;
//   edges mode: launch_cut_bins searches d_edges (device float64[nedges], strictly increasing, nedges >= 2).
struct CutCoef { double a, b; int32_t shift, na; };
int launch_cut_coef(const ColStats* d_stats, int stype, int nbins, int right_closed, CutCoef* coef, cudaStream_t s);
int launch_cut_emit(const void* v, int stype, int64_t nv, const void* order, int order_is64, int64_t n,
                    const CutCoef* coef, int32_t* out, cudaStream_t s);
int launch_cut_bins(const void* v, int stype, int64_t nv, const void* order, int order_is64, int64_t n,
                    const double* d_edges, int64_t nedges, int right_closed, int32_t* out, cudaStream_t s);
// part DTB_TIME_* of a date32 / time64 column over the n positions of a RowIndex (dtb_time_part, dtb_time.cu); order
// NULL = identity.  out: int32[n].
int launch_time_part(int part, const void* v, int stype, int64_t nv, const void* order, int order_is64, int64_t n,
                     int32_t* out, cudaStream_t s);
// cumsum / cumprod / cummin / cummax inside every group (dtb_cumulative, dtb_reduce.cu): op DTB_OP_SUM / PROD / MIN /
// MAX; out[p]: n elements of cumulative_out_stype(op, stype) (0: the op refuses the stype) for RowIndex position p.
// scratch: cumulative_scratch_bytes(n) of device memory.
int cumulative_out_stype(int op, int stype);
size_t cumulative_scratch_bytes(int64_t n);
int launch_cumulative(int op, int reverse, const void* v, int stype, int64_t nv, const void* order, int order_is64,
                      const int32_t* offsets, int64_t ng, int64_t n, void* scratch, void* out, cudaStream_t s);
// shift / fillna / cumcount / ngroup inside every group (dtb_shift, dtb_fillna, dtb_group_index, dtb_reduce.cu):
// out[p] for RowIndex position p, n elements of the value's stype (shift, fillna) or of int64 (group_index, kind
// DTB_GROUP_CUMCOUNT / DTB_GROUP_NGROUP).  fillna's scratch: cumulative_scratch_bytes(n) of device memory.
int launch_shift(const void* v, int stype, int64_t nv, const void* order, int order_is64, const int32_t* offsets,
                 int64_t ng, int64_t n, int64_t shift, void* out, cudaStream_t s);
int launch_fillna(int reverse, const void* v, int stype, int64_t nv, const void* order, int order_is64,
                  const int32_t* offsets, int64_t ng, int64_t n, void* scratch, void* out, cudaStream_t s);
int launch_group_index(int kind, int reverse, const int32_t* offsets, int64_t ng, int64_t n, int64_t* out,
                       cudaStream_t s);
int launch_set_select(const int32_t* order, const int32_t* offsets, int64_t ng, const int64_t* d_sizes, int K,
                      int mode, uint8_t* flags, cudaStream_t s);
int launch_set_emit(const int32_t* pos, int64_t nsel, const int32_t* order, const int32_t* offsets, int32_t* out_rows,
                    cudaStream_t s);
int launch_largest_group(const int32_t* offsets, int64_t ng, int64_t skip, unsigned long long* d_result, cudaStream_t s);
int launch_lower_bound(const void* sorted, int stype, int64_t n, const void* values, int64_t m, int64_t* out, cudaStream_t s);
// natural join (dtb_join_gather): index[r] (may be NULL) = J's row matched by X row r or INT32_MIN, and for each of
// the nvals value columns of J vout[c][r] = vals[c][that row], or the stype's NA
constexpr int JOIN_MAX_VALS = 16;
int launch_join(int nkeys, const void* const* xcols, const int* xst, const void* const* jcols, const int* jst,
                int64_t nx, int64_t nj, int32_t* index, int nvals, const void* const* vals, const int* vst,
                void* const* vout, cudaStream_t s);

}  // namespace dtb
