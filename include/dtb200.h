/*
 * dtb200.h -- C-ABI of the H100-native groupby/sort engine that sits behind
 * h2oai/datatable's DT[i, j, by(), sort()] hot path.
 *
 * The reference has no FFI seam on this path (SURVEY.md 8b): the boundary is
 * its internal C++ function group() and the materialize() of its reducer /
 * view columns.  Every entry point below names the reference interface it
 * replaces (paths relative to the reference's src/core/).  INTEGRATION.md
 * shows the reference-side binding.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch types cross this boundary.
 *   - every data pointer may be DEVICE memory or HOST memory (pinned or
 *     pageable); the engine detects which (cudaPointerGetAttributes).  Host
 *     inputs are staged to HBM, host outputs are copied back, inside the call.
 *   - `stream` is a cudaStream_t (NULL = legacy default stream).  Calls that
 *     return scalars (dtb_group*) block until their results are final; calls
 *     whose outputs are all in device memory (dtb_reduce, dtb_gather) only
 *     enqueue work on `stream`.  Host outputs are always complete on return.
 *   - return value 0 = success, negative = DTB_E*; dtb_last_error() gives the
 *     thread-local message (the reference throws dt::Error subclasses,
 *     utils/exceptions.h:43; a C ABI must not throw).
 *   - there is NO CPU fallback: without a usable CUDA device every compute
 *     call fails with DTB_ECUDA once its arguments pass the checks that need
 *     no device.
 */
#ifndef DTB200_H
#define DTB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DTB_ABI_VERSION 1

#if defined(__GNUC__)
#  define DTB_API __attribute__((visibility("default")))
#else
#  define DTB_API
#endif

/* stype codes == DtStype_* of src/datatable/include/datatable.h:32-42 */
#define DTB_STYPE_BOOL     1
#define DTB_STYPE_INT8     2
#define DTB_STYPE_INT16    3
#define DTB_STYPE_INT32    4
#define DTB_STYPE_INT64    5
#define DTB_STYPE_FLOAT32  6
#define DTB_STYPE_FLOAT64  7
#define DTB_STYPE_DATE32   17   /* sorted as int32, sort.cc:666 */
#define DTB_STYPE_TIME64   18   /* sorted as int64, sort.cc:668 */

/* SortFlag bits, sort.h:36-41 */
#define DTB_FLAG_NONE        0
#define DTB_FLAG_DESCENDING  2
#define DTB_FLAG_SORT_ONLY   4

/* NaPosition, sort.h:43-48 */
#define DTB_NA_FIRST   1
#define DTB_NA_LAST    2
#define DTB_NA_REMOVE  3

/* reducers: one per reference ColumnImpl */
#define DTB_OP_SUM      1   /* SumProd_ColumnImpl<T,true,..>  column/sumprod.h:30-62 */
#define DTB_OP_MEAN     2   /* Mean_ColumnImpl                column/mean.h:29-52    */
#define DTB_OP_MIN      3   /* MinMax_ColumnImpl<T,true>      column/minmax.h:29-62  */
#define DTB_OP_MAX      4   /* MinMax_ColumnImpl<T,false>                            */
#define DTB_OP_COUNT    5   /* CountUnary_ColumnImpl<T,false> column/count.h:31-56   */
#define DTB_OP_COUNTNA  6   /* CountUnary_ColumnImpl<T,true>                         */
#define DTB_OP_NROWS    7   /* CountNullary_ColumnImpl        column/count.h:60-89   */
/* within-group ordered reducers (SURVEY.md 8f; expr/head_reduce_unary.cc) */
#define DTB_OP_FIRST    8   /* FirstLast_ColumnImpl<true>     head_reduce_unary.cc:120-170: value of the group's first row */
#define DTB_OP_LAST     9   /* FirstLast_ColumnImpl<false>                                                                  */
#define DTB_OP_SD      10   /* sd_reducer                     head_reduce_unary.cc:197-219: sample sd, count <= 1 -> NA    */
#define DTB_OP_MEDIAN  11   /* Median_ColumnImpl              head_reduce_unary.cc:421-468: needs dtb_sort_grouped's order */
#define DTB_OP_NUNIQUE 12   /* op_nunique                     head_reduce_unary.cc:383-394: needs dtb_sort_grouped's order */
#define DTB_OP_PROD    13   /* SumProd_ColumnImpl<T,false,..> column/sumprod.h:34-59, fexpr_sumprod.cc:47-67       */
/* two-column reducers: dtb_reduce2 / dtb_groupby_reduce2 only (the one-column entry points return DTB_EINVAL) */
#define DTB_OP_COV     14   /* cov_reducer                    head_reduce_binary.cc:114-138: sample covariance       */
#define DTB_OP_CORR    15   /* corr_reducer                   head_reduce_binary.cc:168-200: Pearson correlation     */

/* set operations, set_funcs.cc:126-456 */
#define DTB_SET_UNION      0
#define DTB_SET_INTERSECT  1
#define DTB_SET_SETDIFF    2
#define DTB_SET_SYMDIFF    3

/* error codes */
#define DTB_OK         0
#define DTB_EINVAL    -1   /* bad argument (ValueError / TypeError in the reference) */
#define DTB_ENOTIMPL  -2   /* unsupported stype (NotImplError, sort.cc:673): caller falls back outside the path */
#define DTB_ECUDA     -3   /* CUDA runtime failure or no device */
#define DTB_ENOMEM    -4
#define DTB_ENOSPACE  -5   /* caller-provided output too small; *ngroups_out still set */

typedef void* dtb_stream;           /* cudaStream_t */

/* A material fixed-width column: raw typed buffer with NA sentinels
 * (SentinelFw_ColumnImpl, column/sentinel_fw.h:34-78; NA constants stype.h:186-197). */
typedef struct dtb_col {
  const void* data;
  int32_t     stype;
  int32_t     reserved;
} dtb_col;

/* Thread-local message of the last failing call on this thread ("" if none). */
DTB_API const char* dtb_last_error(void);

/* DTB_ABI_VERSION of the loaded library (cf. DtABIVersion(), datatable.h:49). */
DTB_API int dtb_abi_version(void);

/* Bytes per element of an stype (0 = unsupported on this path). */
DTB_API int dtb_stype_size(int stype);

/* Output stype of reducer `op` applied to a column of `stype`
 * (expr/fexpr_sumprod.cc:50-66, fexpr_mean.cc:49-78, fexpr_minmax.cc:50-72,
 *  fexpr_count.cc:47-128); 0 if the combination is invalid. */
DTB_API int dtb_reduce_out_stype(int op, int stype);

/* Selects the CUDA device used by this thread's subsequent calls and creates
 * the engine context on it.  Optional: the first compute call does it for the
 * current device. */
DTB_API int dtb_init(int device);

/*
 * dtb_group -- replaces RiGb group(columns, flags, na_pos)  (sort.h:56-58,
 * sort.cc:1411-1495) for material bool/int/float key columns.
 *
 *   keys[nkeys], flags[nkeys] : key columns (by-columns first) and their
 *                               SortFlag bits
 *   na_pos                    : DTB_NA_*
 *   nrows                     : rows per column (<= INT32_MAX; more: dtb_group64)
 *   order_out                 : int32[nrows]  -- the ARR32 RowIndex payload
 *                               (sort.cc:598-608); with DTB_NA_REMOVE only the
 *                               first *norder_out entries are written
 *   offsets_out               : int32[offsets_cap] -- Groupby offsets,
 *                               offsets[0]=0 .. offsets[ng]=nrows
 *                               (groupby.h:41-47); may be NULL when flags[0]
 *                               has SORT_ONLY
 *   *ngroups_out              : number of groups; -1 when the reference
 *                               returns an empty Groupby (sort.cc:1491-1493)
 *   *norder_out               : valid entries in order_out
 *
 * Groups are defined by the LEADING run of columns without SORT_ONLY (sort.cc:1478-1480): a column after
 * the first SORT_ONLY one only orders the rows, whatever its flag.  DTB_NA_REMOVE is refused with
 * DTB_EINVAL when groups are requested (flags[0] without SORT_ONLY): the RowIndex would drop rows that
 * the groups still count.  A single row is never removed (sort.cc:1435-1439).
 *
 * Bit-exact with the reference for order and offsets.
 */
DTB_API int dtb_group(const dtb_col* keys, int nkeys, const int* flags, int na_pos,
              int64_t nrows, dtb_stream stream,
              void* order_out, void* offsets_out, int64_t offsets_cap,
              int64_t* ngroups_out, int64_t* norder_out);

/*
 * dtb_group64 -- dtb_group with the ARR64 layout: order_out is int64[nrows] (RowIndex ARR64,
 * rowindex_array.cc:50-60; the reference's new sorter emits it above INT32_MAX rows, sort/sorter.cc:74-81)
 * and offsets_out is int64[offsets_cap] (the reference's Groupby is int32-only, sort.h:119-124 "TODO: Add
 * support for 64-bit groups" -- this is the variant SURVEY.md 8b asks for).  nrows < 2^32 - 65536 on one
 * GPU (beyond that the frame is row-partitioned across GPUs, datatable_b200/dist.py); works for any
 * smaller nrows too.  Same ordering, groups and NA rules as dtb_group.
 */
DTB_API int dtb_group64(const dtb_col* keys, int nkeys, const int* flags, int na_pos,
              int64_t nrows, dtb_stream stream,
              void* order_out, void* offsets_out, int64_t offsets_cap,
              int64_t* ngroups_out, int64_t* norder_out);

/*
 * Handle variant: results stay resident in HBM (no worst-case caller buffers,
 * no host round trip before the reducers).  The handle owns order/offsets.
 */
typedef struct dtb_groupby dtb_groupby;

DTB_API int dtb_groupby_create(const dtb_col* keys, int nkeys, const int* flags,
                       int na_pos, int64_t nrows, dtb_stream stream,
                       dtb_groupby** out);
/*
 * Fused variant: group() plus `nreducers` per-group reducers in one call (the j-expressions of
 * DT[:, {sum(f.v), ...}, by(f.k)] are known before group() runs, expr/eval_context.cc:144-172).
 * When the group-key domain is small the reducers only need the key columns: once the groups are
 * known they stream the key and value columns in storage order.  Results are owned by the handle:
 * dtb_groupby_reduced(g, i) = device buffer of ngroups elements of stype
 * dtb_reduce_out_stype(op, value.stype).  Equivalent to dtb_groupby_create + dtb_groupby_reduce.
 */
typedef struct dtb_reduce_spec {
  int32_t op;          /* DTB_OP_* */
  int32_t reserved;
  dtb_col value;       /* ignored for DTB_OP_NROWS */
} dtb_reduce_spec;

DTB_API int dtb_groupby_create_reduce(const dtb_col* keys, int nkeys, const int* flags,
                       int na_pos, int64_t nrows, dtb_stream stream,
                       const dtb_reduce_spec* reducers, int nreducers, dtb_groupby** out);
DTB_API const void* dtb_groupby_reduced(const dtb_groupby* g, int i);

DTB_API int64_t     dtb_groupby_norder(const dtb_groupby* g);    /* RowIndex length               */
DTB_API int64_t     dtb_groupby_ngroups(const dtb_groupby* g);   /* -1 = no Groupby (sort only)   */
DTB_API const void* dtb_groupby_order(const dtb_groupby* g);     /* device int32[norder]          */
DTB_API const void* dtb_groupby_offsets(const dtb_groupby* g);   /* device int32[ngroups+1]/NULL  */
DTB_API int         dtb_groupby_destroy(dtb_groupby* g, dtb_stream stream);

/*
 * Per-group functions: dtb_reduce, dtb_reduce2, dtb_cumulative, dtb_shift, dtb_fillna, dtb_group_index, dtb_qcut,
 * dtb_sort_grouped, and the handle variants dtb_groupby_reduce / dtb_groupby_reduce2, share one argument contract.
 * The value columns hold nrows_value rows each and are seen through the RowIndex `order` (NULL = identity;
 * order_is64: int64 row ids, where the function takes them, else int32).  `offsets` (int32[ngroups+1]) cuts the
 * n = offsets[ngroups] positions of the RowIndex into groups; a call without by() passes one group [0, n].  Every
 * pointer may be host or device memory.  The arguments are checked in this order, all on the host before any CUDA
 * call, so that without a device an argument error still returns its own code:
 *   1. the function's own argument (op, kind, nquantiles): DTB_EINVAL;
 *   2. the stype: one without a fixed width gives DTB_ENOTIMPL, one the op refuses DTB_EINVAL;
 *   3. ngroups < 0;  4. offsets NULL;  5. nrows_value < 0;  6. value data NULL while nrows_value > 0;
 *   7. out NULL while ngroups > 0 (for one output per position: unless the only group is [0, 0]): DTB_EINVAL.
 * ngroups == 0 then returns at once.  Caller offsets must be a Groupby (groupby.h:41-47): offsets[0] = 0 and
 * strictly increasing, so no group is empty; otherwise DTB_EINVAL (device offsets are checked on the device; a
 * handle's own offsets are not checked).  The one exception is ngroups == 1 with offsets [0, 0], the single group
 * of zero rows a query without by() reduces over (Groupby::single_group(0), groupby.cc:60-68): the reducers write
 * its one result -- SUM 0, PROD 1, COUNT / COUNTNA / NROWS / NUNIQUE 0, every other reducer NA -- and the functions
 * with one output per position write nothing.  No kernel reads a row or a RowIndex position for it.  Positions beyond the value column: without an order, n > nrows_value is
 * DTB_EINVAL for the row functions (dtb_cumulative, dtb_shift, dtb_fillna, dtb_qcut); the reducers and
 * dtb_sort_grouped read those positions as NA (nrows_value bounds the gather).
 */

/*
 * dtb_reduce -- replaces ColumnImpl::materialize() of the per-group reducer
 * columns (column/reduce_unary.h:30-68 driven by column/latent.cc:103-135 and
 * column/column_impl.cc:78-103): value column viewed through the RowIndex
 * `order` (NULL = identity), segmented by `offsets`; arguments as in
 * "Per-group functions" above.
 *
 *   out : ngroups elements of stype dtb_reduce_out_stype(op, value.stype);
 *         NA results are written as the stype's NA sentinel.
 *   nrows_value : rows in the value column (bounds the gather).
 *
 * SUM over integers/bool (wrapping modulo 2^64), MIN, MAX (the sign of a zero
 * included: the group's first valid zero in RowIndex order), COUNT*, NROWS are
 * bit-exact.  Floating SUM/MEAN are accumulated in float64 in an unspecified
 * order: a group of m valid rows has a sum within gamma(m-1) * sum|x| of the
 * exact sum, gamma(k) = k*u / (1 - k*u), u = 2^-53; MEAN is that sum over the
 * count; float32 results add their final rounding.  A cancelling group can
 * differ from the reference's sequential sum by that much, in relative terms
 * without limit.  SD of a group whose valid values are all equal is 0.0.
 *
 * PROD skips NA rows and starts at 1, so a group without valid rows gives 1.
 * Over integers/bool it is an INT64 product wrapping modulo 2^64, bit-exact.
 * Over floats (FLOAT32 -> FLOAT32, FLOAT64 -> FLOAT64) the engine keeps the
 * significand and the binary exponent apart, in float64, so no intermediate
 * product overflows or underflows: a group of m valid finite non-zero rows
 * gives the exact product times (1 + d), |d| <= gamma(m-1), rounded once to
 * the output stype.  A zero and an infinity in the same group give NA (the
 * reference's 0 * inf = NaN); a zero alone gives 0 and an infinity alone gives
 * inf, signed by the parity of the negative rows.  Two deviations from the
 * reference, which multiplies in order in the column's own type: float32
 * groups are multiplied in float64, and where the reference's running product
 * overflows to inf or underflows to 0 part-way although the exact product is
 * in range, the engine returns the in-range value (so such a group that also
 * holds a zero or an inf is not NA here).  Streaming and piecewise paths do
 * not exist for PROD: dtb_groupby_reduce and dtb_groupby_create_reduce take
 * the RowIndex, and dtb_groupby_reduce_begin returns DTB_ENOTIMPL.
 */
DTB_API int dtb_reduce(int op, dtb_col value, int64_t nrows_value,
               const void* order, int order_is64,
               const void* offsets, int64_t ngroups,
               dtb_stream stream, void* out);

/*
 * dtb_groupby_reduce -- dtb_reduce over the handle's RowIndex / offsets.  When the handle's
 * key domain is small (normalised group key < 2^22 values) and the key columns passed to
 * dtb_groupby_create live in device memory, the reducer streams the key and value columns in
 * storage order and accumulates with L2 atomics instead of gathering through the RowIndex;
 * the caller must keep those key columns alive and unchanged while the handle is used.
 * Results are identical to dtb_reduce (floating sums up to association order).
 */
DTB_API int dtb_groupby_reduce(dtb_groupby* g, int op, dtb_col value, int64_t nrows_value,
                       dtb_stream stream, void* out);

/*
 * The same reducer fed piecewise: the value column arrives in row ranges (e.g. the chunks of a host
 * column on their way over PCIe, each folded as soon as it is in HBM -- the reference's reducers,
 * column/sumprod.h / minmax.h / count.h, need the whole column before they start).  Streaming path only
 * (see dtb_groupby_reduce: small key domain, device key columns) and DTB_OP_SUM .. DTB_OP_COUNTNA;
 * otherwise _begin returns DTB_ENOTIMPL and the caller uses dtb_groupby_reduce on the whole column.
 *   _begin : allocates and initialises the accumulator tables
 *   _add   : value_rows = DEVICE pointer to rows [row0, row0 + nrows) of the value column, enqueued on `stream`
 *            (the caller orders it after the piece's upload); every row exactly once over all calls
 *   _end   : finalises into out (host or device, ngroups elements of dtb_reduce_out_stype) and frees the state
 *            (also on error).  Results as dtb_groupby_reduce.
 * Float DTB_OP_MIN / DTB_OP_MAX: the sign of a zero result is that of the group's first valid zero in RowIndex
 * order, and the values are gone by _end.  So the state also holds the inverse RowIndex, int32[nrows] (4 GB at
 * 1e9 rows, for every such state alive at once), built by _begin, and the first zero of every group
 * (uint64[ngroups]); every _add makes one more pass over its rows to update it.
 */
typedef struct dtb_reduce_state dtb_reduce_state;
DTB_API int dtb_groupby_reduce_begin(dtb_groupby* g, int op, int value_stype, dtb_stream stream, dtb_reduce_state** out);
DTB_API int dtb_groupby_reduce_add(dtb_reduce_state* st, const void* value_rows, int64_t row0, int64_t nrows, dtb_stream stream);
DTB_API int dtb_groupby_reduce_end(dtb_reduce_state* st, dtb_stream stream, void* out);

/*
 * dtb_reduce2 -- cov / corr per group (expr/head_reduce_binary.cc:114-221): the columns x and y, both viewed
 * through the RowIndex `order` (NULL = identity; order_is64: int64 row ids), segmented by `offsets`; arguments as in
 * "Per-group functions".  nrows_value: rows in each of x and y (bounds the gather).
 *   out : ngroups elements of stype dtb_reduce2_out_stype(op, x.stype, y.stype): FLOAT32 when both columns are
 *         FLOAT32, FLOAT64 otherwise (bool and integer columns included); 0 = invalid combination.
 * Only rows where both values are valid count; m = their number.  COV is NA when m <= 1, else
 * sum (x - mx)(y - my) / (m - 1).  CORR is NA unless m > 1 and sxx * syy > 0, else sxy / sqrt(sxx * syy), not
 * clamped.  Accuracy: both columns are widened to float64 (deviation: the reference computes in float32 when both
 * are float32) and the groups are folded in two passes over the values shifted by the group's first valid pair
 * (px, py) -- sums of x - px, y - py, then of the products of the deviations from those shifted means -- instead of
 * the reference's Welford recurrence, in an unspecified order.  Each accumulated sum has the error of a float64
 * summation in any order, gamma(m-1) * sum of |terms|; the result is rounded once to the output stype.  A group
 * whose x (or y) values are all equal gives exactly cov = 0 and corr = NA, as the reference does.
 */
DTB_API int dtb_reduce2_out_stype(int op, int stype_x, int stype_y);
DTB_API int dtb_reduce2(int op, dtb_col x, dtb_col y, int64_t nrows_value, const void* order, int order_is64,
                const void* offsets, int64_t ngroups, dtb_stream stream, void* out);
/* dtb_reduce2 over the handle's RowIndex / offsets (always through the RowIndex: there is no streaming variant). */
DTB_API int dtb_groupby_reduce2(dtb_groupby* g, int op, dtb_col x, dtb_col y, int64_t nrows_value,
                        dtb_stream stream, void* out);

/*
 * dtb_cumulative -- cumsum / cumprod / cummin / cummax inside every group: replaces CumSumProd_ColumnImpl
 * (column/cumsumprod.h) and CumMinMax_ColumnImpl (column/cumminmax.h) as FExpr_CumSumProd / FExpr_CumMinMax run
 * them (expr/fexpr_cumsumprod.cc, expr/fexpr_cumminmax.cc).  op: DTB_OP_SUM, DTB_OP_PROD, DTB_OP_MIN or DTB_OP_MAX.
 * The value column is seen through `order` (NULL = identity; order_is64: int64 row ids) and cut by `offsets`;
 * arguments as in "Per-group functions".  reverse != 0 scans every group from its last position to its first.
 *   out : offsets[ngroups] elements of stype dtb_cumulative_out_stype(op, value.stype), out[p] for position p of
 *         the RowIndex (the GtoALL layout of the grouped frame): SUM / PROD give INT64 for bool and int8-64 and keep FLOAT32 /
 *         FLOAT64; MIN / MAX keep the column's stype (bool, int8-64, float32/64, date32, time64).  0 = refused.
 * Errors: another op, or a stype the op refuses, gives DTB_EINVAL; an stype without a fixed width DTB_ENOTIMPL.
 *
 * SUM / PROD: an NA row adds 0 or multiplies by 1, so no result is NA except a NaN the arithmetic makes (inf - inf,
 * 0 * inf), which then stays for the rest of the group.  Integer results wrap modulo 2^64 and are bit-exact.
 * MIN / MAX: an NA row repeats the previous result, which is NA until the group's first valid row; the update is
 * prev < val ? prev : val (> for MAX), so of equal values the later row wins (-0.0 and +0.0 are equal).  Bit-exact.
 * Float SUM is accumulated in float64 in a fixed, unspecified order, starting at -0.0: the prefix of k rows is
 * within gamma(k-1) * sum|x| of the exact prefix sum, gamma(k) = k*u / (1 - k*u), u = 2^-53, rounded once to the
 * output stype.  Float PROD keeps the significand and the binary exponent apart, as dtb_reduce's PROD does: the
 * prefix of k valid finite non-zero rows is the exact product times (1 + d), |d| <= gamma(k-1), rounded once; a zero
 * and an infinity in the prefix give NA; a zero alone gives 0 and an infinity alone inf, signed by the parity of the
 * negative rows.  Deviations from the reference, which sums and multiplies in order in the column's own type:
 * float32 is accumulated in float64; a cancelling prefix sum can differ from the sequential one by the bound above,
 * in relative terms without limit; where the reference's running sum or product overflows or underflows part-way
 * although the exact prefix is in range, the engine returns the in-range value (so such a prefix that also holds a
 * zero or an inf is not NA here).  Results are deterministic: two calls on the same input give the same bytes.
 * Up to INT32_MAX positions.
 */
DTB_API int dtb_cumulative_out_stype(int op, int stype);
DTB_API int dtb_cumulative(int op, int reverse, dtb_col value, int64_t nrows_value, const void* order,
                           int order_is64, const void* offsets, int64_t ngroups, dtb_stream stream, void* out);

/*
 * dtb_shift, dtb_fillna, dtb_group_index -- the row functions that return one value per position inside every group
 * (the GtoALL layout of the grouped frame).  Like dtb_cumulative, the value column is seen through `order` (NULL =
 * identity; order_is64: int64 row ids) and cut by `offsets`; arguments as in "Per-group functions".
 * Up to INT32_MAX positions.  out holds offsets[ngroups] elements, out[p] for position p of the RowIndex.  Results
 * are deterministic: every output element is computed by one thread, so two calls give the same bytes.
 *
 * dtb_shift: replaces compute_lag_rowindex (expr/head_func_shift.cc:40-64) and Shift_ColumnImpl (column/shift.h:37-88).
 *   out[p] = value[order[p - n]] when p - n lies in p's group, else NA: n > 0 lags, n < 0 leads, n = 0 gathers the
 *   column, and |n| >= the group's size gives a group of NA.  out has value.stype (every fixed-width stype).  The rule
 *   holds for every int64 n, where the reference computes p - n in int32 and compares against nrows - |n| in size_t
 *   (so its results for |n| beyond the positions come from overflow and are not followed).  NA: a source that is NA,
 *   or outside the group, gives the stype's NA (a float NaN comes out as the quiet NaN 0x7FC00000 / 0x7FF8...);
 *   every valid value keeps its bits, -0.0 included.  Bit-exact.
 * dtb_fillna: replaces fill_rowindex (expr/fexpr_fillna.cc:66-118): fillna(cols) without a value.  out[p] = the
 *   latest valid value of p's group at or before p (reverse != 0: the earliest at or after p), or NA where there is
 *   none.  out has value.stype.  NA and bits as for dtb_shift; bit-exact.  fillna(cols, value=) is not this call.
 * dtb_group_index: replaces CumcountNgroup_ColumnImpl (column/cumcountngroup.h:30-73).  Writes int64[offsets[ngroups]]:
 *   DTB_GROUP_CUMCOUNT  p - start of p's group (reverse != 0: end - 1 - p);
 *   DTB_GROUP_NGROUP    the index g of p's group (reverse != 0: ngroups - 1 - g).
 *   Never NA.
 */
#define DTB_GROUP_CUMCOUNT 1
#define DTB_GROUP_NGROUP   2
DTB_API int dtb_shift(dtb_col value, int64_t nrows_value, const void* order, int order_is64,
                      const void* offsets, int64_t ngroups, int64_t n, dtb_stream stream, void* out);
DTB_API int dtb_fillna(int reverse, dtb_col value, int64_t nrows_value, const void* order, int order_is64,
                       const void* offsets, int64_t ngroups, dtb_stream stream, void* out);
DTB_API int dtb_group_index(int kind, int reverse, const void* offsets, int64_t ngroups,
                            dtb_stream stream, void* out);

/*
 * dtb_gather -- replaces materialisation of ArrayView_ColumnImpl<int32/int64>
 * (column/view.cc:88-155): out[i] = order[i] < 0 ? NA : src[order[i]].
 */
DTB_API int dtb_gather(dtb_col src, int64_t nrows_src,
               const void* order, int order_is64, int64_t n,
               dtb_stream stream, void* out);

/*
 * dtb_slice_groups -- the `i` node of DT[i, j, by(), sort()] when i is an integer slice (or an integer: the
 * slice [i, i+1)); replaces FExpr_Literal_SliceInt::evaluate_iby (expr/fexpr_literal_sliceint.cc:82-170) and
 * FExpr_Literal_Int::evaluate_iby (expr/fexpr_literal_int.cc:146-192): the slice is applied inside every group
 * of the grouped frame.  offsets: int32[ngroups+1] (the Groupby; one group [0, n] under sort() alone).
 * start / stop / step: DTB_SLICE_NA for a missing member; step 0 = `stop` copies of row `start` (the reference's
 * repeat slice).  rows_out: int32 positions INTO THE ROWINDEX of group() (the caller composes: RowIndex product =
 * dtb_gather on the index buffer, eval_context.cc:154-163), at most rows_capacity of them (DTB_ENOSPACE with
 * *nrows_out = the number needed otherwise; the grouped frame's row count always suffices for step != 0);
 * offsets_out: int32[ngroups+1], the remaining groups -- groups that select nothing disappear.
 * Host or device pointers.
 */
#define DTB_SLICE_NA INT64_MIN
DTB_API int dtb_slice_groups(const void* offsets, int64_t ngroups, int64_t start, int64_t stop, int64_t step,
                     dtb_stream stream, void* rows_out, int64_t rows_capacity, void* offsets_out,
                     int64_t* ngroups_out, int64_t* nrows_out);

/*
 * dtb_mask_rows -- the `i` node of DT[i, j] when i is a boolean column (DT[f.b, j], DT[dt.Frame(b), j]); replaces
 * ArrayRowIndexImpl::init_from_boolean_column (rowindex_array.cc:130-170).  mask: a bool8 column of nrows rows
 * (0 <= nrows <= INT32_MAX).  rows_out receives the ascending int32 positions of the rows whose byte is neither 0
 * nor the NA -128, at most rows_capacity of them (DTB_ENOSPACE with *nrows_out = the number needed otherwise;
 * nrows always suffices); *nrows_out = how many.  Two passes over the mask (count per tile, scan, emit); the call
 * waits once, for the count.  The arguments are checked, in this order, before any CUDA call: nrows_out NULL,
 * stype, nrows, rows_capacity < 0, mask data NULL (nrows > 0), rows_out NULL (rows_capacity > 0): DTB_EINVAL.
 * Host or device buffers.
 */
DTB_API int dtb_mask_rows(dtb_col mask, int64_t nrows, dtb_stream stream, void* rows_out, int64_t rows_capacity,
                          int64_t* nrows_out);

/*
 * dtb_int_rows -- the `i` node of DT[i, j] when i is an integer column (DT[dt.Frame(idx), j]); the checks and the
 * RowIndex of FExpr_Frame::evaluate_i (expr/fexpr_frame.cc:175-198) and RowIndex(const Column&)
 * (rowindex_array.cc:63-128).  sel: an int8 / int16 / int32 / int64 column of nrows rows (<= INT32_MAX).
 * *min_out / *max_out: the smallest / largest valid value (0 when every value is NA), *nacount_out: the NA values;
 * the caller checks them against the frame's rows.  rows_out: int32[nrows], sel's values in its order with NA as
 * INT32_MIN (the NA row); it may be NULL for an int32 column, which is the RowIndex as it stands.  The call waits
 * once, for the statistics.  The arguments are checked, in this order, before any CUDA call: min_out / max_out /
 * nacount_out NULL, stype, nrows, selector data NULL (nrows > 0), rows_out NULL (nrows > 0, not int32): DTB_EINVAL.
 * Host or device buffers.
 */
DTB_API int dtb_int_rows(dtb_col sel, int64_t nrows, dtb_stream stream, void* rows_out, int64_t* min_out,
                         int64_t* max_out, int64_t* nacount_out);

/*
 * dtb_sort_grouped -- replaces Column::sort_grouped (sort.cc:1499-1530): reorders the rows INSIDE every
 * group of (order, offsets) by `value` ascending, NA first, stable; the groups themselves stay where
 * they are.  order: int32 RowIndex; arguments as in "Per-group functions", order_out is its `out`.
 * order_out: int32[offsets[ngroups]].  DTB_OP_MEDIAN / DTB_OP_NUNIQUE expect this order
 * (the reference's Median_ColumnImpl calls sort_grouped in its pre_materialize_hook).
 */
DTB_API int dtb_sort_grouped(dtb_col value, int64_t nrows_value, const void* order, const void* offsets,
                     int64_t ngroups, dtb_stream stream, void* order_out);

/*
 * dtb_qcut -- replaces Qcut_ColumnImpl::materialize (column/qcut.h:78-155) run on every group, as
 * FExpr_Qcut::evaluate_n does under by() (expr/fexpr_qcut.cc:64-158).  The value column is seen through `order`
 * (int32 RowIndex; NULL = identity) and cut by `offsets`; arguments as in "Per-group functions".  Inside every
 * group the distinct values are numbered
 * i = 0 .. G-1 in group()'s order, NA first; has_na = the first one is NA, V = G - has_na, q = nquantiles:
 *   V <= 1:  a = 0, b = (q - 1) / 2 (integer division)
 *   else:    a = q * (1 - FLT_EPSILON) / (V - 1), b = -a * has_na
 * and every row of value i gets int32(a * i + b), truncated; the rows of the NA value get NA.
 *   - Values are told apart as group() tells them: -0.0 and +0.0 are different values, every NaN is the NA value.
 *   - a * i + b is a multiply and an add, each rounded to nearest (no fused multiply-add), as the reference
 *     computes it.
 * out: int32[offsets[ngroups]], out[p] = the bin of the row at position p of the RowIndex (the GtoALL layout of
 * the grouped frame).  nquantiles <= 0: DTB_EINVAL.  Up to INT32_MAX rows.
 */
DTB_API int dtb_qcut(dtb_col value, int64_t nrows_value, const void* order, const void* offsets, int64_t ngroups,
                     int nquantiles, dtb_stream stream, void* out);

/*
 * dtb_cut -- replaces CutNbins_ColumnImpl and CutBins_ColumnImpl (column/cut.h:91-281) as FExpr_Cut::evaluate_n runs
 * them over a whole column (expr/fexpr_cut.cc:88-170; the reference refuses cut() under by()).  The value column
 * (nrows_value rows) is seen through `order`: n positions, int32 row ids or int64 when order_is64; an index outside
 * [0, nrows_value) is an NA row, as in dtb_gather.  order NULL = the identity, and then n must be 0 or nrows_value.
 * Values are compared and scaled as float64: int64 rounded to nearest, NaN and the integer sentinels are NA.
 *   edges NULL (nbins mode): min and max of the valid values at the n positions, as float64.  No valid value, or an
 *     infinite min or max: every row is NA.  Else, rc = right_closed != 0:
 *       min == max:  a = 0, b = (nbins - rc) / 2 (integer division), shift = 0
 *       else:        a = (1 - FLT_EPSILON) * nbins / (max - min), b = -a * min, shift = 0 (rc), or
 *                    b = -a * max, shift = nbins - 1 (not rc); max - min may overflow to inf, giving a = 0
 *     and every valid v gets int32(a * v + b) + shift.  a * v + b is a multiply and an add, each rounded to nearest
 *     (no fused multiply-add), as the reference computes it.  int32(r) truncates, and is INT32_MIN for a NaN or an r
 *     outside the int32 range (x86-64's conversion, which the reference's static_cast compiles to); the add of shift
 *     wraps.  The coefficients are computed on the device: the call does not wait for the statistics.
 *   edges != NULL: a host float64[nedges] array, nedges >= 2, strictly increasing; nbins is ignored.  With
 *     c = #{k : edges[k] < v} (right_closed) or #{k : edges[k] <= v} (not), v gets c - 1 when 1 <= c <= nedges - 1,
 *     i.e. v in (edges[0], edges[nedges-1]] (right_closed) or [edges[0], edges[nedges-1]); else NA.  That is the
 *     reference's bisection with v > e or v >= e.
 * out: int32[n], out[p] = the bin of the row at position p, NA as INT32_MIN.  Host or device pointers (edges: host).
 * Bit-exact.  Asynchronous unless out is host memory.  Arguments are checked in this order, on the host before any
 * CUDA call: nbins <= 0 (nbins mode), or nedges < 2, a NaN edge, edges not strictly increasing: DTB_EINVAL; an stype
 * without a fixed width: DTB_ENOTIMPL; date32 / time64: DTB_EINVAL; n < 0 or nrows_value < 0, value data NULL while
 * nrows_value > 0, order NULL while 0 < n != nrows_value, out NULL while n > 0: DTB_EINVAL.  n == 0 then returns at once.
 */
DTB_API int dtb_cut(dtb_col value, int64_t nrows_value, const void* order, int order_is64, int64_t n, int nbins,
                    const double* edges, int64_t nedges, int right_closed, dtb_stream stream, void* out);

/* the parts of dtb_time_part: YearMonthDay_ColumnImpl<1..3> (expr/time/fexpr_year_month_day.cc), DayOfWeek_ColumnImpl
 * (fexpr_day_of_week.cc), HourMinSec_ColumnImpl<1..4> (fexpr_hour_min_sec.cc) */
#define DTB_TIME_YEAR         1
#define DTB_TIME_MONTH        2
#define DTB_TIME_DAY          3
#define DTB_TIME_DAY_OF_WEEK  4
#define DTB_TIME_HOUR         5
#define DTB_TIME_MINUTE       6
#define DTB_TIME_SECOND       7
#define DTB_TIME_NANOSECOND   8

/*
 * dtb_time_part -- one calendar or clock part of a date32 or time64 column, as dt.time.year() .. nanosecond() compute
 * it.  The value column (nrows_value rows) is seen through `order`: n positions, int32 row ids or int64 when
 * order_is64; an index outside [0, nrows_value) is an NA row, as in dtb_gather.  order NULL = the identity, and then n
 * must be 0 or nrows_value.  NA (INT32_MIN / INT64_MIN) gives NA.
 *   date32 v (days since 1970-01-01): YEAR / MONTH / DAY of the proleptic Gregorian calendar, DAY_OF_WEEK 1 (Monday)
 *     .. 7 (Sunday).  Day numbers near the ends of the int32 range wrap in the conversion's int32 adds, as the
 *     reference's do.
 *   time64 v (nanoseconds since 1970-01-01T00:00): the four above of the day floor(v / DAY) (the time64 -> date32
 *     cast; for v < 0 it computes v - (DAY - 1) with int64 wrap-around), and HOUR / MINUTE / SECOND / NANOSECOND
 *     = ((v mod DAY) / SCALE) % MODULO with the floor modulo, DAY = 86400e9 ns.
 * out: int32[n], out[p] = the part of the row at position p, NA as INT32_MIN.  Host or device pointers.  Bit-exact.
 * Asynchronous unless out is host memory.  Arguments are checked in this order, on the host before any CUDA call:
 * part outside DTB_TIME_YEAR .. DTB_TIME_NANOSECOND: DTB_EINVAL; an stype without a fixed width: DTB_ENOTIMPL; an stype
 * other than date32 / time64, or a clock part (HOUR .. NANOSECOND) of date32: DTB_EINVAL; n < 0 or nrows_value < 0,
 * value data NULL while nrows_value > 0, order NULL while 0 < n != nrows_value, out NULL while n > 0: DTB_EINVAL.
 * n == 0 then returns at once.
 */
DTB_API int dtb_time_part(int part, dtb_col value, int64_t nrows_value, const void* order, int order_is64, int64_t n,
                          dtb_stream stream, void* out);

/*
 * dtb_set_select -- the group-selection step of union / intersect / setdiff / symdiff
 * (set_funcs.cc:126-456).  The caller concatenated K single-column inputs (input k holds the rows
 * cum_sizes[k-1] .. cum_sizes[k]-1), grouped the result with dtb_group and passes its (order, offsets).
 * rows_out: int32[ngroups] receives, for every group that the operation keeps, the row index of the
 * group's first row (ascending group order); *nout = how many.  Gathering the concatenated column
 * through rows_out gives the result column.
 */
DTB_API int dtb_set_select(int mode, const void* order, const void* offsets, int64_t ngroups,
                   const int64_t* cum_sizes, int ninputs, dtb_stream stream, void* rows_out, int64_t* nout);

/*
 * dtb_largest_group -- the mode / nmodal scan of NumericStats<T>::compute_sorted_stats
 * (stats.cc:984-991): index and size of the first largest group among groups [skip, ngroups)
 * (skip = 1 when the first group holds the NA rows).  *index_out = -1 when there is no such group.
 */
DTB_API int dtb_largest_group(const void* offsets, int64_t ngroups, int64_t skip, dtb_stream stream,
                      int64_t* index_out, int64_t* size_out);

/*
 * dtb_join -- replaces natural_join(xdt, jdt) (frame/join.cc:392-470): for every row of X the index
 * of the row of the keyed frame J whose key columns all compare equal (FwCmp, join.cc:199-232: NA
 * matches NA; an X value that J's integer key type cannot represent matches nothing), or the NA
 * index INT32_MIN.  jkeys must be sorted ascending, NA first, with unique rows -- what setting a key
 * produces (DataTable::set_key, frame/key.cc:118-180 = dtb_group + uniqueness check + dtb_gather).
 * index_out: int32[nrows_x], the ARR32 RowIndex the reference applies to J's non-key columns.
 */
DTB_API int dtb_join(const dtb_col* xkeys, const dtb_col* jkeys, int nkeys, int64_t nrows_x, int64_t nrows_j,
             dtb_stream stream, void* index_out);

/*
 * dtb_join_gather -- dtb_join that also reads J's columns through the match: for each of the nvals fixed-width
 * columns jvals[c] (nrows_j rows, J's row order) vals_out[c][r] = jvals[c][match of X row r], or the stype's NA
 * where X row r matches nothing -- the column of J that a query sees through natural_join's RowIndex
 * (eval_context.cc:577-582), without materialising the index.  index_out may be NULL (then nvals >= 1);
 * dtb_join is the nvals = 0 case.  Same lookup, same key rules.  A single integer / date32 / time64 key column of J
 * whose valid keys are consecutive is addressed directly instead of searched.  Host or device buffers.
 */
DTB_API int dtb_join_gather(const dtb_col* xkeys, const dtb_col* jkeys, int nkeys, int64_t nrows_x, int64_t nrows_j,
                    const dtb_col* jvals, int nvals, dtb_stream stream, void* index_out, void* const* vals_out);

/*
 * Multi-GPU merge of per-group partials over a small group-key domain (one process per GPU; the
 * reference is single-process, SURVEY.md 8e -- this is north_star's "final NCCL reduce of per-group
 * partials").  Each rank scatters its (group key, 8-byte partial) list into a dense table indexed by
 * key - kmin; the caller all-reduces `table` (SUM, typed as the partials are) and `present` (uint32
 * SUM) in place with NCCL; dtb_dense_compact then lists the keys that occur on any rank, ascending,
 * with their merged partials.  Device buffers only.  table/present must be zeroed before the scatter;
 * table_size: multiple of 1024, at most 2^22 (both functions refuse any other with DTB_EINVAL).  key_stype:
 * DTB_STYPE_INT32 or DTB_STYPE_INT64.  The scatter skips a key outside [kmin, kmin + table_size): the caller
 * chooses kmin and the size so that every key fits, or counts the keys that do not.
 */
DTB_API int dtb_dense_scatter(const void* keys, int key_stype, const void* vals, int64_t n, int64_t kmin,
                      int64_t table_size, void* table, void* present, dtb_stream stream);
DTB_API int dtb_dense_compact(const void* table, const void* present, int64_t table_size, int64_t kmin,
                      int key_stype, void* out_keys, void* out_vals, int64_t* ngroups_out, dtb_stream stream);

/*
 * dtb_lower_bound -- out[i] (int64) = number of rows of the ascending, NA-free column `sorted` that are
 * smaller than values[i]: the cut points of the key-range exchange between GPUs (no reference analogue;
 * SURVEY.md 8e).  Both columns share one stype.
 */
DTB_API int dtb_lower_bound(dtb_col sorted, int64_t nrows, dtb_col values, int64_t nvalues,
                    dtb_stream stream, void* out);

/*
 * Residency bracket for HOST buffers: between dtb_cache_begin() and the matching dtb_cache_end() (calls
 * nest; per thread) a host input staged into HBM by any entry point stays there and is reused by later
 * calls that pass the same (pointer, size); the RowIndex / offsets that dtb_group copied to host memory
 * are remembered too, so dtb_reduce / dtb_gather on them upload nothing.  The reference-side hook puts
 * the bracket around EvalContext::evaluate() (INTEGRATION.md): one upload per column per query, where the
 * reference's Buffers are host memory (buffer.cc:261-300).  The caller promises that the bracketed host
 * buffers do not change; dtb_cache_end() releases the copies.  dtb_last_call_stats().cache_hits counts the
 * cache hits of the last call.
 */
DTB_API int dtb_cache_begin(void);
DTB_API int dtb_cache_end(void);

/* Copies nbytes between any two host/device buffers on `stream`
 * (cudaMemcpyDefault) and waits for completion.  Lets a binding read the
 * HBM-resident results of a dtb_groupby without linking the CUDA runtime. */
DTB_API int dtb_memcpy(void* dst, const void* src, int64_t nbytes, dtb_stream stream);

/*
 * Engine options, the analogue of dt.options.sort.* (sort.cc:259-349).
 *   "radix_bits"   largest digit width of the LSD passes: 4..8, or 0 (default) = 8 bits (wider digits were
 *                  built and measured slower three times, the last time on H100, DESIGN.md 4.2)
 *   "verbose"      1 = print the pass plan to stderr: the key columns' bits and shifts, and per sort round
 *                  its passes, the pass that narrows 64-bit keys to 32 bits (-1 = none), whether the first pass
 *                  takes the statistics kernel's histogram, and whether the last pass fills the count table
 *   "profile"      1 = bracket every kernel with CUDA events on the call's stream (the calls do not wait for
 *                  them; dtb_profile_count / dtb_profile_reset do)
 *   "bucketed_reducers" 1 (default) = value columns that would cost two or more L2 atomics per row (mean, or
 *                  several reducers of one column) take the bucketed multi-reducer (dtb_bucket.cu); 0 = always
 *                  one streaming pass per reducer
 *   "trim_scratch" (set only) release the calling thread's cached HBM scratch slab and the memory the current
 *                  device's stream-ordered pool keeps from freed handles
 */
DTB_API int dtb_set_option(const char* name, int64_t value);
DTB_API int dtb_get_option(const char* name, int64_t* value);

/* Kernel timings collected while option "profile" is on (accumulated on the calling
 * thread until dtb_profile_reset): record i = (kernel family name, milliseconds).
 * dtb_profile_count waits for the recorded events of earlier calls before it answers. */
DTB_API int dtb_profile_count(void);
DTB_API int dtb_profile_get(int i, char* name, int cap, double* ms);
DTB_API int dtb_profile_reset(void);

/* Per-call statistics of the last dtb_group / dtb_groupby_create on this thread:
 * number of kernels launched, radix passes, significant key bits. */
typedef struct dtb_call_stats {
  int32_t kernels_launched;
  int32_t radix_passes;
  int32_t key_bits;
  int32_t cache_hits;        /* host inputs served from the dtb_cache_begin/end residency cache */
  int64_t scratch_bytes;
} dtb_call_stats;
DTB_API int dtb_last_call_stats(dtb_call_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* DTB200_H */
