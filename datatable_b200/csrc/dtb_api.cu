// dtb_api.cu -- the C-ABI (include/dtb200.h): call planning, HBM scratch,
// host<->device staging and error reporting.  No compute happens on the host:
// without a CUDA device every entry point whose arguments pass the host checks
// fails with DTB_ECUDA.
#include <stdio.h>
#include <chrono>
#include <string.h>
#include <mutex>
#include <optional>
#include <string>
#include <vector>
#include "dtb_common.cuh"

namespace dtb {

// ---------------------------------------------------------------------------
// thread-local state
// ---------------------------------------------------------------------------
static thread_local std::string t_error;
static thread_local dtb_call_stats t_stats = {0, 0, 0, 0, 0};

void set_error(const std::string& msg) { t_error = msg; }
void count_launch(int n) { t_stats.kernels_launched += n; }

// ---------------------------------------------------------------------------
// options (analogue of dt.options.sort.*, sort.cc:259-349)
// ---------------------------------------------------------------------------
static int64_t opt_radix_bits = 0;     // 0 = default (8-bit digits); 4..8 = largest digit width
static int64_t opt_verbose = 0;
static int64_t opt_profile = 0;
static int64_t opt_bucketed = 1;       // 1 = columns with >= 2 L2 atomics per row take the bucketed multi-reducer (dtb_bucket.cu)

// ---------------------------------------------------------------------------
// optional per-kernel timing with CUDA events on the launching stream
// (option "profile"): the reference only times whole calls (call_logger.cc:153-174)
// ---------------------------------------------------------------------------
struct ProfRec { const char* name; cudaEvent_t a, b; };
static thread_local std::vector<ProfRec> t_prof_open;
static thread_local std::vector<std::pair<std::string, double>> t_prof_done;

ProfScope::ProfScope(const char* name_, cudaStream_t stream) : on(opt_profile != 0), s(stream), name(name_) {
  if (!on) return;
  cudaEventCreate(&a); cudaEventCreate(&b);
  cudaEventRecord(a, s);
}
ProfScope::~ProfScope() { if (on) { cudaEventRecord(b, s); t_prof_open.push_back({name, a, b}); } }

// Lazy: the calls only record events; the first query (dtb_profile_count / _reset) waits for them.  (A sync at the
// end of every profiled call kept the host from running ahead and lengthened bench.py's timed steps.)
static void prof_collect() {
  for (auto& r : t_prof_open) {
    float ms = 0.f;
    if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess)
      t_prof_done.emplace_back(r.name, (double)ms);
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  t_prof_open.clear();
}

// ---------------------------------------------------------------------------
// per-device context: the stream-ordered memory pool keeps scratch resident
// ---------------------------------------------------------------------------
static std::mutex g_ctx_mutex;
static bool g_ctx_ready[64] = {false};

static thread_local double t_tl0 = 0;   // start of the current group() call (DTB_TL)
static double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
#define DTB_TL(label) do { if (opt_verbose >= 2) fprintf(stderr, "[dtb200]   t=%9.3f ms  %s\n", now_ms() - t_tl0, label); } while (0)

// Waits for the stream by polling.  cudaStreamSynchronize parks the thread (the context is usually created by the
// host framework with the default scheduling policy) and wakes it 50-100 us after the stream drained; group() has
// two such waits on its critical path (the statistics, the number of groups) with the GPU idle behind them.
static cudaError_t stream_wait(cudaStream_t s) {
  cudaError_t e;
  while ((e = cudaStreamQuery(s)) == cudaErrorNotReady) {}
  return e;
}

static int ensure_context() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_error(std::string("no usable CUDA device: ") + cudaGetErrorString(e));
    return DTB_ECUDA;
  }
  if (dev < 0 || dev >= 64) { set_error("device ordinal out of range"); return DTB_EINVAL; }
  if (g_ctx_ready[dev]) return DTB_OK;
  std::lock_guard<std::mutex> lock(g_ctx_mutex);
  if (g_ctx_ready[dev]) return DTB_OK;
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) {
    set_error(std::string("no usable CUDA device: ") + cudaGetErrorString(e));
    return DTB_ECUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    set_error("dtb200 is built for sm_90a (H100) only; device is sm_" + std::to_string(prop.major) +
              std::to_string(prop.minor));
    return DTB_ECUDA;
  }
  cudaMemPool_t pool;
  DTB_CUDA_CHECK(cudaDeviceGetDefaultMemPool(&pool, dev));
  uint64_t thresh = UINT64_MAX;          // keep freed scratch cached in the pool
  DTB_CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
  g_ctx_ready[dev] = true;
  return DTB_OK;
}

// ---------------------------------------------------------------------------
// Scratch arena.  Every API call carves its temporaries out of one HBM slab that the
// calling thread keeps between calls: after the first call of a given size there are
// no allocator calls at all on the hot path (cudaMallocAsync of multi-GB blocks costs
// milliseconds even when the pool already holds the memory).  The slab only grows.
// ---------------------------------------------------------------------------
struct Arena {
  struct Slab { char* p; size_t cap; };
  std::vector<Slab> slabs;
  size_t cur = 0, off = 0;
  int depth = 0;
  int device = -1;              // the slabs (and last_stream) belong to this device
  cudaStream_t last_stream = nullptr;
  bool have_last = false;

  int begin(cudaStream_t s) {
    if (depth++ > 0) return DTB_OK;
    // A thread may move between devices (dtb_init(d) / cudaSetDevice): scratch carved out of another
    // device's slab would be an illegal address, so the arena follows the thread's current device and
    // gives the old device's slabs back first.
    int dev = 0;
    DTB_CUDA_CHECK(cudaGetDevice(&dev));
    if (device != dev) {
      if (device >= 0 && (!slabs.empty() || have_last)) {
        DTB_CUDA_CHECK(cudaSetDevice(device));
        trim();
        DTB_CUDA_CHECK(cudaSetDevice(dev));
      }
      device = dev; have_last = false; last_stream = nullptr;
    }
    // work enqueued by the previous call may still be using the slab on another stream
    if (have_last && last_stream != s) DTB_CUDA_CHECK(cudaStreamSynchronize(last_stream));
    last_stream = s; have_last = true;
    if (slabs.size() > 1) {                         // coalesce what the last call needed into one slab
      size_t total = 0;
      for (auto& sl : slabs) total += sl.cap;
      DTB_CUDA_CHECK(cudaDeviceSynchronize());
      for (auto& sl : slabs) cudaFree(sl.p);
      slabs.clear();
      char* p = nullptr;
      cudaError_t e = cudaMalloc(&p, total);
      if (e != cudaSuccess) { cudaGetLastError(); }   // fall back to growing on demand
      else slabs.push_back({p, total});
    }
    cur = 0; off = 0;
    return DTB_OK;
  }
  void end() { if (depth > 0) depth--; }
  // bytes the current slab can still hand out without an allocator call
  size_t room() const { return cur < slabs.size() ? slabs[cur].cap - off : 0; }
  int take(size_t bytes, void** out) {
    bytes = (bytes + 255) & ~(size_t)255;
    while (cur < slabs.size()) {
      if (off + bytes <= slabs[cur].cap) { *out = slabs[cur].p + off; off += bytes; return DTB_OK; }
      cur++; off = 0;
    }
    size_t cap = bytes < ((size_t)64 << 20) ? ((size_t)64 << 20) : bytes;
    char* p = nullptr;
    cudaError_t e = cudaMalloc(&p, cap);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(" + std::to_string(cap) + " bytes): " + cudaGetErrorString(e));
      cudaGetLastError();
      return e == cudaErrorMemoryAllocation ? DTB_ENOMEM : DTB_ECUDA;
    }
    slabs.push_back({p, cap});
    cur = slabs.size() - 1; off = bytes;
    *out = p;
    return DTB_OK;
  }
  void trim() {
    cudaDeviceSynchronize();
    for (auto& sl : slabs) cudaFree(sl.p);
    slabs.clear(); cur = 0; off = 0;
  }
};
static thread_local Arena t_arena;

struct ArenaScope {
  int rc;
  explicit ArenaScope(cudaStream_t s) { rc = t_arena.begin(s); }
  ~ArenaScope() { t_arena.end(); }
};

// Device buffer: arena scratch by default (lives until the end of the API call), or an owned
// stream-ordered allocation for results that outlive the call (RowIndex / offsets of a handle).
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  cudaStream_t s = nullptr;
  bool owned = false;
  DevBuf() {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  int alloc(size_t nbytes, cudaStream_t stream) {
    release();
    s = stream; bytes = nbytes ? nbytes : 16; owned = false;
    t_stats.scratch_bytes += (int64_t)bytes;
    return t_arena.take(bytes, &p);
  }
  int alloc_owned(size_t nbytes, cudaStream_t stream) {
    release();
    s = stream; bytes = nbytes ? nbytes : 16; owned = true;
    cudaError_t e = cudaMallocAsync(&p, bytes, s);
    if (e != cudaSuccess) {
      p = nullptr;
      set_error("cudaMallocAsync(" + std::to_string(bytes) + " bytes): " + cudaGetErrorString(e));
      cudaGetLastError();
      return e == cudaErrorMemoryAllocation ? DTB_ENOMEM : DTB_ECUDA;
    }
    return DTB_OK;
  }
  void release() { if (p && owned) cudaFreeAsync(p, s); p = nullptr; }
  void* detach() { void* q = p; p = nullptr; return q; }
  template <typename T> T* as() { return reinterpret_cast<T*>(p); }
};

static bool is_device_ptr(const void* p) {
  if (!p) return false;
  cudaPointerAttributes at;
  cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

// Host inputs kept resident in HBM between the calls of one query (dtb_cache_begin / dtb_cache_end): the
// reference-side hook calls dtb_group on the key columns and then dtb_reduce / dtb_gather on the value
// columns and on the RowIndex it just received, all inside one EvalContext::evaluate(); without the cache
// every call uploads its host buffers again.  Entries are keyed by (host pointer, bytes) and are only valid
// while the caller guarantees the host buffers do not change -- the bracket is the caller's promise.
struct InputCache {
  struct Entry { const void* host; size_t bytes; void* dev; int device; };
  std::vector<Entry> entries;
  int depth = 0;
  void* find(const void* p, size_t bytes, int dev) const {
    for (const Entry& e : entries) if (e.host == p && e.bytes == bytes && e.device == dev) return e.dev;
    return nullptr;
  }
  void clear() {
    for (Entry& e : entries) { int cur = 0; cudaGetDevice(&cur); if (cur != e.device) cudaSetDevice(e.device); cudaFree(e.dev); if (cur != e.device) cudaSetDevice(cur); }
    entries.clear();
  }
};
static thread_local InputCache t_cache;

// Input that may live on the host: staged into HBM when needed.
struct DevIn {
  const void* dptr = nullptr;
  DevBuf buf;
  int bind(const void* p, size_t bytes, cudaStream_t s) {
    if (!p || bytes == 0) { dptr = p; return DTB_OK; }
    if (is_device_ptr(p)) { dptr = p; return DTB_OK; }
    if (t_cache.depth > 0) {
      int dev = 0; DTB_CUDA_CHECK(cudaGetDevice(&dev));
      if (void* d = t_cache.find(p, bytes, dev)) { dptr = d; t_stats.cache_hits += 1; return DTB_OK; }
      void* d = nullptr;
      cudaError_t e = cudaMalloc(&d, bytes);
      if (e == cudaSuccess) {
        DTB_CUDA_CHECK(cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, s));
        t_cache.entries.push_back({p, bytes, d, dev});
        dptr = d;
        return DTB_OK;
      }
      cudaGetLastError();                           // no room to keep it: stage it for this call only
    }
    DTB_TRY(buf.alloc(bytes, s));
    DTB_CUDA_CHECK(cudaMemcpyAsync(buf.p, p, bytes, cudaMemcpyHostToDevice, s));
    dptr = buf.p;
    return DTB_OK;
  }
};

// Output that may live on the host: computed in HBM, copied back by finish().
struct DevOut {
  void* dptr = nullptr;
  void* host = nullptr;
  size_t bytes = 0;
  DevBuf buf;
  int bind(void* p, size_t nbytes, cudaStream_t s) {
    bytes = nbytes;
    if (!p) { dptr = nullptr; return DTB_OK; }
    if (is_device_ptr(p)) { dptr = p; return DTB_OK; }
    host = p;
    DTB_TRY(buf.alloc(nbytes, s));
    dptr = buf.p;
    return DTB_OK;
  }
  bool staged() const { return host != nullptr; }
  int finish(size_t nbytes, cudaStream_t s) {
    if (host && nbytes) DTB_CUDA_CHECK(cudaMemcpyAsync(host, dptr, nbytes, cudaMemcpyDeviceToHost, s));
    return DTB_OK;
  }
  // inside a cache bracket: keep a device copy of a result that went to the host (the hook hands the RowIndex
  // of dtb_group straight back to dtb_reduce / dtb_gather)
  static void remember(const void* host_ptr, const void* dev_src, size_t nbytes, cudaStream_t s) {
    if (t_cache.depth <= 0 || !host_ptr || !nbytes) return;
    int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess) return;
    if (t_cache.find(host_ptr, nbytes, dev)) return;
    void* d = nullptr;
    if (cudaMalloc(&d, nbytes) != cudaSuccess) { cudaGetLastError(); return; }
    if (cudaMemcpyAsync(d, dev_src, nbytes, cudaMemcpyDeviceToDevice, s) != cudaSuccess) { cudaGetLastError(); cudaFree(d); return; }
    t_cache.entries.push_back({host_ptr, nbytes, d, dev});
  }
};

static int bitlen(u64 v) { int b = 0; while (v) { b++; v >>= 1; } return b; }
static int ctz64(u64 v) { int c = 0; while (!(v & 1)) { v >>= 1; c++; } return c; }

static bool stype_supported(int st) { return stype_bytes(st) != 0; }

// ---------------------------------------------------------------------------
// group(): validate -> stage the keys, read their statistics (first wait) -> plan -> sort rounds -> offsets
// (second wait) -> fused reducers
// ---------------------------------------------------------------------------
// Reducers evaluated inside the group() call (dtb_groupby_create_reduce).
struct FusedReducers {
  const dtb_reduce_spec* spec = nullptr;
  int n = 0;
  std::vector<void*> out;       // owned device buffers, ngroups elements each
};

// L2 atomics per row that the reducers spec[i..n) of spec[i]'s value column cost on the one-atomic-per-row
// path (mean = sum + count).  For the first reducer of a column: the whole column's cost.
static int column_atomics(const dtb_reduce_spec* spec, int n, int i) {
  int cost = 0;
  for (int j = i; j < n; j++) {
    const dtb_reduce_spec& sj = spec[j];
    if (sj.op == DTB_OP_NROWS || sj.value.data != spec[i].value.data || sj.value.stype != spec[i].value.stype) continue;
    cost += sj.op == DTB_OP_MEAN ? 2 : (sj.op >= DTB_OP_SUM && sj.op <= DTB_OP_COUNTNA ? 1 : 0);
  }
  return cost;
}

// What the direct-address reducers need once the groups are known (small key domains, device-resident key
// columns).  A handle keeps it; it stays valid while the caller keeps the key columns alive and unchanged.
struct DirectGroups {
  bool    on = false;
  int64_t gmax = 0;          // rows of the largest group
  KeyPlan kp;
  int64_t table = 0;
  void*   gkeys = nullptr;   // device uint32[ngroups], an owned allocation
};

struct GroupResult {
  DevBuf order;          // int32[n]
  DevBuf offsets;        // int32[ng+1] (capacity n+1) when groups were requested
  int64_t n = 0;
  int64_t nskip = 0;     // leading NA rows to drop (na_position = remove)
  int64_t ngroups = -1;
  DirectGroups direct;   // its group keys are freed with the result unless a handle takes them
  cudaStream_t s = nullptr;
  ~GroupResult() { if (direct.gkeys) cudaFreeAsync(direct.gkeys, s); }
};

// The reducer's output stype, or the error for a column it cannot reduce.
static int reducer_out_stype(int op, int stype, int& out_st) {
  if (op == DTB_OP_COV || op == DTB_OP_CORR) {
    set_error("cov / corr take two columns: use dtb_reduce2 / dtb_groupby_reduce2"); return DTB_EINVAL;
  }
  out_st = reduce_out_stype_host(op, stype);
  if (out_st) return DTB_OK;
  set_error("Invalid column of stype " + std::to_string(stype) + " in reducer " + std::to_string(op));
  return stype_supported(stype) ? DTB_EINVAL : DTB_ENOTIMPL;
}

// Builds the per-column normalisation from device-computed stats.
static void plan_keys(const dtb_col* keys, const void* const* dptrs, int nkeys, const int* flags,
                      int na_pos, const ColStats* st, KeyPlan& kp)
{
  kp.nkeys = nkeys;
  int total = 0;
  // the last key is the least significant part of the composite
  for (int c = nkeys - 1; c >= 0; c--) {
    KeyNorm& k = kp.k[c];
    const ColStats& cs = st[c];
    k.data = dptrs[c];
    k.stype = keys[c].stype;
    k.desc = (flags[c] & DTB_FLAG_DESCENDING) ? 1 : 0;
    k.pad = 0;
    u64 lo = cs.lo, hi = cs.hi;
    if (cs.nvalid == 0) { lo = hi = 0; }
    const u64 vary = cs.nvalid ? (cs.bits_or ^ cs.bits_and) : 0;
    k.cshift = vary ? ctz64(vary) : 0;
    const u64 rng = (hi - lo) >> k.cshift;                 // values span 0..rng after the shift
    k.edge = k.desc ? hi : lo;
    if (cs.nacount == 0) {                                 // no NA slot needed
      k.inc = 0; k.na_value = 0; k.bits = bitlen(rng);
    } else if (na_pos == DTB_NA_LAST) {                    // sort.cc:749-751: NA -> max-min+1, increment 0
      k.inc = 0; k.na_value = rng + 1; k.bits = bitlen(rng + 1);
    } else {                                               // NA -> 0, values shifted up by one
      k.inc = 1; k.na_value = 0; k.bits = bitlen(rng + 1);
    }
    if (cs.nvalid == 0) { k.bits = 0; k.na_value = 0; }    // all-NA column is constant
    k.lshift = total;
    total += k.bits;
  }
  kp.total_bits = total;
  // groups are defined by the leading by-columns only (sort.cc:1471-1482)
  int gs = 0;
  for (int c = nkeys - 1; c >= 0 && (flags[c] & DTB_FLAG_SORT_ONLY); c--) gs = kp.k[c].lshift + kp.k[c].bits;
  kp.group_shift = gs;
}

static void plan_passes(int total_bits, int width, PassPlan& pp) {
  int np = (total_bits + width - 1) / width;
  if (np < 1) np = 1;
  pp.npasses = np;
  int base = total_bits / np, extra = total_bits % np, sh = 0;
  for (int p = 0; p < np; p++) {
    int b = base + (p < extra ? 1 : 0);
    if (b < 1) b = 1;
    pp.shift[p] = sh; pp.bits[p] = b; sh += b;
  }
}

// One stable sort round over the key columns that fit in 64 bits.
struct RoundPlan {
  KeyPlan  kp;
  bool     has_by;            // holds a by-column: its group boundaries count
  int      key_bytes;         // 4 or 8: the width of its composite keys
  PassPlan pp;
  int      narrow_after;      // 64-bit keys: the passes are planned so that this pass leaves 32 key bits, -1: none
  int      kin_bytes[MAX_PASSES];   // width of the keys pass p reads (pass 0: of the composite)
  int      kout_bytes[MAX_PASSES];  // width of the keys pass p writes, 0: none
  int      kdrop[MAX_PASSES];       // low key bits the keys pass p reads no longer hold (consumed earlier)
  int      low_bits;          // count-table last pass: the low key bits it recovers from the rows' slots, 0: none
  bool     fold;              // the first pass takes its histogram from the statistics kernel
  bool     want_sorted_keys;  // the last pass writes the sorted keys (the offsets and the group keys read them)
  bool     keep_composite;    // the composite keys go to a buffer that the bucketed reducers read again
};

// A value column of the bucketed multi-reducer and the accumulator words its reducers need.
struct BucketCol { const void* data; int stype; bool want[BK_NWORDS]; };

// The accumulator words of the bucketed multi-reducer that `op` finalizes from: {acc0, acc1}, -1 = none.
struct BucketWords { int a0, a1; };
static BucketWords bucket_words(int op, int stype) {
  const bool vflt = stype == DTB_STYPE_FLOAT32 || stype == DTB_STYPE_FLOAT64;
  switch (op) {
    case DTB_OP_SUM:     return {vflt ? BK_SUMF : BK_SUMI, -1};
    case DTB_OP_MEAN:    return {BK_SUMF, BK_CNT};
    case DTB_OP_MIN:     return {BK_MIN, -1};
    case DTB_OP_MAX:     return {BK_MAX, -1};
    case DTB_OP_COUNT:   return {BK_CNT, -1};
    case DTB_OP_COUNTNA: return {BK_CNTNA, -1};
  }
  return {-1, -1};
}

// Everything a group() call decides: from the key columns' statistics, the call's arguments and the options.
struct GroupPlan {
  int     flags[MAX_KEYS];        // effective flags (see plan_group)
  KeyPlan kp;                     // every key column in one composite; the rounds split it
  int64_t nskip = 0;
  bool    groups_k = false;       // group boundaries come from the kernels (some by-column varies)
  std::vector<RoundPlan> rounds;  // least significant first
  bool    fused_raw = false;      // one round of one column: the passes normalise the raw column on the fly
  int     buf_key_bytes = 4;
  int     dbits = 99;             // group-key bits of a single round
  bool    direct_ok = false;      // the groups can be addressed by group key
  bool    count_table = false;    // the last pass counts the rows of every group key; the offsets come from that table
  bool    fused_direct = false;   // the fused reducers stream the rows by group key
  int64_t ctable = 0;             // entries of the count table
  int64_t ftable = 0;             // entries of each streaming reducer's accumulator tables
  std::vector<BucketCol> bcols;   // the bucketed multi-reducer's value columns
  std::vector<int> bcol_of;       // per fused reducer: its column in bcols, or -1
  // The first pass carries the value column of fused reducer region_col, and every fused SUM of that column adds the
  // rows up per digit region of that pass (launch_region_sum) instead of with one L2 atomic per row
  bool    region_sum = false;
  int     region_col = -1;
  dtb_col region_value = {};
};

// What the stages of one group() call share besides the plan: the key columns in HBM and their statistics, the
// sort rounds' scratch, and where the last round left the sorted keys.
struct GroupBufs {
  DevIn  in[MAX_KEYS];
  const void* dptrs[MAX_KEYS];
  bool   staged = false;          // some key column was copied from the host
  bool   fr_streamable = false;   // the fused reducers are sum..nrows over device columns
  ColStats st[MAX_KEYS];
  DevBuf rawhist, rawna;          // single key column: the first pass's histogram
  DevBuf keyA, keyB, idxA, idxB, idxR0, idxR1;
  DevBuf gcount;                  // the count table (GroupPlan::count_table)
  DevBuf facc;                    // the streaming fused reducers' accumulator tables
  DevBuf bxk;                     // the rows' composite keys, kept for the bucketed reducers
  DevBuf vperm, rbases;           // region sum: the values in the first pass's slot order, and that pass's digit bases
  void*  region_keys = nullptr;   // region sum: the keys the first pass wrote
  void*  sorted_keys = nullptr;   // the last round's sorted composite keys
};

// Stages host key columns into HBM and reads their statistics: the call's first wait.  A single key column's
// statistics kernel also counts the low 8 bits of every tile, which becomes the first pass's histogram once edge /
// inc are known (no count kernel, one read of the column less).
static int stage_inputs(const dtb_col* keys, int nkeys, int64_t n, const FusedReducers* fr, cudaStream_t s,
                        GroupBufs& b)
{
  for (int c = 0; c < nkeys; c++) {
    DTB_TRY(b.in[c].bind(keys[c].data, (size_t)n * stype_bytes(keys[c].stype), s));
    b.dptrs[c] = b.in[c].dptr;
    b.staged = b.staged || b.in[c].buf.p != nullptr;
  }
  b.fr_streamable = fr && fr->n > 0;                  // streaming modes exist for sum..nrows only
  for (int i = 0; b.fr_streamable && i < fr->n; i++)
    b.fr_streamable = fr->spec[i].op <= DTB_OP_NROWS &&
                       (fr->spec[i].op == DTB_OP_NROWS || is_device_ptr(fr->spec[i].value.data));
  DevBuf d_stats; DTB_TRY(d_stats.alloc(sizeof(ColStats) * nkeys, s));
  if (nkeys == 1) {
    DTB_TRY(b.rawhist.alloc(stats_hist_bytes(n), s));
    DTB_TRY(b.rawna.alloc(stats_na_bytes(n), s));
    ProfScope ps("col_stats", s);
    DTB_TRY(launch_col_stats_hist(b.dptrs[0], keys[0].stype, n, d_stats.as<ColStats>(), b.rawhist.as<unsigned short>(),
                                  b.rawna.as<unsigned short>(), s));
  } else for (int c = 0; c < nkeys; c++) {
    ProfScope ps("col_stats", s);
    DTB_TRY(launch_col_stats(b.dptrs[c], keys[c].stype, n, d_stats.as<ColStats>() + c, s));
  }
  DTB_CUDA_CHECK(cudaMemcpyAsync(b.st, d_stats.p, sizeof(ColStats) * nkeys, cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(stream_wait(s));
  return DTB_OK;
}

// The plan of a group() call.  Host only: no CUDA call.
static void plan_group(const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t n, const GroupBufs& b,
                       bool want_direct, const FusedReducers* fr, GroupPlan& gp)
{
  // groups come from the leading run of by-columns (sort.cc:1478-1480): a by-column after a SORT_ONLY one only
  // orders the rows, so from the first SORT_ONLY column on every column counts as SORT_ONLY
  for (int c = 0; c < nkeys; c++)
    gp.flags[c] = flags[c] | ((c > 0 && (gp.flags[c - 1] & DTB_FLAG_SORT_ONLY)) ? DTB_FLAG_SORT_ONLY : 0);
  memset(&gp.kp, 0, sizeof(gp.kp));
  plan_keys(keys, b.dptrs, nkeys, gp.flags, na_pos, b.st, gp.kp);
  // sort.cc:598-605; a single row returns before that, NA or not (sort.cc:1435-1439)
  if (na_pos == DTB_NA_REMOVE && n > 1) gp.nskip = (int64_t)b.st[nkeys - 1].nacount;
  if (gp.kp.total_bits == 0) return;                   // every key column is constant

  // by-columns that are all constant (0 bits) while sort columns vary: one group, and no kernel may
  // shift a key by its full width (composite >> group_shift with group_shift == key width is undefined).
  // (A sort-only call has no by-column under the effective flags.)
  int by_bits = 0;
  for (int c = 0; c < nkeys; c++) if (!(gp.flags[c] & DTB_FLAG_SORT_ONLY)) by_bits += gp.kp.k[c].bits;
  gp.groups_k = by_bits > 0;

  // rounds: a composite wider than 64 bits is sorted in several stable rounds, least significant key columns
  // first (the reference refines column by column, sort.cc:561-595; here a round covers as many columns as fit
  // in 64 bits)
  for (int c = nkeys - 1; c >= 0;) {
    int cols[MAX_KEYS], nc = 0, bits = 0;
    while (c >= 0 && bits + gp.kp.k[c].bits <= 64) { cols[nc++] = c; bits += gp.kp.k[c].bits; c--; }
    RoundPlan r; memset(&r, 0, sizeof(r));
    int sh = 0, gs = 0;
    for (int j = 0; j < nc; j++) {
      KeyNorm kn = gp.kp.k[cols[j]];
      kn.lshift = sh; sh += kn.bits;
      r.kp.k[nc - 1 - j] = kn;
      if (gp.flags[cols[j]] & DTB_FLAG_SORT_ONLY) gs = sh; else r.has_by = true;
    }
    r.kp.nkeys = nc; r.kp.total_bits = sh; r.kp.group_shift = gs;
    if (sh > 0) gp.rounds.push_back(r);
  }
  const int nrounds = (int)gp.rounds.size();
  gp.fused_raw = nrounds == 1 && gp.rounds[0].kp.nkeys == 1;
  for (const RoundPlan& r : gp.rounds) if (r.kp.total_bits > 32) gp.buf_key_bytes = 8;

  // Streaming by group key needs one round of at most 22 group-key bits, key columns that are still in
  // device memory after the call, and every row in a group.
  if (nrounds == 1) gp.dbits = gp.rounds[0].kp.total_bits - gp.rounds[0].kp.group_shift;
  gp.direct_ok = gp.groups_k && nrounds == 1 && !b.staged && gp.dbits <= 22 && na_pos != DTB_NA_REMOVE;
  gp.fused_direct = gp.direct_ok && b.fr_streamable;
  // Small key domain + handle path: the last pass counts rows per group key instead of writing
  // the sorted keys, and the offsets come from a scan over that table.
  gp.count_table = want_direct && gp.direct_ok;
  if (gp.count_table) gp.ctable = (int64_t)1 << (gp.dbits < 10 ? 10 : gp.dbits);
  if (gp.fused_direct) gp.ftable = (int64_t)1 << gp.dbits;

  // Bucketed multi-reducer: value columns that would cost two or more L2 atomics per row (mean = sum + count;
  // several reducers of one column) are partitioned by key bucket once and folded in shared memory, all their
  // reducers together (dtb_bucket.cu).
  if (fr) gp.bcol_of.assign(fr->n, -1);
  if (gp.fused_direct && opt_bucketed && gp.dbits >= BK_MIN_DBITS && gp.dbits <= BK_MAX_DBITS)
    for (int i = 0; i < fr->n; i++) {
      const dtb_col& v = fr->spec[i].value;
      if (fr->spec[i].op == DTB_OP_NROWS || gp.bcol_of[i] >= 0 || !reduce_out_stype_host(fr->spec[i].op, v.stype)) continue;
      if (column_atomics(fr->spec, fr->n, i) < 2) continue;
      BucketCol bc = {v.data, v.stype, {}};
      for (int j = i; j < fr->n; j++) {
        const dtb_reduce_spec& sj = fr->spec[j];
        if (sj.op == DTB_OP_NROWS || sj.value.data != v.data || sj.value.stype != v.stype) continue;
        gp.bcol_of[j] = (int)gp.bcols.size();
        const BucketWords w = bucket_words(sj.op, v.stype);
        if (w.a0 >= 0) bc.want[w.a0] = true;
        if (w.a1 >= 0) bc.want[w.a1] = true;
      }
      gp.bcols.push_back(bc);
    }

  int width = (int)opt_radix_bits;                     // digits of at most 8 bits (256 bins), see dtb_radix.cu
  if (width <= 0 || width > 8) width = 8;
  if (width < 4) width = 4;                            // 64 bits / 4 = MAX_PASSES
  for (int ri = 0; ri < nrounds; ri++) {
    RoundPlan& r = gp.rounds[ri];
    r.key_bytes = r.kp.total_bits <= 32 ? 4 : 8;
    plan_passes(r.kp.total_bits, width, r.pp);
    r.want_sorted_keys = ri == nrounds - 1 && gp.groups_k && r.has_by && !gp.count_table;
    // 64-bit keys whose sorted values are not needed afterwards: the passes over the low T-32 bits run
    // on 64-bit keys, the last of them leaves 32 bits, and the remaining passes run on 32-bit keys (8 instead
    // of 12 bytes per row and pass in flight).  Never more passes than before.
    r.narrow_after = -1;
    if (r.key_bytes == 8 && !r.want_sorted_keys && !gp.count_table && width == 8 && r.kp.total_bits > 32) {
      PassPlan lo, hi;
      plan_passes(r.kp.total_bits - 32, width, lo);
      plan_passes(32, width, hi);
      if (lo.npasses + hi.npasses <= r.pp.npasses) {
        r.pp.npasses = lo.npasses + hi.npasses;
        for (int p = 0; p < lo.npasses; p++) { r.pp.shift[p] = lo.shift[p]; r.pp.bits[p] = lo.bits[p]; }
        for (int p = 0; p < hi.npasses; p++) {
          r.pp.shift[lo.npasses + p] = r.kp.total_bits - 32 + hi.shift[p]; r.pp.bits[lo.npasses + p] = hi.bits[p];
        }
        r.narrow_after = lo.npasses - 1;
      }
    }
    // Every pass but the last writes only the key bits later passes read (key >> (shift + bits)), in the narrowest
    // of 1 / 2 / 4 / 8 bytes, and the next pass takes its digit from bit 0: C2's 20-bit keys move 2 + 1 instead of
    // 4 + 4 bytes per row.  Not when the last pass writes the sorted keys.  The last pass of a count table needs the
    // whole group key: it recovers the low bits the earlier passes consumed from the rows' slots, which takes one
    // level of slot regions (at most 3 passes) and a table of 2^low_bits bases (at most 16 bits); beyond that the
    // keys keep their full width.
    const int np = r.pp.npasses;
    const int low = gp.count_table && np > 1 ? r.pp.shift[np - 1] : 0;
    const bool narrow = !r.want_sorted_keys && !(gp.count_table && (np > 3 || low > 16));
    r.low_bits = narrow ? low : 0;
    for (int p = 0; p < np; p++) {
      const bool lastp = p == np - 1;
      const int left = r.kp.total_bits - r.pp.shift[p] - r.pp.bits[p];      // key bits the later passes read
      r.kdrop[p] = narrow && p > 0 ? r.pp.shift[p] : 0;
      r.kin_bytes[p] = p == 0 ? r.key_bytes : r.kout_bytes[p - 1];
      r.kout_bytes[p] = lastp ? (r.want_sorted_keys ? r.key_bytes : 0)
                      : !narrow ? r.key_bytes : left <= 8 ? 1 : left <= 16 ? 2 : left <= 32 ? 4 : 8;
    }
    // single key column: the first pass takes its histogram from the statistics kernel (see stage_inputs)
    r.fold = nkeys == 1 && ri == 0 && gp.fused_raw && r.kp.k[0].cshift == 0 && r.kp.k[0].lshift == 0;
    // multi-column keys whose reducers will take the bucketed path: the composite keys are composed ONCE into a
    // buffer the passes only read, and the bucket kernels read them again afterwards
    r.keep_composite = !gp.bcols.empty() && !gp.fused_raw && nrounds == 1 && r.key_bytes == 4;
  }

  // Region sum: a sum over spread-out group keys (more than SMALL_TABLE, every one in its own accumulator) costs one
  // L2 atomic per row on the direct path.  The first pass puts every row in the region of its first digit and writes
  // the key bits above it; with at most REGION_MAX_LBITS of them a region's groups fit a 64 KB shared-memory table.
  // The pass then carries the value column too, and the next passes must leave its keys alone (at most 3 passes).
  // Few groups in a wide key domain (DIRECT_SMALL, known only after the sort) keep their own path.
  if (gp.fused_direct && gp.fused_raw && gp.bcols.empty() && gp.ftable > SMALL_TABLE) {
    const RoundPlan& r = gp.rounds[0];
    const int np = r.pp.npasses;
    const bool layout = np >= 2 && np <= 3 && r.pp.shift[0] == 0 && r.kp.group_shift == 0 && r.kdrop[1] == r.pp.bits[0] &&
                        (r.kout_bytes[0] == 1 || r.kout_bytes[0] == 2) && gp.dbits - r.pp.bits[0] <= REGION_MAX_LBITS;
    for (int i = 0; layout && i < fr->n; i++)
      if (fr->spec[i].op == DTB_OP_SUM && reduce_out_stype_host(DTB_OP_SUM, fr->spec[i].value.stype)) {
        gp.region_sum = true; gp.region_col = i; gp.region_value = fr->spec[i].value;
        break;
      }
  }
}

// The fused reducer `sp` is a sum over the column the first pass carried (GroupPlan::region_sum).
static bool takes_region_sum(const GroupPlan& gp, const dtb_reduce_spec& sp) {
  return gp.region_sum && sp.op == DTB_OP_SUM && sp.value.data == gp.region_value.data &&
         sp.value.stype == gp.region_value.stype;
}

static void print_plan(const GroupPlan& gp, int64_t n, int nkeys, const ColStats* st) {
  if (!opt_verbose) return;
  const int nrounds = (int)gp.rounds.size();
  fprintf(stderr, "[dtb200] group: n=%lld keys=%d bits=%d rounds=%d\n", (long long)n, nkeys, gp.kp.total_bits, nrounds);
  for (int c = 0; c < nkeys; c++)
    fprintf(stderr, "[dtb200]   key %d: stype=%d desc=%d bits=%d cshift=%d lshift=%d na=%llu\n", c,
            gp.kp.k[c].stype, gp.kp.k[c].desc, gp.kp.k[c].bits, gp.kp.k[c].cshift, gp.kp.k[c].lshift,
            (unsigned long long)st[c].nacount);
  for (int ri = 0; ri < nrounds; ri++) {
    const RoundPlan& r = gp.rounds[ri];
    std::string kw;                                    // key bytes read:written by every pass
    for (int p = 0; p < r.pp.npasses; p++)
      kw += (p ? "," : "") + std::to_string(r.kin_bytes[p]) + ":" + std::to_string(r.kout_bytes[p]);
    fprintf(stderr, "[dtb200]   round %d: keys=%d bits=%d group_shift=%d passes=%d narrow_after=%d fold=%d count_table=%d"
            " key_bytes=%s low_bits=%d\n",
            ri, r.kp.nkeys, r.kp.total_bits, r.kp.group_shift, r.pp.npasses, r.narrow_after, (int)r.fold,
            (int)(gp.count_table && ri == nrounds - 1), kw.c_str(), r.low_bits);
  }
  if (gp.region_sum)                                   // planned: the first pass carries the column
    fprintf(stderr, "[dtb200]   region_sum: reducer=%d stype=%d regions=%d bits_per_region=%d\n", gp.region_col,
            gp.region_value.stype, 1 << gp.rounds[0].pp.bits[0], gp.dbits - gp.rounds[0].pp.bits[0]);
}

// The stable LSD passes of every round; the last round writes the RowIndex into `order`.
static int sort_rounds(GroupPlan& gp, int64_t n, int nfused, int32_t* order, cudaStream_t s, GroupBufs& b)
{
  const int nrounds = (int)gp.rounds.size();
  DTB_TRY(b.keyA.alloc((size_t)n * gp.buf_key_bytes, s));
  DTB_TRY(b.keyB.alloc((size_t)n * gp.buf_key_bytes, s));
  DTB_TRY(b.idxA.alloc((size_t)n * 4, s));
  DTB_TRY(b.idxB.alloc((size_t)n * 4, s));
  if (nrounds > 1) { DTB_TRY(b.idxR0.alloc((size_t)n * 4, s)); }
  if (nrounds > 2) { DTB_TRY(b.idxR1.alloc((size_t)n * 4, s)); }
  if (gp.count_table) {
    DTB_TRY(b.gcount.alloc(sizeof(u32) * (size_t)gp.ctable, s));
    DTB_CUDA_CHECK(cudaMemsetAsync(b.gcount.p, 0, sizeof(u32) * (size_t)gp.ctable, s));
  }
  if (gp.fused_direct) DTB_TRY(b.facc.alloc(sizeof(u64) * (size_t)gp.ftable * 2 * (size_t)nfused, s));
  // The region sum's copy of the values is the last large buffer of the call.  It is taken only if the call's later
  // scratch (offsets scans, group keys, maps, reducer outputs: O(key domain + groups), at most 2^22 entries of a few
  // words each) still fits afterwards, in the arena's slab or in free device memory; otherwise the sum takes the
  // direct path and the arena hands out the same memory as before.
  if (gp.region_sum) {
    const size_t arena_cur = t_arena.cur, arena_off = t_arena.off;
    const int64_t scratch0 = t_stats.scratch_bytes;
    const size_t later = sizeof(u64) * 8 * (size_t)gp.ftable + ((size_t)64 << 20);
    size_t free_b = 0, total_b = 0;
    bool ok = b.rbases.alloc(sizeof(u32) * 256, s) == DTB_OK &&
              b.vperm.alloc((size_t)n * stype_bytes(gp.region_value.stype), s) == DTB_OK;
    if (ok && t_arena.room() < later) ok = cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && free_b >= later;
    if (!ok) {
      cudaGetLastError();
      gp.region_sum = false;
      t_arena.cur = arena_cur; t_arena.off = arena_off;
      t_stats.scratch_bytes = scratch0;
      set_error("");
    }
  }
  DTB_TL("scratch allocated");
  const int32_t* idx_cur = nullptr;        // rows in the order established by the previous rounds
  for (int ri = 0; ri < nrounds; ri++) {
    const RoundPlan& r = gp.rounds[ri];
    const KeyPlan& rk = r.kp;
    const PassPlan& pp = r.pp;
    t_stats.radix_passes += pp.npasses;
    int src_kind = 1;
    if (r.keep_composite) DTB_TRY(b.bxk.alloc(sizeof(u32) * (size_t)n, s));
    if (!gp.fused_raw) {
      ProfScope ps("compose_keys", s);
      DTB_TRY(launch_compose_keys(rk, n, idx_cur, r.keep_composite ? b.bxk.p : b.keyA.p, r.key_bytes, s)); src_kind = 0;
    }

    // per-pass scratch: chunk x digit counts + digit totals/bases
    DevBuf work; DTB_TRY(work.alloc(radix_pass_work_bytes(n), s));

    // the last pass of a count table recovers the consumed low key bits from the rows' slots: their bases are the
    // first pass's digit bases (2 passes) or the scan of the rows per (second digit, first digit) (3 passes)
    DevBuf lowbuf;
    u32* low_base = nullptr; u32* regions = nullptr;
    if (r.low_bits) {
      DTB_TRY(lowbuf.alloc(sizeof(u32) * ((size_t)1 << 16) + sizeof(u32) * 256, s));
      low_base = lowbuf.as<u32>(); regions = low_base + ((size_t)1 << 16);
      if (pp.npasses == 3) DTB_CUDA_CHECK(cudaMemsetAsync(low_base, 0, sizeof(u32) * ((size_t)1 << r.low_bits), s));
    }

    int32_t* round_out = ri == nrounds - 1 ? order : ((ri & 1) ? b.idxR1.as<int32_t>() : b.idxR0.as<int32_t>());
    void* kin = r.keep_composite ? b.bxk.p : b.keyA.p; void* kout = b.keyB.p;
    const int32_t* iin = idx_cur;
    for (int p = 0; p < pp.npasses; p++) {
      const bool last = (p == pp.npasses - 1);
      PassIO io;
      io.src_kind = (p == 0) ? src_kind : 0;
      io.keys_in = kin;
      io.out_shift = last ? 0 : r.kdrop[p + 1] - r.kdrop[p];
      io.out_bytes = r.kout_bytes[p];
      if (r.fold && p == 0 && pp.shift[0] == 0) {
        io.raw_hist = b.rawhist.as<unsigned short>(); io.raw_na = b.rawna.as<unsigned short>();
      }
      if (r.low_bits) {
        if (p == 0) io.bases_out = pp.npasses == 2 ? low_base : regions;
        if (p == 1 && !last) { io.regions = regions; io.region_bits = pp.bits[0]; io.low_hist = low_base; }
        if (last) { io.low_base = low_base; io.low_bits = r.low_bits; }
      }
      io.idx_in = iin;
      io.keys_out = (last && !r.want_sorted_keys) ? nullptr : kout;
      int32_t* iout = last ? round_out : ((p & 1) ? b.idxB.as<int32_t>() : b.idxA.as<int32_t>());
      io.idx_out = iout;
      const bool carry = gp.region_sum && p == 0;
      if (carry) {
        io.vals = gp.region_value.data; io.vperm = b.vperm.p; io.vbytes = stype_bytes(gp.region_value.stype);
        if (!io.bases_out) io.bases_out = b.rbases.as<u32>();
        b.region_keys = kout;                          // no later pass of the round writes this buffer (<= 3 passes)
      }
      DTB_TRY(launch_radix_pass(io, rk, r.kin_bytes[p], n, pp.shift[p] - r.kdrop[p], pp.bits[p], work.as<u32>(), s,
                                (gp.count_table && last) ? b.gcount.as<u32>() : nullptr, rk.group_shift));
      if (carry && io.bases_out != b.rbases.p)
        DTB_CUDA_CHECK(cudaMemcpyAsync(b.rbases.p, io.bases_out, sizeof(u32) * 256, cudaMemcpyDeviceToDevice, s));
      if (last && r.want_sorted_keys) b.sorted_keys = kout;
      kin = kout;
      kout = (kout == b.keyA.p) ? b.keyB.p : b.keyA.p;
      iin = iout;
    }
    idx_cur = round_out;
  }
  return DTB_OK;
}

// The Groupby offsets (the call's second wait), and the group keys of the direct-address reducers.
static int group_offsets(const GroupPlan& gp, int64_t n, const int32_t* order, int32_t* offsets, GroupBufs& b,
                         GroupResult& res, cudaStream_t s)
{
  if (res.ngroups < 0) return DTB_OK;                  // sort only
  if (!gp.groups_k) {                                  // every by-column is constant: one group
    int32_t h[2] = {0, (int32_t)n};
    DTB_CUDA_CHECK(cudaMemcpyAsync(offsets, h, sizeof(h), cudaMemcpyHostToDevice, s));
    DTB_CUDA_CHECK(cudaStreamSynchronize(s));
    res.ngroups = 1;
    return DTB_OK;
  }
  const int nrounds = (int)gp.rounds.size();
  const int64_t otiles = offsets_num_tiles(n);
  DevBuf oscr; DTB_TRY(oscr.alloc(sizeof(u64) * (size_t)(otiles + 4), s));
  DTB_CUDA_CHECK(cudaMemsetAsync(oscr.p, 0, oscr.bytes, s));
  u64* d_ng = oscr.as<u64>() + otiles + 2;
  DevBuf headflags;
  if (gp.count_table) {
    ProfScope ps("group_offsets_from_counts", s);
    DevBuf gk; DTB_TRY(gk.alloc_owned(sizeof(u32) * (size_t)(gp.ctable + 1), s));   // trimmed by the handle's lifetime
    res.direct.gkeys = gk.detach();
    DevBuf cscr; DTB_TRY(cscr.alloc(sizeof(u64) * (size_t)(2 * gp.ctable / 1024 + 2), s));
    DTB_TRY(launch_offsets_from_counts(b.gcount.as<u32>(), gp.ctable, n, offsets, (u32*)res.direct.gkeys, d_ng,
                                       cscr.as<u64>(), s));
  } else if (nrounds == 1) {
    ProfScope ps("group_offsets", s);
    DTB_TRY(launch_group_offsets(b.sorted_keys, gp.rounds[0].key_bytes, gp.rounds[0].kp.group_shift, n, offsets, d_ng,
                                 oscr.as<u64>(), s));
  } else {
    // heads = rows where any by-column differs from the previous row: OR the per-round
    // comparisons; earlier rounds' keys are re-composed through the final RowIndex.
    DTB_TRY(headflags.alloc((size_t)n + 32, s));
    DTB_CUDA_CHECK(cudaMemsetAsync(headflags.p, 0, headflags.bytes, s));
    for (int ri = 0; ri < nrounds; ri++) {
      if (!gp.rounds[ri].has_by) continue;
      const KeyPlan& rk = gp.rounds[ri].kp;
      const void* ks = b.sorted_keys;
      if (ri != nrounds - 1 || !b.sorted_keys) {
        void* tmp = (b.sorted_keys == b.keyA.p) ? b.keyB.p : b.keyA.p;
        DTB_TRY(launch_compose_keys(rk, n, order, tmp, gp.rounds[ri].key_bytes, s));
        ks = tmp;
      }
      DTB_TRY(launch_mark_heads(ks, gp.rounds[ri].key_bytes, rk.group_shift, n, headflags.as<uint8_t>(), s));
    }
    DTB_TRY(launch_group_offsets(headflags.p, 1, 0, n, offsets, d_ng, oscr.as<u64>(), s));
  }
  u64 h_ng[2] = {0, 0};                    // {groups, rows of the largest group (count-table path only)}
  DTB_CUDA_CHECK(cudaMemcpyAsync(h_ng, d_ng, 2 * sizeof(u64), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(stream_wait(s));
  res.ngroups = (int64_t)h_ng[0];
  // group key of every group, for the direct-address reducers
  if (gp.count_table || gp.fused_direct) {
    if (!gp.count_table) {
      DevBuf gk; DTB_TRY(gk.alloc_owned(sizeof(u32) * (size_t)(res.ngroups + 1), s));
      res.direct.gkeys = gk.detach();
      DTB_TRY(launch_group_keys(b.sorted_keys, gp.rounds[0].key_bytes, offsets, gp.rounds[0].kp.group_shift, res.ngroups,
                                (u32*)res.direct.gkeys, s));
    }
    res.direct.on = true;
    res.direct.gmax = gp.count_table ? (int64_t)h_ng[1] : n;       // unknown: assume the worst
    res.direct.kp = gp.rounds[0].kp;
    res.direct.table = (int64_t)1 << gp.dbits;
  }
  return DTB_OK;
}

// The bucketed multi-reducer's sweeps (dtb_bucket.cu).  tables[c * BK_NWORDS + w]: word w of gp.bcols[c] (arena
// scratch: it lives until the call returns).
static int bucketed_reduce(const GroupPlan& gp, int64_t n, GroupBufs& b, std::vector<u64*>& tables, cudaStream_t s)
{
  const int ncols = (int)gp.bcols.size();
  tables.assign((size_t)ncols * BK_NWORDS, nullptr);
  for (int c = 0; c < ncols; c++)
    for (int w = 0; w < BK_NWORDS; w++) {
      if (!gp.bcols[c].want[w]) continue;
      DevBuf t; DTB_TRY(t.alloc(sizeof(u64) * (size_t)gp.ftable, s));
      tables[(size_t)c * BK_NWORDS + w] = t.as<u64>();
      fill_u64(t.as<u64>(), gp.ftable, w == BK_MIN ? ~0ull : 0ull, s);
    }
  const int nb = 1 << (gp.dbits > 11 ? gp.dbits - 11 : 0);
  // sweeps of up to BK_MAXCOLS columns / 32 value bytes per row (the partitioned copies live in scratch)
  std::vector<std::pair<int, int>> sweeps;           // [first, last) into bcols
  size_t scr = 0;
  for (int c = 0; c < ncols;) {
    int e = c, bytes = 0;
    while (e < ncols && e - c < BK_MAXCOLS && (e == c || bytes + stype_bytes(gp.bcols[e].stype) <= 32))
      bytes += stype_bytes(gp.bcols[e++].stype);
    const size_t need = bucket_scratch_bytes(n, bytes, e - c);
    scr = need > scr ? need : scr;
    sweeps.push_back({c, e});
    c = e;
  }
  DevBuf bstart, bscr;
  DTB_TRY(bstart.alloc(bucket_starts_bytes(n) + sizeof(u32) * (size_t)(nb + 8), s));
  DTB_TRY(bscr.alloc(scr, s));
  // the sweep reads bxk[i] >> bshift = the row's group key
  int bshift = gp.rounds[0].kp.group_shift;
  if (!b.bxk.p) {
    // a single raw key column, or several whose composite is wider than 32 bits (by() + sort()): the
    // group keys are composed once; a wider composite is stored as the group key itself
    const int cshift = gp.rounds[0].kp.total_bits > 32 ? bshift : 0;
    DTB_TRY(b.bxk.alloc(sizeof(u32) * (size_t)n, s));
    ProfScope ps("compose_keys", s); DTB_TRY(launch_compose_keys(gp.rounds[0].kp, n, nullptr, b.bxk.p, 4, s, cshift));
    bshift -= cshift;
  }
  u32* slab_starts = bstart.as<u32>(); u32* start = slab_starts + bucket_starts_bytes(n) / sizeof(u32);
  DTB_TRY(launch_bucket_starts(b.bxk.as<u32>(), bshift, n, nb, slab_starts, start, s));
  for (auto& sw : sweeps) {
    const void* vals[BK_MAXCOLS]; int sts[BK_MAXCOLS]; unsigned long long* words[BK_MAXCOLS][BK_NWORDS];
    const int nc = sw.second - sw.first;
    for (int c = 0; c < nc; c++) {
      const BucketCol& bc = gp.bcols[sw.first + c];
      vals[c] = bc.data; sts[c] = bc.stype;
      for (int w = 0; w < BK_NWORDS; w++) words[c][w] = tables[(size_t)(sw.first + c) * BK_NWORDS + w];
    }
    DTB_TRY(launch_bucketed_reduce(b.bxk.as<u32>(), bshift, gp.dbits, nc, vals, sts, n, slab_starts,
                                   start, words, bscr.p, s));
  }
  return DTB_OK;
}

// A reducer of the direct-address path (sum..countna over a device column): out[g] = finalize(acc0 / acc1 at the key
// of group g).  accumulate: every row first folds into the accumulators of its key, in plan_direct's streaming mode
// dp; otherwise the bucketed sweep has filled them.
// region (a sum over the column the first pass carried, GroupPlan::region_sum): the rows are added up per digit region
// of that pass.
static int direct_reduce(const DirectGroups& dg, const DirectPlan& dp, int op, dtb_col value, const int32_t* order,
                         const int32_t* offsets, int64_t n, int64_t ng, u64* acc0, u64* acc1, bool accumulate,
                         void* out, cudaStream_t s, const GroupPlan* region = nullptr, const GroupBufs* rb = nullptr)
{
  GroupRows rows;                                  // for the zero lookup: every row is in a group (no NA_REMOVE)
  rows.v = value.data; rows.nv = n; rows.order = order; rows.offsets = offsets; rows.n = n;
  DevBuf zscr;                                     // float min / max: the zero lookup's marks
  if (minmax_zero_sign(op, value.stype)) { DTB_TRY(zscr.alloc(zero_fix_bytes(ng), s)); rows.zpos = zscr.as<u64>(); }
  if (accumulate && ng > 0) {
    ProfScope ps("reduce_direct", s);
    DTB_TRY(launch_direct_init(op, dp, dg.table, acc0, acc1, s));
    if (region) {
      const bool hot = dp.kind == DIRECT_HOT;
      ProfScope pr(hot ? "region_sum_hot" : "region_sum", s);     // inside reduce_direct: tells the paths apart
      const RoundPlan& r = region->rounds[0];
      DTB_TRY(launch_region_sum(rb->region_keys, r.kout_bytes[0], r.pp.bits[0], region->dbits - r.pp.bits[0],
                                (const u32*)rb->rbases.p, rb->vperm.p, value.stype, n,
                                hot ? (const uint8_t*)dp.map : nullptr, acc0, s));
    } else {
      DTB_TRY(launch_direct_accumulate_rows(op, dg.kp, dp, value.data, value.stype, n, acc0, acc1, s));
    }
  }
  return launch_direct_finalize(op, value.stype, acc0, acc1, dp, (const uint32_t*)dg.gkeys, ng, out, rows, s);
}

// A reducer over the device column `value` seen through the RowIndex `order` (order_is64: int64 row ids); acc: 2 * ng
// u64 of scratch.
static int reduce_rowindex(int op, const void* value, int stype, int64_t nrows_value, const void* order, int order_is64,
                           const int32_t* offsets, int64_t ng, int64_t n, u64* acc, void* out, cudaStream_t s)
{
  DevBuf extra;
  const size_t xb = reduce_extra_bytes(op, stype, ng, n);
  if (xb) DTB_TRY(extra.alloc(xb, s));
  ProfScope ps("reduce", s);
  return launch_reduce_impl(op, value, stype, nrows_value, order, order_is64, offsets, ng, n, acc, acc + ng, out, s,
                            xb ? extra.p : nullptr);
}

// The fused reducers, once the groups are known.  When the group key domain is small they only need the key
// columns, not the RowIndex: they stream the rows in storage order (the streaming mode -- plain / shared-memory
// table / hot-key cache -- depends on the number of groups and the size of the largest one, see plan_direct).
// They run on `s` after the offsets: measured on C2, running them on a second stream under the sort passes gained
// ~2 % for the accumulation (both want the same SMs) and made every scatter launch ~40 % slower.  Otherwise every
// reducer reads its column through the RowIndex.
static int fused_reduce(const GroupPlan& gp, int64_t n, const int32_t* order, const int32_t* offsets, GroupBufs& b,
                        const GroupResult& res, FusedReducers& fr, cudaStream_t s)
{
  const int64_t ng = res.ngroups;
  fr.out.assign(fr.n, nullptr);
  DirectPlan dp = {DIRECT_PLAIN, nullptr, gp.ftable};
  DevBuf dmap;
  if (gp.fused_direct && ng > 0) {
    DTB_TRY(dmap.alloc(direct_map_bytes(gp.ftable), s));
    DTB_TRY(plan_direct(gp.ftable, (const uint32_t*)res.direct.gkeys, offsets, ng, n, res.direct.gmax, dmap.p, s, dp));
  }
  DevBuf gacc;
  if (!gp.fused_direct) DTB_TRY(gacc.alloc(sizeof(u64) * (size_t)(ng > 0 ? ng : 1) * 2, s));
  // spread-out keys only: few groups and hot keys have their own streaming modes (plan_direct)
  const bool bucketed = !gp.bcols.empty() && ng > 0 && dp.kind == DIRECT_PLAIN;
  std::vector<u64*> tables;
  if (bucketed) DTB_TRY(bucketed_reduce(gp, n, b, tables, s));
  for (int i = 0; i < fr.n; i++) {
    const dtb_reduce_spec& sp = fr.spec[i];
    int out_st = 0;
    DTB_TRY(reducer_out_stype(sp.op, sp.value.stype, out_st));
    DevBuf ob; DTB_TRY(ob.alloc_owned((size_t)(ng > 0 ? ng : 1) * stype_bytes(out_st), s));
    if (sp.op == DTB_OP_NROWS) {
      DTB_TRY(launch_nrows(offsets, ng, ob.p, s));
    } else if (bucketed && gp.bcol_of[i] >= 0) {
      u64* const* w = &tables[(size_t)gp.bcol_of[i] * BK_NWORDS];
      const BucketWords bw = bucket_words(sp.op, sp.value.stype);
      DTB_TRY(direct_reduce(res.direct, dp, sp.op, sp.value, order, offsets, n, ng, w[bw.a0],
                            bw.a1 >= 0 ? w[bw.a1] : nullptr, false, ob.p, s));
    } else if (gp.fused_direct) {
      u64* acc = b.facc.as<u64>() + (size_t)gp.ftable * 2 * i;
      const bool region = takes_region_sum(gp, sp) && dp.kind != DIRECT_SMALL;
      if (opt_verbose && takes_region_sum(gp, sp))
        fprintf(stderr, "[dtb200]   reducer %d: %s\n", i, region ? "region sum" : "direct (few groups)");
      DTB_TRY(direct_reduce(res.direct, dp, sp.op, sp.value, order, offsets, n, ng, acc, acc + gp.ftable, true, ob.p, s,
                            region ? &gp : nullptr, &b));
    } else {
      DevIn dv;
      if (sp.op != DTB_OP_NROWS) DTB_TRY(dv.bind(sp.value.data, (size_t)n * stype_bytes(sp.value.stype), s));
      DTB_TRY(reduce_rowindex(sp.op, dv.dptr, sp.value.stype, n, order, 0, offsets, ng, n, gacc.as<u64>(), ob.p, s));
    }
    fr.out[i] = ob.detach();
  }
  return DTB_OK;
}

// wide == dtb_group64: up to 2^32 - 1 rows.  The passes carry row ids and output slots as 32-bit words
// whose arithmetic is unsigned throughout, so ids >= 2^31 are just bit patterns in the int32 buffers;
// the caller zero-extends order / offsets to int64 (ARR64, rowindex_array.cc:50-60).
static int validate_group(const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t n, bool handle,
                          bool wide)
{
  if (nkeys < 1 || nkeys > MAX_KEYS) { set_error("number of key columns must be in 1.." + std::to_string(MAX_KEYS)); return DTB_EINVAL; }
  if (!keys || !flags) { set_error("keys/flags must not be NULL"); return DTB_EINVAL; }
  if (na_pos < DTB_NA_FIRST || na_pos > DTB_NA_REMOVE) { set_error("na position value is not supported"); return DTB_EINVAL; }
  if (na_pos == DTB_NA_REMOVE && !(flags[0] & DTB_FLAG_SORT_ONLY)) {
    // the RowIndex drops the first nacount(last key) rows while the groups would still count them
    set_error("na_position = remove is only supported without groups (the first key column must be SORT_ONLY)");
    return DTB_EINVAL;
  }
  if (n < 0) { set_error("nrows must be non-negative"); return DTB_EINVAL; }
  for (int c = 0; c < nkeys; c++) {
    if (!stype_supported(keys[c].stype)) {
      set_error("Unable to sort Column of stype " + std::to_string(keys[c].stype));   // sort.cc:673
      return DTB_ENOTIMPL;
    }
    if (n > 0 && !keys[c].data) { set_error("key column data is NULL"); return DTB_EINVAL; }
  }
  if (n > (int64_t)INT32_MAX && !wide) { set_error("nrows > INT32_MAX needs an ARR64 RowIndex: use dtb_group64"); return DTB_ENOTIMPL; }
  if (n > (int64_t)0xFFFFFFFFll - 65536) { set_error("nrows >= 2^32 is beyond one GPU's passes (32-bit output slots): partition the frame"); return DTB_ENOTIMPL; }
  if (wide && handle) { set_error("internal: the ARR64 path has no fused reducers"); return DTB_EINVAL; }
  return DTB_OK;
}

static int group_core(const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t n,
                      cudaStream_t s, int32_t* order_dev /*optional caller buffer*/,
                      int32_t* offsets_dev /*optional caller buffer, n+1*/, GroupResult& res,
                      bool want_direct = false, FusedReducers* fr = nullptr, bool wide = false)
{
  // want_direct == the handle path: the RowIndex outlives the call and must be an owned allocation
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  t_tl0 = now_ms();
  DTB_TRY(validate_group(keys, nkeys, flags, na_pos, n, want_direct || fr, wide));
  DTB_TRY(ensure_context());
  const bool do_groups = !(flags[0] & DTB_FLAG_SORT_ONLY);
  res.n = n; res.nskip = 0; res.ngroups = do_groups ? 0 : -1; res.s = s;
  int32_t* order = order_dev;
  if (!order) {
    if (want_direct) DTB_TRY(res.order.alloc_owned(sizeof(int32_t) * (size_t)n, s));
    else             DTB_TRY(res.order.alloc(sizeof(int32_t) * (size_t)n, s));
    order = res.order.as<int32_t>();
  }
  int32_t* offsets = offsets_dev;
  if (do_groups && !offsets) {
    DTB_TRY(res.offsets.alloc(sizeof(int32_t) * (size_t)(n + 1), s)); offsets = res.offsets.as<int32_t>();
  }
  if (n == 0) {                                           // sort.cc:1431-1434
    if (do_groups) DTB_CUDA_CHECK(cudaMemsetAsync(offsets, 0, sizeof(int32_t), s));
    return DTB_OK;
  }

  GroupBufs b;
  DTB_TRY(stage_inputs(keys, nkeys, n, fr, s, b));
  DTB_TL("stats synced");
  GroupPlan gp;
  plan_group(keys, nkeys, flags, na_pos, n, b, want_direct, fr, gp);
  res.nskip = gp.nskip;
  t_stats.key_bits = gp.kp.total_bits;
  if (gp.kp.total_bits == 0) {          // every key column is constant: identity order, one group (cf. sort.cc:1435-1439)
    DTB_TRY(launch_iota32(order, n, s));
    DTB_TRY(group_offsets(gp, n, order, offsets, b, res, s));
  } else {
    print_plan(gp, n, nkeys, b.st);
    DTB_TRY(sort_rounds(gp, n, fr ? fr->n : 0, order, s, b));
    DTB_TL("passes enqueued");
    DTB_TRY(group_offsets(gp, n, order, offsets, b, res, s));
    DTB_TL("offsets synced");
  }
  if (fr && fr->n > 0 && do_groups) DTB_TRY(fused_reduce(gp, n, order, offsets, b, res, *fr, s));
  return DTB_OK;
}

}  // namespace dtb

using namespace dtb;

// ===========================================================================
// extern "C"
// ===========================================================================
struct dtb_groupby {
  void* order = nullptr;      // device int32[norder] (view into order_base)
  void* order_base = nullptr;
  void* offsets = nullptr;    // device int32[ngroups+1]
  int64_t norder = 0;
  int64_t ngroups = -1;
  int64_t nrows = 0;
  dtb::DirectGroups direct;   // the direct-address reducers' groups
  std::vector<void*> reduced; // outputs of the reducers evaluated by dtb_groupby_create_reduce
};

// A reducer fed piecewise (dtb_groupby_reduce_begin / _add / _end): the accumulator tables live across calls.
struct dtb_reduce_state {
  dtb_groupby* g = nullptr;
  int op = 0, stype = 0, out_stype = 0;
  void* acc = nullptr;        // device u64[2 * table]
  void* dmap = nullptr;       // plan_direct's map (shared-memory table / hot-key modes)
  dtb::DirectPlan dp;
  int64_t rows_added = 0;
  // float min / max: inverse RowIndex (int32[nrows]) and every group's first valid zero (u64[ngroups], GroupRows)
  void* inv = nullptr;
  void* first_zero = nullptr;
};

extern "C" {

const char* dtb_last_error(void) { return t_error.c_str(); }
int dtb_abi_version(void) { return DTB_ABI_VERSION; }
int dtb_stype_size(int stype) { return stype_bytes(stype); }
int dtb_reduce_out_stype(int op, int stype) { return reduce_out_stype_host(op, stype); }

int dtb_init(int device) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    set_error(std::string("cudaSetDevice: ") + cudaGetErrorString(e));
    return DTB_ECUDA;
  }
  return ensure_context();
}

int dtb_memcpy(void* dst, const void* src, int64_t nbytes, dtb_stream stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (nbytes < 0 || (nbytes > 0 && (!dst || !src))) { set_error("bad dtb_memcpy arguments"); return DTB_EINVAL; }
  if (nbytes == 0) return DTB_OK;
  DTB_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)nbytes, cudaMemcpyDefault, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  return DTB_OK;
}

int dtb_set_option(const char* name, int64_t value) {
  if (!name) { set_error("option name is NULL"); return DTB_EINVAL; }
  if (!strcmp(name, "radix_bits")) {
    if (value != 0 && (value < 4 || value > 8)) { set_error("radix_bits must be 0 (default) or 4..8"); return DTB_EINVAL; }
    opt_radix_bits = value; return DTB_OK;
  }
  if (!strcmp(name, "verbose")) { opt_verbose = value; return DTB_OK; }
  if (!strcmp(name, "profile")) { opt_profile = value; return DTB_OK; }
  if (!strcmp(name, "bucketed_reducers")) { opt_bucketed = value ? 1 : 0; return DTB_OK; }
  if (!strcmp(name, "trim_scratch")) {
    if (t_arena.depth == 0 && t_arena.device >= 0) {
      int cur = 0; cudaGetDevice(&cur);
      if (cur != t_arena.device) cudaSetDevice(t_arena.device);
      t_arena.trim();
      if (cur != t_arena.device) cudaSetDevice(cur);
    }
    // handles' RowIndex / offsets / results come from the device's stream-ordered pool, which keeps what they
    // freed (release threshold = max): give that back too, so that one large call can use the whole HBM
    int dev = 0;
    cudaMemPool_t pool;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      DTB_CUDA_CHECK(cudaDeviceSynchronize());
      DTB_CUDA_CHECK(cudaMemPoolTrimTo(pool, 0));
    }
    return DTB_OK;
  }
  set_error(std::string("unknown option ") + name);
  return DTB_EINVAL;
}

int dtb_profile_count(void) { prof_collect(); return (int)t_prof_done.size(); }

int dtb_profile_get(int i, char* name, int cap, double* ms) {
  if (i < 0 || i >= (int)t_prof_done.size() || !name || cap < 1 || !ms) { set_error("bad dtb_profile_get arguments"); return DTB_EINVAL; }
  strncpy(name, t_prof_done[i].first.c_str(), (size_t)cap - 1);
  name[cap - 1] = 0;
  *ms = t_prof_done[i].second;
  return DTB_OK;
}

int dtb_profile_reset(void) { prof_collect(); t_prof_done.clear(); return DTB_OK; }

int dtb_get_option(const char* name, int64_t* value) {
  if (!name || !value) { set_error("NULL argument"); return DTB_EINVAL; }
  if (!strcmp(name, "radix_bits")) { *value = opt_radix_bits; return DTB_OK; }
  if (!strcmp(name, "verbose")) { *value = opt_verbose; return DTB_OK; }
  if (!strcmp(name, "profile")) { *value = opt_profile; return DTB_OK; }
  if (!strcmp(name, "bucketed_reducers")) { *value = opt_bucketed; return DTB_OK; }
  set_error(std::string("unknown option ") + name);
  return DTB_EINVAL;
}

int dtb_last_call_stats(dtb_call_stats* out) {
  if (!out) { set_error("NULL argument"); return DTB_EINVAL; }
  *out = t_stats;
  return DTB_OK;
}

// Copies `count` 32-bit row ids or offsets of group() to the caller's buffer: as they are for ARR32, zero-extended
// to int64 for ARR64 (rowindex_array.cc:50-60).
static int copy_out(bool wide, void* dst, const void* src, int64_t count, cudaStream_t s) {
  if (!wide) {
    DTB_CUDA_CHECK(cudaMemcpyAsync(dst, src, sizeof(int32_t) * (size_t)count, cudaMemcpyDefault, s));
    if (!is_device_ptr(dst)) DevOut::remember(dst, src, sizeof(int32_t) * (size_t)count, s);
    return DTB_OK;
  }
  DevOut d; DTB_TRY(d.bind(dst, sizeof(int64_t) * (size_t)count, s));
  DTB_TRY(launch_widen_u32((const uint32_t*)src, count, (int64_t*)d.dptr, s));
  if (d.staged()) DTB_TRY(d.finish(sizeof(int64_t) * (size_t)count, s));
  return DTB_OK;
}

// dtb_group (wide = false) and dtb_group64 (wide = true)
static int group_out(bool wide, const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t nrows,
                     dtb_stream stream, void* order_out, void* offsets_out, int64_t offsets_cap,
                     int64_t* ngroups_out, int64_t* norder_out)
{
  cudaStream_t s = (cudaStream_t)stream;
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  if (!order_out && nrows > 0) { set_error("order_out is NULL"); return DTB_EINVAL; }
  if (nkeys >= 1 && flags && !(flags[0] & DTB_FLAG_SORT_ONLY) && !offsets_out) {
    set_error("offsets_out is NULL but groups were requested"); return DTB_EINVAL;
  }
  GroupResult res;
  // ARR32: compute straight into the caller's device buffers when they are large enough
  int32_t* order_dev = (!wide && nrows > 0 && is_device_ptr(order_out) && na_pos != DTB_NA_REMOVE) ? (int32_t*)order_out : nullptr;
  int32_t* offsets_dev = (!wide && offsets_out && is_device_ptr(offsets_out) && offsets_cap >= nrows + 1) ? (int32_t*)offsets_out : nullptr;
  DTB_TRY(group_core(keys, nkeys, flags, na_pos, nrows, s, order_dev, offsets_dev, res, false, nullptr, wide));
  const int64_t norder = res.n - res.nskip;
  if (norder_out) *norder_out = norder;
  if (ngroups_out) *ngroups_out = res.ngroups;
  if (!order_dev && norder > 0) DTB_TRY(copy_out(wide, order_out, res.order.as<int32_t>() + res.nskip, norder, s));
  if (res.ngroups >= 0 && !offsets_dev) {
    if (offsets_cap < res.ngroups + 1) {
      cudaStreamSynchronize(s);
      set_error("offsets_out holds " + std::to_string(offsets_cap) + " entries, need " + std::to_string(res.ngroups + 1));
      return DTB_ENOSPACE;
    }
    DTB_TRY(copy_out(wide, offsets_out, res.offsets.p, res.ngroups + 1, s));
  }
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  return DTB_OK;
}

int dtb_group(const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t nrows,
              dtb_stream stream, void* order_out, void* offsets_out, int64_t offsets_cap,
              int64_t* ngroups_out, int64_t* norder_out)
{
  return group_out(false, keys, nkeys, flags, na_pos, nrows, stream, order_out, offsets_out, offsets_cap, ngroups_out,
                   norder_out);
}

int dtb_group64(const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t nrows, dtb_stream stream,
                void* order_out, void* offsets_out, int64_t offsets_cap, int64_t* ngroups_out, int64_t* norder_out)
{
  return group_out(true, keys, nkeys, flags, na_pos, nrows, stream, order_out, offsets_out, offsets_cap, ngroups_out,
                   norder_out);
}

int dtb_groupby_create(const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t nrows,
                       dtb_stream stream, dtb_groupby** out)
{
  return dtb_groupby_create_reduce(keys, nkeys, flags, na_pos, nrows, stream, nullptr, 0, out);
}

int dtb_groupby_create_reduce(const dtb_col* keys, int nkeys, const int* flags, int na_pos, int64_t nrows,
                              dtb_stream stream, const dtb_reduce_spec* reducers, int nreducers,
                              dtb_groupby** out)
{
  cudaStream_t s = (cudaStream_t)stream;
  if (!out) { set_error("out is NULL"); return DTB_EINVAL; }
  *out = nullptr;
  if (nreducers < 0 || (nreducers > 0 && !reducers)) { set_error("bad reducer list"); return DTB_EINVAL; }
  if (nreducers > 0 && flags && nkeys > 0 && (flags[0] & DTB_FLAG_SORT_ONLY)) {
    set_error("reducers need a Groupby: the first key column must not be SORT_ONLY"); return DTB_EINVAL;
  }
  for (int i = 0; i < nreducers; i++) {
    if (reducers[i].op == DTB_OP_COV || reducers[i].op == DTB_OP_CORR) {
      set_error("cov / corr take two columns: use dtb_groupby_reduce2 on the handle"); return DTB_EINVAL;
    }
    if (reducers[i].op == DTB_OP_MEDIAN || reducers[i].op == DTB_OP_NUNIQUE) {
      set_error("median/nunique read rows sorted inside their group: use dtb_sort_grouped + dtb_reduce"); return DTB_EINVAL;
    }
  }
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  GroupResult res;
  FusedReducers fr; fr.spec = reducers; fr.n = nreducers;
  int rc = group_core(keys, nkeys, flags, na_pos, nrows, s, nullptr, nullptr, res, true, nreducers ? &fr : nullptr);
  if (rc != DTB_OK) { for (void* p : fr.out) if (p) cudaFreeAsync(p, s); return rc; }
  dtb_groupby* g = new dtb_groupby();
  g->reduced = fr.out;
  g->norder = res.n - res.nskip;
  g->ngroups = res.ngroups;
  g->nrows = res.n;
  g->direct = res.direct;
  res.direct.gkeys = nullptr;
  if (res.ngroups >= 0) {
    // shrink the worst-case offsets buffer to ngroups+1 entries
    DevBuf exact;
    // on failure the handle already owns the detached group keys and the fused reducer outputs:
    // dtb_groupby_destroy releases them (res.order is still owned by `res`)
    rc = exact.alloc_owned(sizeof(int32_t) * (size_t)(res.ngroups + 1), s);
    if (rc != DTB_OK) { dtb_groupby_destroy(g, stream); return rc; }
    cudaError_t e = cudaMemcpyAsync(exact.p, res.offsets.p, sizeof(int32_t) * (size_t)(res.ngroups + 1),
                                    cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); dtb_groupby_destroy(g, stream); return DTB_ECUDA; }
    g->offsets = exact.detach();
  }
  g->order_base = res.order.detach();
  g->order = (int32_t*)g->order_base + res.nskip;
  *out = g;
  return DTB_OK;
}

int64_t dtb_groupby_norder(const dtb_groupby* g) { return g ? g->norder : 0; }
int64_t dtb_groupby_ngroups(const dtb_groupby* g) { return g ? g->ngroups : -1; }
const void* dtb_groupby_order(const dtb_groupby* g) { return g ? g->order : nullptr; }
const void* dtb_groupby_offsets(const dtb_groupby* g) { return g ? g->offsets : nullptr; }
const void* dtb_groupby_reduced(const dtb_groupby* g, int i) {
  return (g && i >= 0 && i < (int)g->reduced.size()) ? g->reduced[i] : nullptr;
}

int dtb_groupby_destroy(dtb_groupby* g, dtb_stream stream) {
  if (!g) return DTB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (g->order_base) cudaFreeAsync(g->order_base, s);
  if (g->offsets) cudaFreeAsync(g->offsets, s);
  if (g->direct.gkeys) cudaFreeAsync(g->direct.gkeys, s);
  for (void* p : g->reduced) if (p) cudaFreeAsync(p, s);
  delete g;
  return DTB_OK;
}

// Binds the caller's Groupby offsets (host or device) and reads n = offsets[ngroups].  check_offsets = false: they come
// from group() (a handle's own), so they need no device check.
static int bind_groupby(const void* offsets, int64_t ngroups, bool check_offsets, cudaStream_t s, DevIn& d_off,
                        int64_t& n)
{
  DTB_TRY(d_off.bind(offsets, sizeof(int32_t) * (size_t)(ngroups + 1), s));
  // caller-supplied offsets must be a Groupby: offsets[0] = 0, strictly increasing (groupby.h:41-47), or the one
  // empty group [0, 0] of zero rows (Groupby::single_group(0), groupby.cc:60-68)
  int32_t n32 = 0;
  int bad = 0;
  if (is_device_ptr(offsets)) {
    DevBuf d_bad; DTB_TRY(d_bad.alloc(sizeof(int), s));
    DTB_CUDA_CHECK(cudaMemsetAsync(d_bad.p, 0, sizeof(int), s));
    if (check_offsets) DTB_TRY(launch_offsets_check((const int32_t*)offsets, ngroups, d_bad.as<int>(), s));
    DTB_CUDA_CHECK(cudaMemcpyAsync(&n32, (const int32_t*)offsets + ngroups, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    DTB_CUDA_CHECK(cudaMemcpyAsync(&bad, d_bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  } else {
    const int32_t* ho = (const int32_t*)offsets;
    n32 = ho[ngroups];
    if (ho[0] != 0) bad = 1;
    const bool single_empty = ngroups == 1 && n32 == 0;
    for (int64_t g = 0; g < ngroups && !bad; g++)
      if (ho[g] >= ho[g + 1] && !single_empty) bad = (int)(g < INT32_MAX ? g + 1 : INT32_MAX);
  }
  if (bad) {
    set_error("offsets is not a Groupby: offsets[0] must be 0 and offsets strictly increasing (group " +
              std::to_string(bad - 1) + " is empty or out of order)");
    return DTB_EINVAL;
  }
  n = n32;
  return DTB_OK;
}

// The arguments every per-group entry point shares (include/dtb200.h, "Per-group functions"): value columns of
// nrows_value rows seen through the RowIndex `order` (NULL = identity), cut by the Groupby `offsets`, and one output.
// An entry point constructs it first (which resets the call statistics), then checks its own argument and the stype;
// enter() runs the shared checks on the host, then makes the context and opens the arena; bind() reads n and binds the
// buffers; finish() copies a staged output back.
struct Grouped {
  cudaStream_t s;
  dtb_col value[2] = {};
  int nvalues;                  // value columns: 0 (dtb_group_index, DTB_OP_NROWS), 1, or 2 (dtb_reduce2)
  int64_t nrows_value;
  const void* order;
  int order_is64;
  const void* offsets;
  int64_t ngroups;
  void* out;
  bool handle = false;          // a handle's own offsets: group() made them, so they need no device check
  bool within_column = false;   // without an order, positions beyond the value column are an error (the row
                                // functions); otherwise they read as NA (the reducers, dtb_sort_grouped)
  bool per_position = false;    // out holds one element per position, else one per group
  std::optional<ArenaScope> scope;
  DevIn off, ord, val[2];
  DevOut dout;
  int64_t n = 0;                // positions: offsets[ngroups]

  Grouped(dtb_stream stream, std::initializer_list<dtb_col> values, int64_t nrows_value_, const void* order_,
          int order_is64_, const void* offsets_, int64_t ngroups_, void* out_)
    : s((cudaStream_t)stream), nvalues((int)values.size()), nrows_value(nrows_value_), order(order_),
      order_is64(order_is64_), offsets(offsets_), ngroups(ngroups_), out(out_)
  {
    int i = 0;
    for (const dtb_col& v : values) value[i++] = v;
    t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  }

  // ngroups == 0 leaves nothing to do: the caller returns.
  int enter() {
    if (ngroups < 0) { set_error("ngroups must be non-negative"); return DTB_EINVAL; }
    if (!offsets) { set_error("offsets is NULL"); return DTB_EINVAL; }
    if (nrows_value < 0) { set_error("nrows_value must be non-negative"); return DTB_EINVAL; }
    for (int i = 0; i < nvalues; i++)
      if (!value[i].data && nrows_value > 0) { set_error("value column data is NULL"); return DTB_EINVAL; }
    // one output per position: the one empty group [0, 0] has none, so out may be NULL there (a 0-element tensor's
    // data pointer); device offsets are read in bind()
    if (!out && ngroups > 0 &&
        !(per_position && ngroups == 1 && (is_device_ptr(offsets) || ((const int32_t*)offsets)[1] == 0))) {
      set_error("out is NULL"); return DTB_EINVAL;
    }
    DTB_TRY(ensure_context());
    if (ngroups == 0) return DTB_OK;
    scope.emplace(s);
    return scope->rc;
  }

  // out_esz: bytes per output element.
  int bind(int out_esz) {
    DTB_TRY(bind_groupby(offsets, ngroups, !handle, s, off, n));
    if (!out && n > 0) { set_error("out is NULL"); return DTB_EINVAL; }
    if (within_column && !order && n > nrows_value) {
      set_error("offsets cover more rows than the value column has"); return DTB_EINVAL;
    }
    for (int i = 0; i < nvalues; i++)
      DTB_TRY(val[i].bind(value[i].data, (size_t)nrows_value * stype_bytes(value[i].stype), s));
    DTB_TRY(ord.bind(order, (size_t)n * (order_is64 ? 8 : 4), s));
    return dout.bind(out, (size_t)(per_position ? n : ngroups) * out_esz, s);
  }

  // Afterwards n == 0 (no group, or the one empty group [0, 0]) leaves a per-position function nothing to write: it
  // returns without a launch.  A reducer still writes the empty group's one result.
  int open(int out_esz) {
    DTB_TRY(enter());
    return ngroups ? bind(out_esz) : DTB_OK;
  }

  // Waits for the stream when the output was staged, or always when sync.
  int finish(bool sync = false) {
    if (dout.staged()) DTB_TRY(dout.finish(dout.bytes, s));
    if (sync || dout.staged()) DTB_CUDA_CHECK(cudaStreamSynchronize(s));
    return DTB_OK;
  }

  const int32_t* offs() const { return (const int32_t*)off.dptr; }
};

// The stype check of the functions that take every fixed-width stype.
static int fixed_width(int stype, const char* fname) {
  if (stype_supported(stype)) return DTB_OK;
  set_error(std::string(fname) + " cannot be applied to columns of stype " + std::to_string(stype));
  return DTB_ENOTIMPL;
}

// dtb_reduce, and dtb_groupby_reduce with its handle g: where the handle's key domain is small, sum..countna over a
// device column stream the key and value columns in storage order instead of reading through the RowIndex.
static int reduce_groups(int op, Grouped& c, const dtb_groupby* g)
{
  const dtb_col value = c.value[0];
  if (op < DTB_OP_SUM || op > DTB_OP_CORR) { set_error("unknown reducer " + std::to_string(op)); return DTB_EINVAL; }
  int out_st = 0;
  DTB_TRY(reducer_out_stype(op, value.stype, out_st));
  if (op == DTB_OP_NROWS) { c.nvalues = 0; c.order = nullptr; }   // reads neither the column nor the RowIndex
  DTB_TRY(c.enter());
  if (c.ngroups == 0) return DTB_OK;
  if (g && g->direct.on && op < DTB_OP_NROWS && c.nrows_value == g->nrows && is_device_ptr(value.data)) {
    const DirectGroups& dg = g->direct;
    DTB_TRY(c.dout.bind(c.out, (size_t)c.ngroups * stype_bytes(out_st), c.s));
    DevBuf acc; DTB_TRY(acc.alloc(sizeof(u64) * (size_t)dg.table * 2, c.s));
    DevBuf dmap; DTB_TRY(dmap.alloc(direct_map_bytes(dg.table), c.s));
    DirectPlan dp;
    DTB_TRY(plan_direct(dg.table, (const uint32_t*)dg.gkeys, (const int32_t*)g->offsets, g->ngroups, g->nrows,
                        dg.gmax, dmap.p, c.s, dp));
    DTB_TRY(direct_reduce(dg, dp, op, value, (const int32_t*)g->order, (const int32_t*)g->offsets, g->nrows, g->ngroups,
                          acc.as<u64>(), acc.as<u64>() + dg.table, true, c.dout.dptr, c.s));
  } else {
    DTB_TRY(c.bind(stype_bytes(out_st)));
    DevBuf acc; DTB_TRY(acc.alloc(sizeof(u64) * (size_t)c.ngroups * 2, c.s));
    DTB_TRY(reduce_rowindex(op, c.val[0].dptr, value.stype, c.nrows_value, c.ord.dptr, c.order_is64, c.offs(),
                            c.ngroups, c.n, acc.as<u64>(), c.dout.dptr, c.s));
  }
  return c.finish();
}

int dtb_reduce(int op, dtb_col value, int64_t nrows_value, const void* order, int order_is64,
               const void* offsets, int64_t ngroups, dtb_stream stream, void* out)
{
  Grouped c(stream, {value}, nrows_value, order, order_is64, offsets, ngroups, out);
  return reduce_groups(op, c, nullptr);
}

int dtb_groupby_reduce(dtb_groupby* g, int op, dtb_col value, int64_t nrows_value, dtb_stream stream, void* out)
{
  if (!g) { set_error("groupby handle is NULL"); return DTB_EINVAL; }
  if (g->ngroups < 0) { set_error("the handle holds no Groupby (sort-only call)"); return DTB_EINVAL; }
  Grouped c(stream, {value}, nrows_value, g->order, 0, g->offsets, g->ngroups, out);
  c.handle = true;
  return reduce_groups(op, c, g);
}

int dtb_reduce2_out_stype(int op, int stype_x, int stype_y) { return reduce2_out_stype_host(op, stype_x, stype_y); }

// dtb_reduce2 and dtb_groupby_reduce2: c holds the columns x and y.
static int reduce2_groups(int op, Grouped& c)
{
  const dtb_col x = c.value[0], y = c.value[1];
  if (op != DTB_OP_COV && op != DTB_OP_CORR) { set_error("dtb_reduce2 takes DTB_OP_COV or DTB_OP_CORR"); return DTB_EINVAL; }
  const int out_st = reduce2_out_stype_host(op, x.stype, y.stype);
  if (!out_st) {
    set_error("Invalid columns of stypes " + std::to_string(x.stype) + ", " + std::to_string(y.stype) + " in reducer " +
              std::to_string(op));
    return (stype_supported(x.stype) && stype_supported(y.stype)) ? DTB_EINVAL : DTB_ENOTIMPL;
  }
  DTB_TRY(c.open(stype_bytes(out_st)));
  if (c.ngroups == 0) return DTB_OK;
  DevBuf scr; DTB_TRY(scr.alloc(reduce2_scratch_bytes(c.ngroups), c.s));
  {
    ProfScope ps("reduce2", c.s);
    DTB_TRY(launch_reduce2(op, c.val[0].dptr, x.stype, c.val[1].dptr, y.stype, c.nrows_value, c.ord.dptr, c.order_is64,
                           c.offs(), c.ngroups, c.n, scr.as<u64>(), out_st == DTB_STYPE_FLOAT32, c.dout.dptr, c.s));
  }
  return c.finish();
}

int dtb_reduce2(int op, dtb_col x, dtb_col y, int64_t nrows_value, const void* order, int order_is64,
                const void* offsets, int64_t ngroups, dtb_stream stream, void* out)
{
  Grouped c(stream, {x, y}, nrows_value, order, order_is64, offsets, ngroups, out);
  return reduce2_groups(op, c);
}

int dtb_groupby_reduce2(dtb_groupby* g, int op, dtb_col x, dtb_col y, int64_t nrows_value, dtb_stream stream, void* out)
{
  if (!g) { set_error("groupby handle is NULL"); return DTB_EINVAL; }
  if (g->ngroups < 0) { set_error("the handle holds no Groupby (sort-only call)"); return DTB_EINVAL; }
  Grouped c(stream, {x, y}, nrows_value, g->order, 0, g->offsets, g->ngroups, out);
  c.handle = true;
  return reduce2_groups(op, c);
}

int dtb_cumulative_out_stype(int op, int stype) { return cumulative_out_stype(op, stype); }

int dtb_cumulative(int op, int reverse, dtb_col value, int64_t nrows_value, const void* order, int order_is64,
                   const void* offsets, int64_t ngroups, dtb_stream stream, void* out)
{
  Grouped c(stream, {value}, nrows_value, order, order_is64, offsets, ngroups, out);
  if (op != DTB_OP_SUM && op != DTB_OP_PROD && op != DTB_OP_MIN && op != DTB_OP_MAX) {
    set_error("dtb_cumulative takes DTB_OP_SUM, DTB_OP_PROD, DTB_OP_MIN or DTB_OP_MAX"); return DTB_EINVAL;
  }
  DTB_TRY(fixed_width(value.stype, "cumulative functions"));
  const int out_st = cumulative_out_stype(op, value.stype);
  if (!out_st) {
    set_error("Invalid column of stype " + std::to_string(value.stype) + " in cumulative function " + std::to_string(op));
    return DTB_EINVAL;
  }
  c.within_column = c.per_position = true;
  DTB_TRY(c.open(stype_bytes(out_st)));
  if (c.n == 0) return DTB_OK;
  DevBuf scr; DTB_TRY(scr.alloc(cumulative_scratch_bytes(c.n), c.s));
  {
    ProfScope ps("cumulative", c.s);
    DTB_TRY(launch_cumulative(op, reverse, c.val[0].dptr, value.stype, nrows_value, c.ord.dptr, order_is64, c.offs(),
                              ngroups, c.n, scr.p, c.dout.dptr, c.s));
  }
  return c.finish();
}

int dtb_shift(dtb_col value, int64_t nrows_value, const void* order, int order_is64, const void* offsets,
              int64_t ngroups, int64_t n, dtb_stream stream, void* out)
{
  Grouped c(stream, {value}, nrows_value, order, order_is64, offsets, ngroups, out);
  DTB_TRY(fixed_width(value.stype, "shift"));
  c.within_column = c.per_position = true;
  DTB_TRY(c.open(stype_bytes(value.stype)));
  if (c.n == 0) return DTB_OK;
  {
    ProfScope ps("shift", c.s);
    DTB_TRY(launch_shift(c.val[0].dptr, value.stype, nrows_value, c.ord.dptr, order_is64, c.offs(), ngroups, c.n, n,
                         c.dout.dptr, c.s));
  }
  return c.finish();
}

int dtb_fillna(int reverse, dtb_col value, int64_t nrows_value, const void* order, int order_is64,
               const void* offsets, int64_t ngroups, dtb_stream stream, void* out)
{
  Grouped c(stream, {value}, nrows_value, order, order_is64, offsets, ngroups, out);
  DTB_TRY(fixed_width(value.stype, "fillna"));
  c.within_column = c.per_position = true;
  DTB_TRY(c.open(stype_bytes(value.stype)));
  if (c.n == 0) return DTB_OK;
  DevBuf scr; DTB_TRY(scr.alloc(cumulative_scratch_bytes(c.n), c.s));
  {
    ProfScope ps("fillna", c.s);
    DTB_TRY(launch_fillna(reverse, c.val[0].dptr, value.stype, nrows_value, c.ord.dptr, order_is64, c.offs(), ngroups,
                          c.n, scr.p, c.dout.dptr, c.s));
  }
  return c.finish();
}

int dtb_group_index(int kind, int reverse, const void* offsets, int64_t ngroups, dtb_stream stream, void* out)
{
  Grouped c(stream, {}, 0, nullptr, 0, offsets, ngroups, out);
  if (kind != DTB_GROUP_CUMCOUNT && kind != DTB_GROUP_NGROUP) {
    set_error("dtb_group_index takes DTB_GROUP_CUMCOUNT or DTB_GROUP_NGROUP"); return DTB_EINVAL;
  }
  c.per_position = true;
  DTB_TRY(c.open(sizeof(int64_t)));
  if (c.n == 0) return DTB_OK;
  {
    ProfScope ps("group_index", c.s);
    DTB_TRY(launch_group_index(kind, reverse, c.offs(), ngroups, c.n, (int64_t*)c.dout.dptr, c.s));
  }
  return c.finish();
}

int dtb_groupby_reduce_begin(dtb_groupby* g, int op, int value_stype, dtb_stream stream, dtb_reduce_state** out)
{
  cudaStream_t s = (cudaStream_t)stream;
  if (!g || !out) { set_error("groupby handle / out is NULL"); return DTB_EINVAL; }
  *out = nullptr;
  if (g->ngroups < 0) { set_error("the handle holds no Groupby (sort-only call)"); return DTB_EINVAL; }
  if (op == DTB_OP_COV || op == DTB_OP_CORR) { set_error("cov / corr take two columns"); return DTB_EINVAL; }
  if (!g->direct.on || op < DTB_OP_SUM || op >= DTB_OP_NROWS) {
    set_error("piecewise reducers exist for the streaming path only (small key domain, device key columns, sum..countna)");
    return DTB_ENOTIMPL;
  }
  int out_st = 0;
  DTB_TRY(reducer_out_stype(op, value_stype, out_st));
  DTB_TRY(ensure_context());
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  const DirectGroups& dg = g->direct;
  dtb_reduce_state* st = new dtb_reduce_state();
  st->g = g; st->op = op; st->stype = value_stype; st->out_stype = out_st;
  const size_t acc_bytes = sizeof(u64) * (size_t)dg.table * 2, map_bytes = direct_map_bytes(dg.table);
  if (cudaMalloc(&st->acc, acc_bytes ? acc_bytes : 8) != cudaSuccess || cudaMalloc(&st->dmap, map_bytes ? map_bytes : 8) != cudaSuccess) {
    cudaGetLastError(); cudaFree(st->acc); delete st; set_error("out of device memory"); return DTB_ENOMEM;
  }
  int rc = DTB_OK;
  if (g->ngroups > 0) {
    rc = plan_direct(dg.table, (const uint32_t*)dg.gkeys, (const int32_t*)g->offsets, g->ngroups, g->nrows, dg.gmax, st->dmap, s, st->dp);
    if (rc == DTB_OK) rc = launch_direct_init(op, st->dp, dg.table, (u64*)st->acc, (u64*)st->acc + dg.table, s);
    if (rc == DTB_OK && minmax_zero_sign(op, value_stype)) {
      if (cudaMalloc(&st->inv, sizeof(int32_t) * (size_t)g->nrows) != cudaSuccess ||
          cudaMalloc(&st->first_zero, sizeof(u64) * (size_t)g->ngroups) != cudaSuccess) {
        cudaGetLastError(); set_error("out of device memory"); rc = DTB_ENOMEM;
      }
      if (rc == DTB_OK) rc = launch_inverse_order((const int32_t*)g->order, g->nrows, (int32_t*)st->inv, s);
      if (rc == DTB_OK) fill_u64((u64*)st->first_zero, g->ngroups, ~0ull, s);
    }
  }
  if (rc != DTB_OK) {
    cudaStreamSynchronize(s);
    cudaFree(st->acc); cudaFree(st->dmap); cudaFree(st->inv); cudaFree(st->first_zero); delete st;
    return rc;
  }
  *out = st;
  return DTB_OK;
}

int dtb_groupby_reduce_add(dtb_reduce_state* st, const void* value_rows, int64_t row0, int64_t nrows, dtb_stream stream)
{
  cudaStream_t s = (cudaStream_t)stream;
  if (!st || !st->g) { set_error("reducer state is NULL"); return DTB_EINVAL; }
  dtb_groupby* g = st->g;
  if (row0 < 0 || nrows < 0 || row0 + nrows > g->nrows) { set_error("row range outside the frame"); return DTB_EINVAL; }
  if (nrows == 0 || g->ngroups == 0) return DTB_OK;
  if (!value_rows || !is_device_ptr(value_rows)) { set_error("piecewise reducers take device rows"); return DTB_EINVAL; }
  KeyPlan kp = g->direct.kp;                        // the key columns, advanced to row0
  for (int c = 0; c < kp.nkeys; c++)
    kp.k[c].data = (const char*)kp.k[c].data + (size_t)row0 * stype_bytes(kp.k[c].stype);
  ProfScope ps("reduce_direct", s);
  DTB_TRY(launch_direct_accumulate_rows(st->op, kp, st->dp, value_rows, st->stype, nrows,
                                        (u64*)st->acc, (u64*)st->acc + g->direct.table, s));
  if (st->first_zero)
    DTB_TRY(launch_first_zero_rows(value_rows, st->stype, row0, nrows, (const int32_t*)st->inv, (const int32_t*)g->offsets,
                                   g->ngroups, (u64*)st->first_zero, s));
  st->rows_added += nrows;
  return DTB_OK;
}

int dtb_groupby_reduce_end(dtb_reduce_state* st, dtb_stream stream, void* out)
{
  cudaStream_t s = (cudaStream_t)stream;
  if (!st || !st->g) { set_error("reducer state is NULL"); return DTB_EINVAL; }
  dtb_groupby* g = st->g;
  int rc = DTB_OK;
  if (g->ngroups > 0) {
    if (!out) { set_error("out is NULL"); rc = DTB_EINVAL; }
    else if (st->rows_added != g->nrows) { set_error("the pieces do not cover the frame's rows exactly once"); rc = DTB_EINVAL; }
    else {
      ArenaScope scope(s);
      rc = scope.rc;
      DevOut d_out;
      if (rc == DTB_OK) rc = d_out.bind(out, (size_t)g->ngroups * stype_bytes(st->out_stype), s);
      GroupRows rows;
      rows.first_zero = (const u64*)st->first_zero;
      if (rc == DTB_OK)
        rc = launch_direct_finalize(st->op, st->stype, (const u64*)st->acc, (const u64*)st->acc + g->direct.table, st->dp,
                                    (const uint32_t*)g->direct.gkeys, g->ngroups, d_out.dptr, rows, s);
      if (rc == DTB_OK && d_out.staged()) rc = d_out.finish((size_t)g->ngroups * stype_bytes(st->out_stype), s);
      if (rc == DTB_OK && cudaStreamSynchronize(s) != cudaSuccess) { set_error("cudaStreamSynchronize failed"); rc = DTB_ECUDA; }
    }
  }
  if (rc != DTB_OK) cudaStreamSynchronize(s);       // the tables may still be in use
  cudaFree(st->acc); cudaFree(st->dmap); cudaFree(st->inv); cudaFree(st->first_zero);
  delete st;
  return rc;
}

int dtb_gather(dtb_col src, int64_t nrows_src, const void* order, int order_is64, int64_t n,
               dtb_stream stream, void* out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  const int esz = stype_bytes(src.stype);
  if (!esz) { set_error("Unable to gather Column of stype " + std::to_string(src.stype)); return DTB_ENOTIMPL; }
  if (n < 0 || nrows_src < 0) { set_error("negative size"); return DTB_EINVAL; }
  if (n > 0 && (!order || !out)) { set_error("order/out is NULL"); return DTB_EINVAL; }
  DTB_TRY(ensure_context());
  if (n == 0) return DTB_OK;
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  DevIn d_src, d_ord;
  DTB_TRY(d_src.bind(src.data, (size_t)nrows_src * esz, s));
  DTB_TRY(d_ord.bind(order, (size_t)n * (order_is64 ? 8 : 4), s));
  DevOut d_out; DTB_TRY(d_out.bind(out, (size_t)n * esz, s));
  DTB_TRY(launch_gather(d_src.dptr, src.stype, nrows_src, d_ord.dptr, order_is64, n, d_out.dptr, s));
  if (d_out.staged()) {
    DTB_TRY(d_out.finish((size_t)n * esz, s));
    DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  return DTB_OK;
}

int dtb_dense_scatter(const void* keys, int key_stype, const void* vals, int64_t n, int64_t kmin, int64_t table_size,
                      void* table, void* present, dtb_stream stream)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  const int kb = (key_stype == DTB_STYPE_INT32) ? 4 : (key_stype == DTB_STYPE_INT64 ? 8 : 0);
  if (!kb) { set_error("dense merge: group keys must be int32 or int64"); return DTB_ENOTIMPL; }
  if (n < 0 || table_size < 1 || (n > 0 && (!keys || !vals)) || !table || !present) { set_error("bad dtb_dense_scatter arguments"); return DTB_EINVAL; }
  if (table_size % 1024 || table_size > ((int64_t)1 << 22)) {
    set_error("dense merge: table size must be a multiple of 1024 and at most 2^22"); return DTB_EINVAL;
  }
  if (!is_device_ptr(table) || !is_device_ptr(present) || (n > 0 && (!is_device_ptr(keys) || !is_device_ptr(vals)))) {
    set_error("dense merge works on device buffers (they are NCCL all-reduced in place)"); return DTB_EINVAL;
  }
  DTB_TRY(ensure_context());
  return launch_dense_scatter(keys, kb, vals, n, kmin, table_size, table, (uint32_t*)present, s);
}

int dtb_dense_compact(const void* table, const void* present, int64_t table_size, int64_t kmin, int key_stype,
                      void* out_keys, void* out_vals, int64_t* ngroups_out, dtb_stream stream)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  const int kb = (key_stype == DTB_STYPE_INT32) ? 4 : (key_stype == DTB_STYPE_INT64 ? 8 : 0);
  if (!kb) { set_error("dense merge: group keys must be int32 or int64"); return DTB_ENOTIMPL; }
  if (!table || !present || !out_keys || !out_vals || !ngroups_out) { set_error("NULL argument"); return DTB_EINVAL; }
  if (table_size < 1024 || table_size % 1024 || table_size > ((int64_t)1 << 22)) {
    set_error("dense merge: table size must be a multiple of 1024 and at most 2^22"); return DTB_EINVAL;
  }
  if (!is_device_ptr(table) || !is_device_ptr(present) || !is_device_ptr(out_keys) || !is_device_ptr(out_vals)) {
    set_error("dense merge works on device buffers"); return DTB_EINVAL;
  }
  DTB_TRY(ensure_context());
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  DevBuf offs, gidx, scr;
  DTB_TRY(offs.alloc(sizeof(int32_t) * (size_t)(table_size + 1), s));
  DTB_TRY(gidx.alloc(sizeof(u32) * (size_t)(table_size + 1), s));
  DTB_TRY(scr.alloc(sizeof(u64) * (size_t)(2 * table_size / 1024 + 4), s));
  u64* d_ng = scr.as<u64>() + 2 * table_size / 1024 + 2;
  DTB_CUDA_CHECK(cudaMemsetAsync(d_ng, 0, 2 * sizeof(u64), s));
  DTB_TRY(launch_offsets_from_counts((const u32*)present, table_size, 0, offs.as<int32_t>(), gidx.as<u32>(), d_ng, scr.as<u64>(), s));
  u64 h_ng = 0;
  DTB_CUDA_CHECK(cudaMemcpyAsync(&h_ng, d_ng, sizeof(u64), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  *ngroups_out = (int64_t)h_ng;
  DTB_TRY(launch_dense_emit(gidx.as<u32>(), table, (int64_t)h_ng, kmin, kb, out_keys, out_vals, s));
  return DTB_OK;
}

// group() of the rows of every group of (order, offsets) by the composite key (group id, value), NA first: the group
// id and the value seen through the RowIndex at every one of its n positions.  flag = DTB_FLAG_SORT_ONLY: the RowIndex
// alone (dtb_sort_grouped); 0: also the Groupby, whose groups are the distinct values inside every group (dtb_qcut).
// gv.res.order holds RowIndex positions; gv.ord is the RowIndex itself (a materialised identity when order is NULL).
struct GroupedByValue {
  DevBuf gid, vg, iota;
  const void* ord = nullptr;
  GroupResult res;
};

static int group_by_value(dtb_col value, int64_t nrows_value, const void* order, const int32_t* offsets,
                          int64_t ngroups, int64_t n, int flag, cudaStream_t s, GroupedByValue& gv)
{
  DTB_TRY(gv.gid.alloc((size_t)n * 4, s));
  DTB_TRY(gv.vg.alloc((size_t)n * stype_bytes(value.stype), s));
  DTB_TRY(launch_expand_gid(offsets, ngroups, n, gv.gid.as<int32_t>(), s));
  gv.ord = order;
  if (!gv.ord) {
    DTB_TRY(gv.iota.alloc((size_t)n * 4, s)); DTB_TRY(launch_iota32(gv.iota.as<int32_t>(), n, s)); gv.ord = gv.iota.p;
  }
  DTB_TRY(launch_gather(value.data, value.stype, nrows_value, gv.ord, 0, n, gv.vg.p, s));
  dtb_col keys[2] = {{gv.gid.p, DTB_STYPE_INT32, 0}, {gv.vg.p, value.stype, 0}};
  const int flags[2] = {flag, flag};
  return group_core(keys, 2, flags, DTB_NA_FIRST, n, s, nullptr, nullptr, gv.res);
}

int dtb_sort_grouped(dtb_col value, int64_t nrows_value, const void* order, const void* offsets, int64_t ngroups,
                     dtb_stream stream, void* order_out)
{
  Grouped c(stream, {value}, nrows_value, order, 0, offsets, ngroups, order_out);
  if (!stype_supported(value.stype)) { set_error("Unable to sort Column of stype " + std::to_string(value.stype)); return DTB_ENOTIMPL; }
  c.per_position = true;
  DTB_TRY(c.open(sizeof(int32_t)));
  if (c.n == 0) return DTB_OK;
  GroupedByValue gv;
  DTB_TRY(group_by_value(dtb_col{c.val[0].dptr, value.stype, 0}, nrows_value, c.ord.dptr, c.offs(), ngroups, c.n,
                         DTB_FLAG_SORT_ONLY, c.s, gv));
  // positions -> rows
  DTB_TRY(launch_gather(gv.ord, DTB_STYPE_INT32, c.n, gv.res.order.p, 0, c.n, c.dout.dptr, c.s));
  return c.finish(true);
}

int dtb_qcut(dtb_col value, int64_t nrows_value, const void* order, const void* offsets, int64_t ngroups,
             int nquantiles, dtb_stream stream, void* out)
{
  Grouped c(stream, {value}, nrows_value, order, 0, offsets, ngroups, out);
  if (nquantiles <= 0) {
    set_error("Number of quantiles must be positive, instead got: " + std::to_string(nquantiles)); return DTB_EINVAL;
  }
  DTB_TRY(fixed_width(value.stype, "qcut()"));
  c.within_column = c.per_position = true;
  DTB_TRY(c.open(sizeof(int32_t)));
  if (c.n == 0) return DTB_OK;
  GroupedByValue gv;
  DTB_TRY(group_by_value(dtb_col{c.val[0].dptr, value.stype, 0}, nrows_value, c.ord.dptr, c.offs(), ngroups, c.n, 0,
                         c.s, gv));
  const int64_t nc = gv.res.ngroups;
  DevBuf scr; DTB_TRY(scr.alloc(qcut_scratch_bytes(nc, ngroups), c.s));
  DTB_TRY(launch_qcut(gv.vg.p, value.stype, gv.res.order.as<int32_t>(), gv.res.offsets.as<int32_t>(), nc,
                      gv.gid.as<int32_t>(), ngroups, c.n, nquantiles, scr.p, (int32_t*)c.dout.dptr, c.s));
  return c.finish(true);
}

int dtb_cut(dtb_col value, int64_t nrows_value, const void* order, int order_is64, int64_t n, int nbins,
            const double* edges, int64_t nedges, int right_closed, dtb_stream stream, void* out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (!edges) {
    if (nbins <= 0) { set_error("Number of bins must be positive, instead got: " + std::to_string(nbins)); return DTB_EINVAL; }
  } else {
    if (nedges < 2) { set_error("To bin data at least two edges are required"); return DTB_EINVAL; }
    if (edges[0] != edges[0]) { set_error("Bin edges must be numeric values only: edge 0 is NaN"); return DTB_EINVAL; }
    for (int64_t i = 1; i < nedges; i++)
      if (!(edges[i] > edges[i - 1])) {            // NaN fails the comparison too
        set_error("Bin edges must be strictly increasing: edges " + std::to_string(i - 1) + " and " + std::to_string(i));
        return DTB_EINVAL;
      }
  }
  DTB_TRY(fixed_width(value.stype, "cut()"));
  if (value.stype == DTB_STYPE_DATE32 || value.stype == DTB_STYPE_TIME64) {
    set_error("cut() can only be applied to numeric columns, instead got stype " + std::to_string(value.stype));
    return DTB_EINVAL;
  }
  if (n < 0 || nrows_value < 0) { set_error("negative size"); return DTB_EINVAL; }
  if (!value.data && nrows_value > 0) { set_error("value column data is NULL"); return DTB_EINVAL; }
  if (!order && n > 0 && n != nrows_value) { set_error("without an order, n must equal nrows_value"); return DTB_EINVAL; }
  if (!out && n > 0) { set_error("out is NULL"); return DTB_EINVAL; }
  DTB_TRY(ensure_context());
  if (n == 0) return DTB_OK;
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  DevIn d_val, d_ord;
  DTB_TRY(d_val.bind(value.data, (size_t)nrows_value * stype_bytes(value.stype), s));
  DTB_TRY(d_ord.bind(order, (size_t)n * (order_is64 ? 8 : 4), s));
  DevOut d_out; DTB_TRY(d_out.bind(out, (size_t)n * 4, s));
  if (!edges) {
    DevBuf st; DTB_TRY(st.alloc(sizeof(ColStats) + sizeof(CutCoef), s));
    ColStats* d_stats = st.as<ColStats>();
    CutCoef* d_coef = (CutCoef*)(d_stats + 1);
    {
      ProfScope ps("cut_stats", s);
      if (d_ord.dptr) DTB_TRY(launch_col_stats_gather(d_val.dptr, value.stype, nrows_value, d_ord.dptr, order_is64, n,
                                                      d_stats, s));
      else            DTB_TRY(launch_col_stats(d_val.dptr, value.stype, n, d_stats, s));
      DTB_TRY(launch_cut_coef(d_stats, value.stype, nbins, right_closed ? 1 : 0, d_coef, s));
    }
    {
      ProfScope ps("cut_emit", s);
      DTB_TRY(launch_cut_emit(d_val.dptr, value.stype, nrows_value, d_ord.dptr, order_is64, n, d_coef,
                              (int32_t*)d_out.dptr, s));
    }
  } else {
    DevIn d_edges; DTB_TRY(d_edges.bind(edges, sizeof(double) * (size_t)nedges, s));
    ProfScope ps("cut_bins", s);
    DTB_TRY(launch_cut_bins(d_val.dptr, value.stype, nrows_value, d_ord.dptr, order_is64, n,
                            (const double*)d_edges.dptr, nedges, right_closed ? 1 : 0, (int32_t*)d_out.dptr, s));
  }
  if (d_out.staged()) {
    DTB_TRY(d_out.finish((size_t)n * 4, s));
    DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  return DTB_OK;
}

int dtb_set_select(int mode, const void* order, const void* offsets, int64_t ngroups, const int64_t* cum_sizes,
                   int ninputs, dtb_stream stream, void* rows_out, int64_t* nout)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (mode < DTB_SET_UNION || mode > DTB_SET_SYMDIFF) { set_error("unknown set operation"); return DTB_EINVAL; }
  if (ngroups < 0 || !nout || ninputs < 1 || ninputs > 64 || !cum_sizes) { set_error("bad dtb_set_select arguments"); return DTB_EINVAL; }
  *nout = 0;
  DTB_TRY(ensure_context());
  if (ngroups == 0) return DTB_OK;
  if (!order || !offsets || !rows_out) { set_error("NULL argument"); return DTB_EINVAL; }
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  const int64_t n = cum_sizes[ninputs - 1];
  DevIn d_ord, d_off;
  DTB_TRY(d_ord.bind(order, (size_t)n * 4, s));
  DTB_TRY(d_off.bind(offsets, sizeof(int32_t) * (size_t)(ngroups + 1), s));
  DevOut d_out; DTB_TRY(d_out.bind(rows_out, (size_t)ngroups * 4, s));
  DevBuf d_sizes, flags, pos, oscr;
  DTB_TRY(d_sizes.alloc(sizeof(int64_t) * (size_t)ninputs, s));
  DTB_CUDA_CHECK(cudaMemcpyAsync(d_sizes.p, cum_sizes, sizeof(int64_t) * (size_t)ninputs, cudaMemcpyHostToDevice, s));
  const int64_t m = ngroups + 1;                          // flags[0] = sentinel head for the compaction
  DTB_TRY(flags.alloc((size_t)m + 64, s));
  DTB_CUDA_CHECK(cudaMemsetAsync(flags.p, 0, (size_t)m + 64, s));
  DTB_TRY(launch_set_select((const int32_t*)d_ord.dptr, (const int32_t*)d_off.dptr, ngroups, d_sizes.as<int64_t>(),
                            ninputs, mode, flags.as<uint8_t>(), s));
  const int64_t otiles = offsets_num_tiles(m);
  DTB_TRY(pos.alloc(sizeof(int32_t) * (size_t)(m + 1), s));
  DTB_TRY(oscr.alloc(sizeof(u64) * (size_t)(otiles + 4), s));
  DTB_CUDA_CHECK(cudaMemsetAsync(oscr.p, 0, oscr.bytes, s));
  u64* d_ng = oscr.as<u64>() + otiles + 2;
  DTB_TRY(launch_group_offsets(flags.p, 1, 0, m, pos.as<int32_t>(), d_ng, oscr.as<u64>(), s));
  u64 h_ng = 0;
  DTB_CUDA_CHECK(cudaMemcpyAsync(&h_ng, d_ng, sizeof(u64), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  const int64_t nsel = (int64_t)h_ng - 1;                 // without the sentinel
  DTB_TRY(launch_set_emit(pos.as<int32_t>(), nsel, (const int32_t*)d_ord.dptr, (const int32_t*)d_off.dptr,
                          (int32_t*)d_out.dptr, s));
  if (d_out.staged()) DTB_TRY(d_out.finish((size_t)nsel * 4, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  *nout = nsel;
  return DTB_OK;
}

int dtb_largest_group(const void* offsets, int64_t ngroups, int64_t skip, dtb_stream stream, int64_t* index_out,
                      int64_t* size_out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (!index_out || !size_out || ngroups < 0 || skip < 0) { set_error("bad dtb_largest_group arguments"); return DTB_EINVAL; }
  *index_out = -1; *size_out = 0;
  DTB_TRY(ensure_context());
  if (ngroups <= skip) return DTB_OK;
  if (!offsets) { set_error("offsets is NULL"); return DTB_EINVAL; }
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  DevIn d_off; DTB_TRY(d_off.bind(offsets, sizeof(int32_t) * (size_t)(ngroups + 1), s));
  DevBuf r; DTB_TRY(r.alloc(sizeof(u64), s));
  DTB_CUDA_CHECK(cudaMemsetAsync(r.p, 0, sizeof(u64), s));
  DTB_TRY(launch_largest_group((const int32_t*)d_off.dptr, ngroups, skip, r.as<u64>(), s));
  u64 h = 0;
  DTB_CUDA_CHECK(cudaMemcpyAsync(&h, r.p, sizeof(u64), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  if (h) { *size_out = (int64_t)(h >> 32); *index_out = (int64_t)(0xffffffffu - (u32)(h & 0xffffffffu)); }
  return DTB_OK;
}

int dtb_slice_groups(const void* offsets, int64_t ngroups, int64_t start, int64_t stop, int64_t step,
                     dtb_stream stream, void* rows_out, int64_t rows_capacity, void* offsets_out,
                     int64_t* ngroups_out, int64_t* nrows_out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (!ngroups_out || !nrows_out || ngroups < 0 || rows_capacity < 0) { set_error("bad dtb_slice_groups arguments"); return DTB_EINVAL; }
  *ngroups_out = 0; *nrows_out = 0;
  if (ngroups > 0 && (!offsets || !offsets_out)) { set_error("offsets / offsets_out is NULL"); return DTB_EINVAL; }
  if (step == DTB_SLICE_NA) step = 1;                                   // fexpr_literal_sliceint.cc:86
  if (step != (int64_t)(int32_t)step) { set_error("slice step does not fit int32"); return DTB_EINVAL; }
  if (step == 0 && (start == DTB_SLICE_NA || stop == DTB_SLICE_NA || stop <= 0 || stop > (int64_t)INT32_MAX)) {
    set_error("a slice with step 0 needs a start and a positive count"); return DTB_EINVAL;    // the reference asserts it (:150-152)
  }
  DTB_TRY(ensure_context());
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  if (ngroups == 0) {
    if (offsets_out) {
      DevOut z; DTB_TRY(z.bind(offsets_out, sizeof(int32_t), s));
      DTB_CUDA_CHECK(cudaMemsetAsync(z.dptr, 0, sizeof(int32_t), s));
      DTB_TRY(z.finish(sizeof(int32_t), s));
      DTB_CUDA_CHECK(cudaStreamSynchronize(s));
    }
    return DTB_OK;
  }
  DevIn d_off; DTB_TRY(d_off.bind(offsets, sizeof(int32_t) * (size_t)(ngroups + 1), s));
  DevOut d_oo; DTB_TRY(d_oo.bind(offsets_out, sizeof(int32_t) * (size_t)(ngroups + 1), s));
  int32_t h_last = 0;                                                   // rows of the grouped frame
  DTB_CUDA_CHECK(cudaMemcpyAsync(&h_last, (const int32_t*)d_off.dptr + ngroups, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  SliceParams p;
  p.has_start = start != DTB_SLICE_NA; p.has_stop = stop != DTB_SLICE_NA;
  p.start = p.has_start ? start : 0; p.stop = p.has_stop ? stop : 0; p.step = step; p.nrows = (long long)(u32)h_last;
  DevBuf scr, gsel, tot;
  DTB_TRY(scr.alloc(slice_scratch_bytes(ngroups), s));
  DTB_TRY(gsel.alloc(sizeof(int32_t) * (size_t)ngroups, s));
  DTB_TRY(tot.alloc(2 * sizeof(u64), s));
  DTB_TRY(launch_slice_groups_plan((const int32_t*)d_off.dptr, ngroups, p, scr.p, (int32_t*)d_oo.dptr, gsel.as<int32_t>(),
                                   tot.as<u64>(), s));
  u64 h_tot[2] = {0, 0};
  DTB_CUDA_CHECK(cudaMemcpyAsync(h_tot, tot.p, sizeof(h_tot), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  const int64_t nout = (int64_t)h_tot[0], ng_out = (int64_t)h_tot[1];
  *nrows_out = nout; *ngroups_out = ng_out;
  if (nout > (int64_t)INT32_MAX) { set_error("the slice selects more than INT32_MAX rows"); return DTB_ENOTIMPL; }
  if (nout > rows_capacity) { set_error("rows_out is too small: " + std::to_string(nout) + " rows selected"); return DTB_ENOSPACE; }
  const int32_t h_end = (int32_t)nout;
  DTB_CUDA_CHECK(cudaMemcpyAsync((int32_t*)d_oo.dptr + ng_out, &h_end, sizeof(int32_t), cudaMemcpyHostToDevice, s));
  if (nout > 0) {
    if (!rows_out) { set_error("rows_out is NULL"); return DTB_EINVAL; }
    DevOut d_rows; DTB_TRY(d_rows.bind(rows_out, sizeof(int32_t) * (size_t)nout, s));
    DevBuf gid; DTB_TRY(gid.alloc(sizeof(int32_t) * (size_t)nout, s));
    DTB_TRY(launch_slice_groups_emit((const int32_t*)d_off.dptr, p, (const int32_t*)d_oo.dptr, gsel.as<int32_t>(), ng_out, nout,
                                     gid.as<int32_t>(), (int32_t*)d_rows.dptr, s));
    DTB_TRY(d_rows.finish(sizeof(int32_t) * (size_t)nout, s));
  }
  DTB_TRY(d_oo.finish(sizeof(int32_t) * (size_t)(ng_out + 1), s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  return DTB_OK;
}

int dtb_mask_rows(dtb_col mask, int64_t nrows, dtb_stream stream, void* rows_out, int64_t rows_capacity,
                  int64_t* nrows_out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (!nrows_out) { set_error("nrows_out is NULL"); return DTB_EINVAL; }
  if (mask.stype != DTB_STYPE_BOOL) {
    set_error("dtb_mask_rows takes a bool8 column, not stype " + std::to_string(mask.stype)); return DTB_EINVAL;
  }
  if (nrows < 0 || nrows > (int64_t)INT32_MAX) { set_error("nrows must be in 0..INT32_MAX"); return DTB_EINVAL; }
  if (rows_capacity < 0) { set_error("rows_capacity must be non-negative"); return DTB_EINVAL; }
  if (nrows > 0 && !mask.data) { set_error("mask data is NULL"); return DTB_EINVAL; }
  if (rows_capacity > 0 && !rows_out) { set_error("rows_out is NULL"); return DTB_EINVAL; }
  *nrows_out = 0;
  DTB_TRY(ensure_context());
  if (nrows == 0) return DTB_OK;
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  DevIn d_mask; DTB_TRY(d_mask.bind(mask.data, (size_t)nrows, s));
  DevBuf tiles, tot;
  DTB_TRY(tiles.alloc(sizeof(u64) * (size_t)mask_num_tiles(nrows), s));
  DTB_TRY(tot.alloc(sizeof(u64), s));
  DTB_TRY(launch_mask_count((const int8_t*)d_mask.dptr, nrows, tiles.as<u64>(), tot.as<u64>(), s));
  u64 h_tot = 0;                                                        // the one wait: the result's size
  DTB_CUDA_CHECK(cudaMemcpyAsync(&h_tot, tot.p, sizeof(u64), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  const int64_t nout = (int64_t)h_tot;
  *nrows_out = nout;
  if (nout > rows_capacity) { set_error("rows_out is too small: " + std::to_string(nout) + " rows selected"); return DTB_ENOSPACE; }
  if (nout == 0) return DTB_OK;
  DevOut d_rows; DTB_TRY(d_rows.bind(rows_out, sizeof(int32_t) * (size_t)nout, s));
  DTB_TRY(launch_mask_emit((const int8_t*)d_mask.dptr, nrows, tiles.as<u64>(), (int32_t*)d_rows.dptr, s));
  if (d_rows.staged()) {
    DTB_TRY(d_rows.finish(sizeof(int32_t) * (size_t)nout, s));
    DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  return DTB_OK;
}

int dtb_int_rows(dtb_col sel, int64_t nrows, dtb_stream stream, void* rows_out, int64_t* min_out, int64_t* max_out,
                 int64_t* nacount_out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (!min_out || !max_out || !nacount_out) { set_error("min_out / max_out / nacount_out is NULL"); return DTB_EINVAL; }
  const int st = sel.stype;
  if (st != DTB_STYPE_INT8 && st != DTB_STYPE_INT16 && st != DTB_STYPE_INT32 && st != DTB_STYPE_INT64) {
    set_error("dtb_int_rows takes an int8, int16, int32 or int64 column, not stype " + std::to_string(st));
    return DTB_EINVAL;
  }
  if (nrows < 0 || nrows > (int64_t)INT32_MAX) { set_error("nrows must be in 0..INT32_MAX"); return DTB_EINVAL; }
  if (nrows > 0 && !sel.data) { set_error("selector data is NULL"); return DTB_EINVAL; }
  if (nrows > 0 && st != DTB_STYPE_INT32 && !rows_out) { set_error("rows_out is NULL"); return DTB_EINVAL; }
  *min_out = 0; *max_out = 0; *nacount_out = 0;
  DTB_TRY(ensure_context());
  if (nrows == 0) return DTB_OK;
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  const size_t esz = stype_bytes(st);
  DevIn d_sel; DTB_TRY(d_sel.bind(sel.data, (size_t)nrows * esz, s));
  DevOut d_rows; DTB_TRY(d_rows.bind(rows_out, sizeof(int32_t) * (size_t)nrows, s));
  if (rows_out) {
    if (st == DTB_STYPE_INT32)
      DTB_CUDA_CHECK(cudaMemcpyAsync(d_rows.dptr, d_sel.dptr, sizeof(int32_t) * (size_t)nrows, cudaMemcpyDeviceToDevice, s));
    else
      DTB_TRY(launch_narrow_rows(d_sel.dptr, st, nrows, (int32_t*)d_rows.dptr, s));
    DTB_TRY(d_rows.finish(sizeof(int32_t) * (size_t)nrows, s));
  }
  DevBuf d_stats; DTB_TRY(d_stats.alloc(sizeof(ColStats), s));
  DTB_TRY(launch_col_stats(d_sel.dptr, st, nrows, d_stats.as<ColStats>(), s));
  ColStats h;
  DTB_CUDA_CHECK(cudaMemcpyAsync(&h, d_stats.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  DTB_CUDA_CHECK(cudaStreamSynchronize(s));                             // the one wait: the statistics
  *nacount_out = (int64_t)h.nacount;
  if (h.nvalid) { *min_out = (int64_t)h.lo; *max_out = (int64_t)h.hi; }
  return DTB_OK;
}

int dtb_join(const dtb_col* xkeys, const dtb_col* jkeys, int nkeys, int64_t nrows_x, int64_t nrows_j,
             dtb_stream stream, void* index_out)
{
  return dtb_join_gather(xkeys, jkeys, nkeys, nrows_x, nrows_j, nullptr, 0, stream, index_out, nullptr);
}

int dtb_join_gather(const dtb_col* xkeys, const dtb_col* jkeys, int nkeys, int64_t nrows_x, int64_t nrows_j,
                    const dtb_col* jvals, int nvals, dtb_stream stream, void* index_out, void* const* vals_out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (nkeys < 1 || nkeys > MAX_KEYS || !xkeys || !jkeys) { set_error("number of key columns must be in 1.." + std::to_string(MAX_KEYS)); return DTB_EINVAL; }
  if (nvals < 0 || (nvals > 0 && (!jvals || !vals_out))) { set_error("bad join value columns"); return DTB_EINVAL; }
  for (int c = 0; c < nvals; c++) {
    if (!stype_supported(jvals[c].stype)) {
      set_error("Unable to join a column of stype " + std::to_string(jvals[c].stype)); return DTB_ENOTIMPL;
    }
  }
  if (nrows_x < 0 || nrows_j < 0 || nrows_j > (int64_t)INT32_MAX) { set_error("bad row counts"); return DTB_EINVAL; }
  for (int c = 0; c < nkeys; c++) {
    if (!stype_supported(xkeys[c].stype) || !stype_supported(jkeys[c].stype)) {
      set_error("join keys of stype " + std::to_string(xkeys[c].stype) + " / " + std::to_string(jkeys[c].stype) + " are not supported");
      return DTB_ENOTIMPL;
    }
    const bool xd = xkeys[c].stype == DTB_STYPE_DATE32 || xkeys[c].stype == DTB_STYPE_TIME64;
    const bool jd = jkeys[c].stype == DTB_STYPE_DATE32 || jkeys[c].stype == DTB_STYPE_TIME64;
    if ((xd || jd) && xkeys[c].stype != jkeys[c].stype) {       // join.cc:384-385: date/time only join their own type
      set_error("a date/time key column can only be joined to a column of the same type"); return DTB_EINVAL;
    }
  }
  DTB_TRY(ensure_context());
  if (nrows_x == 0) return DTB_OK;
  if (!index_out && nvals == 0) { set_error("index_out is NULL"); return DTB_EINVAL; }
  for (int c = 0; c < nvals; c++) if (!vals_out[c]) { set_error("vals_out[" + std::to_string(c) + "] is NULL"); return DTB_EINVAL; }
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  std::vector<DevIn> xin(nkeys), jin(nkeys), vin(nvals);
  std::vector<DevOut> vout(nvals);
  const void* xp[MAX_KEYS]; const void* jp[MAX_KEYS]; int xst[MAX_KEYS], jst[MAX_KEYS];
  for (int c = 0; c < nkeys; c++) {
    DTB_TRY(xin[c].bind(xkeys[c].data, (size_t)nrows_x * stype_bytes(xkeys[c].stype), s));
    DTB_TRY(jin[c].bind(jkeys[c].data, (size_t)nrows_j * stype_bytes(jkeys[c].stype), s));
    xp[c] = xin[c].dptr; jp[c] = jin[c].dptr; xst[c] = xkeys[c].stype; jst[c] = jkeys[c].stype;
  }
  std::vector<const void*> vp(nvals); std::vector<void*> op(nvals); std::vector<int> vst(nvals);
  for (int c = 0; c < nvals; c++) {
    const size_t esz = stype_bytes(jvals[c].stype);
    DTB_TRY(vin[c].bind(jvals[c].data, (size_t)nrows_j * esz, s));
    DTB_TRY(vout[c].bind(vals_out[c], (size_t)nrows_x * esz, s));
    vp[c] = vin[c].dptr; op[c] = vout[c].dptr; vst[c] = jvals[c].stype;
  }
  DevOut d_out; DTB_TRY(d_out.bind(index_out, (size_t)nrows_x * 4, s));
  DTB_TRY(launch_join(nkeys, xp, xst, jp, jst, nrows_x, nrows_j, (int32_t*)d_out.dptr, nvals, vp.data(), vst.data(),
                      op.data(), s));
  bool staged = d_out.staged();
  if (d_out.staged()) DTB_TRY(d_out.finish((size_t)nrows_x * 4, s));
  for (int c = 0; c < nvals; c++) {
    if (!vout[c].staged()) continue;
    DTB_TRY(vout[c].finish((size_t)nrows_x * stype_bytes(jvals[c].stype), s));
    staged = true;
  }
  if (staged) DTB_CUDA_CHECK(cudaStreamSynchronize(s));
  return DTB_OK;
}

int dtb_cache_begin(void) {
  t_cache.depth++;
  return DTB_OK;
}

int dtb_cache_end(void) {
  if (t_cache.depth > 0 && --t_cache.depth == 0) { cudaDeviceSynchronize(); t_cache.clear(); }
  return DTB_OK;
}

int dtb_lower_bound(dtb_col sorted, int64_t nrows, dtb_col values, int64_t nvalues, dtb_stream stream, void* out)
{
  cudaStream_t s = (cudaStream_t)stream;
  t_stats = dtb_call_stats{0, 0, 0, 0, 0};
  if (sorted.stype != values.stype || !stype_supported(sorted.stype)) { set_error("lower_bound: columns must share a supported stype"); return DTB_EINVAL; }
  if (nrows < 0 || nvalues < 0 || (nvalues > 0 && (!values.data || !out))) { set_error("bad dtb_lower_bound arguments"); return DTB_EINVAL; }
  DTB_TRY(ensure_context());
  if (nvalues == 0) return DTB_OK;
  ArenaScope scope(s); if (scope.rc != DTB_OK) return scope.rc;
  const int esz = stype_bytes(sorted.stype);
  DevIn d_s, d_v;
  DTB_TRY(d_s.bind(sorted.data, (size_t)nrows * esz, s));
  DTB_TRY(d_v.bind(values.data, (size_t)nvalues * esz, s));
  DevOut d_out; DTB_TRY(d_out.bind(out, (size_t)nvalues * 8, s));
  DTB_TRY(launch_lower_bound(d_s.dptr, sorted.stype, nrows, d_v.dptr, nvalues, (int64_t*)d_out.dptr, s));
  if (d_out.staged()) { DTB_TRY(d_out.finish((size_t)nvalues * 8, s)); DTB_CUDA_CHECK(cudaStreamSynchronize(s)); }
  return DTB_OK;
}

}  // extern "C"
