// pm_engine.cu — the engine behind include/prime_match.h.
//
// One engine = one CUDA device + one stream.  pm_match() is the management pass
// that replaces NodeGroupsPlugin::try_form_new_groups (reference
// crates/orchestrator/src/plugins/node_groups/mod.rs:478-628): for tiles of asks
// (configurations, priority order) x all candidate workers it builds the int64
// cost matrix in HBM, reduces it (per-ask argmin, per-worker first feasible ask)
// and then runs the resolution sweep that reproduces the reference's sequential
// greedy allocation bit for bit.  There is no CPU fallback: without an sm_90
// device (H100) pm_create fails with PM_E_NO_DEVICE.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>

#include <cuda.h>   // driver types and prototypes only: the entry points are resolved at run time (TileBuf)
#include <dlfcn.h>
#include <nccl.h>   // types and prototypes only: the library is resolved at run time (nccl_api below), never linked

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "pm_guard.hpp"
#include "pm_kernels.cuh"
#include "pm_proximity.cuh"
#include "pm_proximity_grid.cuh"
#include "pm_auction.cuh"
#include "pm_auction_cert.cuh"

struct pm_engine;

namespace {

std::string g_create_error;

template <class T> struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaError_t ensure(size_t want) {
    if (want <= n && p) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
    if (want == 0) want = 1;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) n = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  // capacity >= want, the first `keep` elements preserved, everything after them zero
  cudaError_t grow_keep(size_t want, size_t keep, cudaStream_t st) {
    if (want <= n && p) return cudaSuccess;
    const size_t cap = std::max<size_t>(want + want / 4, 1);
    T* q = nullptr;
    cudaError_t e = cudaMalloc(&q, cap * sizeof(T));
    if (e != cudaSuccess) return e;
    keep = p ? std::min(keep, n) : 0;
    if (keep) e = cudaMemcpyAsync(q, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(q + keep, 0, (cap - keep) * sizeof(T), st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { cudaFree(q); return e; }
    if (p) cudaFree(p);
    p = q;
    n = cap;
    return cudaSuccess;
  }
};
template <class T> struct PinBuf {
  T* p = nullptr;
  size_t n = 0;
  cudaError_t ensure(size_t want) {
    if (want <= n && p) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    n = 0;
    if (want == 0) want = 1;
    cudaError_t e = cudaMallocHost(&p, want * sizeof(T));
    if (e == cudaSuccess) n = want;
    return e;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    n = 0;
  }
};

// The cost tile, in compressible device memory where the device offers it (generic compute-data compression): the L2
// stores runs of equal words — the "infeasible" sentinel of the 32-bit tile, 0x7FFFFFFF_FFFFFFFF of the int64 one — to
// HBM in compressed form and reads them back the same way, so the HBM traffic of a sparse tile shrinks while its layout,
// contents and the kernels stay what they are.  Elsewhere (or when the driver refuses), plain cudaMalloc.  The driver's
// virtual-memory calls are looked up at run time: the library keeps no link-time dependency on libcuda.
//
// `held` describes the buffer, whatever wrote it: one byte per 4 KB of it (a row slot's 1024-column stripe of the 32-bit
// tile), bit j set when its 512-byte block j — one warp's 128 columns — holds kNarrowInfeasible in every word.  Indexed
// by offset, it stays true across changes of ld or of the rows per tile (ld is a multiple of 1024 columns, so every
// layout's blocks are the same 512-byte blocks).  pm_build_argmin_feat reads and writes it, and skips the stores of a
// block that is all infeasible and already holds the sentinel.  Any other writer of the buffer calls overwritten();
// the next pm_build_argmin_feat pass then zeroes the map (prepare_held) and writes every block once more.
//
// `priced` is its twin, indexed the same way: bit j set when block j holds this pass's column prices in every word (a
// row feasible in all 128 columns), and pm_build_argmin_feat skips the store of such a row's block there too.  A
// block's two bits are never both set.  The prices and the column order are the pass's own, so prepare_held zeroes
// `priced` at every pass start; within a pass no other writer touches the buffer.
struct TileBuf {
  long long* p = nullptr;
  size_t n = 0;
  CUmemGenericAllocationHandle h = 0;   // non-zero: compressible mapping of `bytes` bytes at p
  size_t bytes = 0;
  uint8_t* held = nullptr;              // [held_bytes()], then `priced` in the same allocation
  uint8_t* priced = nullptr;            // [held_bytes()]
  bool held_valid = false;              // false: the map is stale, every block must be written

  size_t held_bytes() const { return (n * sizeof(long long) + 4095) / 4096; }
  void overwritten() { held_valid = false; }
  // once per pm_build_argmin_feat pass, in stream order (no host synchronisation): `priced` zeroed, and `held` too
  // when it is stale (one memset over both)
  cudaError_t prepare_held(cudaStream_t st) {
    const cudaError_t e = held_valid ? cudaMemsetAsync(priced, 0, held_bytes(), st)
                                     : cudaMemsetAsync(held, 0, 2 * held_bytes(), st);
    held_valid = e == cudaSuccess;
    return e;
  }

  struct Api {
    decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
    decltype(&cuMemCreate) create = nullptr;
    decltype(&cuMemRelease) release = nullptr;
    decltype(&cuMemAddressReserve) reserve = nullptr;
    decltype(&cuMemAddressFree) address_free = nullptr;
    decltype(&cuMemMap) map = nullptr;
    decltype(&cuMemUnmap) unmap = nullptr;
    decltype(&cuMemSetAccess) set_access = nullptr;
    decltype(&cuMemGetAllocationPropertiesFromHandle) props = nullptr;
    bool ok = false;
  };
  static const Api& api() {
    static const Api a = [] {
      Api x;
      auto get = [](const char* name, auto** fn) {
        cudaDriverEntryPointQueryResult q{};
        void* f = nullptr;
        if (cudaGetDriverEntryPoint(name, &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
          cudaGetLastError();
          return false;
        }
        *fn = reinterpret_cast<std::remove_pointer_t<decltype(fn)>>(f);
        return f != nullptr;
      };
      x.ok = get("cuMemGetAllocationGranularity", &x.granularity) && get("cuMemCreate", &x.create) &&
             get("cuMemRelease", &x.release) && get("cuMemAddressReserve", &x.reserve) &&
             get("cuMemAddressFree", &x.address_free) && get("cuMemMap", &x.map) && get("cuMemUnmap", &x.unmap) &&
             get("cuMemSetAccess", &x.set_access) && get("cuMemGetAllocationPropertiesFromHandle", &x.props);
      return x;
    }();
    return a;
  }

  // one compressible mapping of at least `want_bytes`, or false (nothing held)
  bool map_compressible(int device, size_t want_bytes) {
    const Api& a = api();   // a device without compression fails cuMemCreate or grants an uncompressed handle
    if (!a.ok) return false;
    CUmemAllocationProp prop{};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device;
    prop.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
    size_t gran = 0;
    if (a.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS || gran == 0) return false;
    const size_t size = (want_bytes + gran - 1) / gran * gran;
    CUmemGenericAllocationHandle hh = 0;
    if (a.create(&hh, size, &prop, 0) != CUDA_SUCCESS) return false;
    CUmemAllocationProp got{};
    CUdeviceptr ptr = 0;
    bool ok = a.props(&got, hh) == CUDA_SUCCESS && got.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC &&
              a.reserve(&ptr, size, 0, 0, 0) == CUDA_SUCCESS;
    if (ok && a.map(ptr, size, 0, hh, 0) != CUDA_SUCCESS) {
      a.address_free(ptr, size);
      ok = false;
    }
    if (ok) {
      CUmemAccessDesc acc{};
      acc.location = prop.location;
      acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      if (a.set_access(ptr, size, &acc, 1) != CUDA_SUCCESS) {
        a.unmap(ptr, size);
        a.address_free(ptr, size);
        ok = false;
      }
    }
    if (!ok) {
      a.release(hh);
      return false;
    }
    p = reinterpret_cast<long long*>(ptr);
    h = hh;
    bytes = size;
    return true;
  }

  // capacity >= want elements; the old contents are not kept.  The caller has ordered every use of the old tile before
  // this call (a pass's kernels are joined into the engine stream, which is synchronised here).
  cudaError_t ensure(size_t want, int device, bool compress, cudaStream_t st) {
    if (want <= n && p) return cudaSuccess;
    if (p) {
      cudaError_t e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) return e;
    }
    release();
    if (want == 0) want = 1;
    cudaError_t e = cudaSuccess;
    if (!(compress && map_compressible(device, want * sizeof(long long)))) e = cudaMalloc(&p, want * sizeof(long long));
    if (e != cudaSuccess) {
      p = nullptr;
      return e;
    }
    n = want;
    e = cudaMalloc(&held, 2 * held_bytes());
    if (e != cudaSuccess) {
      held = nullptr;
      release();
      return e;
    }
    priced = held + held_bytes();
    return e;
  }
  void release() {
    if (held) cudaFree(held);
    held = priced = nullptr;
    held_valid = false;
    if (h) {
      const Api& a = api();
      a.unmap(reinterpret_cast<CUdeviceptr>(p), bytes);
      a.address_free(reinterpret_cast<CUdeviceptr>(p), bytes);
      a.release(h);
    } else if (p) {
      cudaFree(p);
    }
    p = nullptr;
    n = 0;
    h = 0;
    bytes = 0;
  }
};

inline unsigned blocks_for(size_t n, unsigned threads) { return (unsigned)((n + threads - 1) / threads); }

// NCCL is plumbing for the one exchange of a sharded pass.  It is looked up at run time so that the library loads
// (and every single-GPU path works) on hosts without it: first among the symbols already in the process (a host that
// has NCCL loaded, e.g. through torch, shares its copy), then by soname.
struct NcclApi {
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommInitAll) CommInitAll = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclCommAbort) CommAbort = nullptr;
  decltype(&ncclAllGather) AllGather = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  bool ok = false;
  std::string err;
};
const NcclApi& nccl_api() {
  static const NcclApi api = [] {
    NcclApi a;
    void* h = dlsym(RTLD_DEFAULT, "ncclAllGather") ? RTLD_DEFAULT : nullptr;
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { a.err = "NCCL not found (libnccl.so.2): multi-GPU matching needs it"; return a; }
#define PM_NCCL_SYM(name) a.name = reinterpret_cast<decltype(a.name)>(dlsym(h, "nccl" #name)); if (!a.name) { a.err = "libnccl: missing nccl" #name; return a; }
    PM_NCCL_SYM(GetUniqueId) PM_NCCL_SYM(CommInitRank) PM_NCCL_SYM(CommInitAll) PM_NCCL_SYM(CommDestroy)
    PM_NCCL_SYM(CommAbort) PM_NCCL_SYM(AllGather) PM_NCCL_SYM(GetErrorString)
#undef PM_NCCL_SYM
    a.ok = true;
    return a;
  }();
  return api;
}

}  // namespace

struct pm_comm {
  ncclComm_t nccl = nullptr;
  uint32_t n_ranks = 1, rank = 0;
  int device = 0;
};

struct pm_engine {
  pm_cfg cfg{};
  int device = 0;
  unsigned sms = 132;     // streaming multiprocessors of the device (an H100 SXM has 132): caps of the grid-stride launches
  cudaStream_t stream = nullptr;
  std::string err;
  std::mutex mu;

  // tables
  uint32_t n_workers = 0, n_asks = 0, n_opts = 0;
  uint32_t n_patterns = 0, n_models = 0, words = 1;
  uint32_t max_pattern_row = 0;
  bool have_workers = false, have_asks = false, have_bits = false, have_loc = false, have_rank = false;
  bool all_solo = true;  // every enabled ask has min == max == 1
  // The enabled-configuration mask (pm_set_ask_enabled): the host copy is the mask; the converted rows carry it
  // (pm_ask_convert).  Per ask its kind (kAskKindNotSolo / kAskKindMaxZero), and how many enabled asks have each kind:
  // the per-table facts all_solo and any_max_zero are taken over the enabled asks.
  std::vector<uint8_t> ask_on, ask_kind;
  uint32_t n_off = 0, n_on_not_solo = 0, n_on_max_zero = 0;
  static constexpr uint8_t kAskKindNotSolo = 1, kAskKindMaxZero = 2;
  void count_kind(uint32_t t, int d) {
    if (ask_kind[t] & kAskKindNotSolo) n_on_not_solo += d;
    if (ask_kind[t] & kAskKindMaxZero) n_on_max_zero += d;
    all_solo = n_on_not_solo == 0;
    any_max_zero = n_on_max_zero != 0;
  }
  int tune_generic = 0, tune_auction = 0, tune_prox = 0, tune_auc_good = 0, tune_auc_extra = 0;   // PM_TUNE_*: diagnostics
  bool tune_wide = false;  // PM_TUNE_BUILD=8: the int64 cost tile on the FastRow path too (the 32-bit tile's reference)
  int tune_compress = 1;  // PM_TUNE_COMPRESS=0: the cost tile in plain cudaMalloc memory (A/B runs)
  DevBuf<uint4> wa, wb;
  DevBuf<double> lat, lon;
  DevBuf<uint32_t> addr_rank;
  DevBuf<pm::DevAsk> asks;
  DevBuf<pm::DevOpt> opts;
  DevBuf<pm::DevOptF> opts_fast;
  DevBuf<pm::FastRow> frows;
  bool rows_bound = false;     // FastRow.wp matches the current model table (pm_bind_rows)
  bool rows_auction = false;   // the enabled max_group_size == 0 asks are in the auction's form (use_ask_form)
  bool rows_bound_wm = false;  // ... bound to the worker-major one-word table
  DevBuf<uint32_t> nacc, bits_wm;   // worker-major acceptance (pm_worker_nacc) and its one-word table ~(1 << row)
  bool nacc_valid = false;
  DevBuf<pm_ask> raw_asks;
  DevBuf<pm_gpu_opt> raw_opts;
  DevBuf<uint32_t> ask_counts, ask_newoff;
  // The caller's rows as raw_asks holds them (opt_off into raw_opts), kept on the host so that pm_update_asks and
  // pm_resize_asks can check a delta against the whole table before anything changes.  raw_n_opts: rows of raw_opts in
  // use (replaced rows leave theirs behind until a compaction); opt_rows / live_opts: the sums over the asks of
  // max(n_opts, 1) (the converted table's rows) and of n_opts.
  std::vector<pm_ask> asks_h;
  uint32_t raw_n_opts = 0;
  uint64_t opt_rows = 0, live_opts = 0;
  DevBuf<pm_ask> upd_asks;             // staging of pm_update_asks / pm_resize_asks
  bool asks_small = true;      // every ask operand fits the fast predicate (pm_device.cuh DevOptF)
  bool workers_small = false;  // ... and every worker operand (checked on the device)
  bool prices_narrow = false;  // every worker price < 0x7FFFFFFF: the first-fit tile can hold the 32-bit cost word alone
  bool workers_checked = false;
  DevBuf<uint32_t> amin, amax, bits;
  DevBuf<uint32_t> scratch_idx, scratch_flags;
  DevBuf<uint4> upd_a, upd_b;          // staging of pm_update_workers (and of pm_insert_workers' rows)
  DevBuf<double> upd_lat, upd_lon;
  // pm_remove_workers / pm_insert_workers: the second buffer of every per-row column (each splice writes the moved
  // table into these and swaps them with the live ones), and the removed rows and positions (wsplice_dev)
  DevBuf<uint4> wa_alt, wb_alt;
  DevBuf<double> lat_alt, lon_alt;
  DevBuf<uint32_t> rank_alt, rep_alt, nacc_alt, first_alt, owner_alt, wsplice_dev;
  DevBuf<long long> price_alt;
  uint64_t table_version = 0;          // bumped by every call that changes a table (pm_table_version)

  // evaluation
  TileBuf cost;
  size_t cost_tile_used = 0;           // bytes of `cost` the last materialised pass laid its tiles over (PM_BUF_COST_TILE)
  DevBuf<uint32_t> first_ask, ask_count;
  DevBuf<long long> ask_best;
  DevBuf<uint32_t> stripe_rank;        // pm_stripe_rank, once per pass of pm_build_argmin: [ld] column -> rank in its stripe
  DevBuf<long long> rank_best;         // ... [ld] stripe * 1024 + rank -> (price << 32) | worker
  // The feature dictionary of the converted ask table (convert_asks; pm_kernels.cuh FeatDict): feat_ok when it fits
  // the 64-bit word, and then pm_build_argmin_feat runs in place of pm_build_argmin.  Its per-pass rows: feat_w
  // [ld] per column, feat_a [n_asks] per ask, feat_o [option rows] per further OR-option.  Its column order
  // (pm_feature_keys): the sort's keys and values feat_key / feat_val, sorted into feat_key_s / feat_perm, all [ld].
  pm::FeatDict feat{};
  bool feat_ok = false;
  DevBuf<uint32_t> feat_buf;
  PinBuf<uint32_t> h_feat;
  DevBuf<uint4> feat_w, feat_a;
  DevBuf<uint2> feat_o;
  DevBuf<unsigned long long> feat_key, feat_key_s;
  DevBuf<uint32_t> feat_val, feat_perm;
  // Its slot schedule (pm_sched_keys / pm_sched_gather), [n_asks] each: the sort's keys and asks sched_key / sched_val,
  // sorted into sched_key_s / sched_val_s; the launches' rows and asks in write order, sched_row / sched_ask.
  DevBuf<unsigned long long> sched_key, sched_key_s;
  DevBuf<uint32_t> sched_val, sched_val_s, sched_ask;
  DevBuf<uint4> sched_row;

  // The stored evaluation of PM_INCREMENTAL: the per-worker first feasible ask of the last evaluation of this engine's
  // range (shard()), PM_NONE outside it, in its own buffer (first_ask is the resolution's working copy: the sweeps, the
  // exchange and the auction overwrite it), and the worker rows written since then.  Rows are tracked on the host,
  // where their indices arrive: a mark per row and the list of marked rows.  The list holds every written row of the
  // range, which the walks re-evaluate, and the written rows outside it, which only the O(W) preludes read (decide_fast,
  // worker_major: they describe the whole replicated table).  `dirty_over` once more rows of the range changed than
  // an incremental pass would take (tune_incr); `rows_over` once more rows outside it did: the list then stops taking
  // them and the preludes check every row.
  DevBuf<uint32_t> eval_first;
  bool eval_valid = false;
  std::vector<uint8_t> dirty_mark;      // [rows of the stored evaluation, grown with the table]; set <=> in dirty_rows
  std::vector<uint32_t> dirty_rows;
  uint32_t dirty_in = 0;                // entries of dirty_rows inside the range
  bool dirty_over = false, rows_over = false;
  bool workers_base = false;            // workers_small / prices_narrow hold for every row outside dirty_rows
  bool nacc_base = false;               // nacc holds every row outside dirty_rows (model table unchanged)
  uint32_t tune_incr = 1u << 18;        // PM_TUNE_INCR: most dirty rows an incremental pass re-evaluates (DESIGN §5)
  PinBuf<uint32_t> h_dirty;
  DevBuf<uint32_t> dirty_dev;
  DevBuf<unsigned long long> incr_evals;
  bool incr_evals_pending = false;      // stats.evals of the incremental pass arrives with the pass's one sync
  // The mask the stored evaluation was taken under (eval_on) and the asks toggled, replaced or appended since (toggled,
  // each once; an ask switched off and on again is listed but has eval_on == ask_on; replaced: repl_mark).  Appended
  // asks have eval_on == 0.  orph_mark: the next kept row of a removed ask that had workers (pm_remove_asks moved their
  // stored first ask onto it).  walk_start: the orphan walk's start bounds.
  std::vector<uint8_t> eval_on, toggle_mark, repl_mark, orph_mark;
  std::vector<uint32_t> toggled;
  DevBuf<uint32_t> walk_start, toggle_dev, splice_dev;   // splice_dev: pm_remove_asks / pm_insert_asks staging

  // E (enabled since the stored evaluation) and D (disabled since), increasing; a D entry is ask << 1 | replaced.  A
  // replaced row counts as disabled and enabled again: in E when it is enabled now, in D when it was at the stored
  // evaluation, its orphans walked from the ask itself.  An orph_mark row is in D with the bit too, whatever its own
  // state: the workers of the removed ask share its index now, and are walked from it (the E-pass skips a worker's
  // stored ask, so listing it in E alone would not test them against it).
  void split_toggles(std::vector<uint32_t>* en, std::vector<uint32_t>* dis) const {
    en->clear();
    dis->clear();
    for (uint32_t t : toggled) {
      if (repl_mark[t]) {
        if (ask_on[t]) en->push_back(t);
        if (eval_on[t] || orph_mark[t]) dis->push_back(t << 1 | 1u);
      } else {
        if (ask_on[t] && !eval_on[t]) en->push_back(t);
        if (orph_mark[t]) dis->push_back(t << 1 | 1u);
        else if (!ask_on[t] && eval_on[t]) dis->push_back(t << 1);
      }
    }
    std::sort(en->begin(), en->end());
    std::sort(dis->begin(), dis->end());
  }
  void clear_toggled() {
    for (uint32_t t : toggled) { toggle_mark[t] = 0; repl_mark[t] = 0; orph_mark[t] = 0; eval_on[t] = ask_on[t]; }
    toggled.clear();
  }
  void mark_toggled(uint32_t t) {
    if (eval_valid && !toggle_mark[t]) {
      toggle_mark[t] = 1;
      toggled.push_back(t);
    }
  }
  void clear_dirty() {
    for (uint32_t i : dirty_rows) dirty_mark[i] = 0;
    dirty_rows.clear();
    dirty_in = 0;
    dirty_over = rows_over = false;
  }
  void invalidate_eval() {
    clear_dirty();
    clear_toggled();
    eval_valid = false;
    workers_base = nacc_base = false;
  }
  bool in_range(uint32_t i) const {
    uint32_t w0 = 0, nw = 0;
    shard(&w0, &nw);
    return i - w0 < nw;
  }
  void mark_dirty(uint32_t i) {
    if (!eval_valid || dirty_over || i >= dirty_mark.size() || dirty_mark[i]) return;
    const bool in = in_range(i);
    if (!in && rows_over) return;
    dirty_mark[i] = 1;
    dirty_rows.push_back(i);
    dirty_in += in;
    if (dirty_in > tune_incr) mark_all_dirty();
    else if (dirty_rows.size() - dirty_in > tune_incr) rows_over = true;
  }
  void mark_range_dirty(uint32_t first, uint32_t n) {
    if (!eval_valid || dirty_over) return;
    uint32_t w0 = 0, nw = 0;
    shard(&w0, &nw);
    const uint64_t lo = std::max<uint64_t>(first, w0), hi = std::min<uint64_t>((uint64_t)first + n, (uint64_t)w0 + nw);
    const uint64_t inside = hi > lo ? hi - lo : 0;
    if (inside > tune_incr) { mark_all_dirty(); return; }
    if (n - inside > tune_incr) rows_over = true;   // the rows outside the range are not listed
    if (rows_over) {
      for (uint64_t i = lo; i < hi; ++i) mark_dirty((uint32_t)i);
    } else {
      for (uint32_t i = 0; i < n; ++i) mark_dirty(first + i);
    }
  }
  void mark_all_dirty() {   // the next pass evaluates everything
    if (!eval_valid) return;
    clear_dirty();
    dirty_over = true;
  }

  // resolution
  DevBuf<uint32_t> keys, keys_sorted, iota, order, hist, seg_start, ngroups, group_base;
  DevBuf<uint32_t> base_len, xhead, xnext, xcount, popped, counters;  // counters: [0]=any_bad [1]=n_bumped
  DevBuf<unsigned char> cub_tmp;
  DevBuf<uint32_t> prox_list, prox_xs, members_raw;
  DevBuf<double> prox_dist;
  DevBuf<double> pg_part_d, pg_clat, pg_clon, pg_ccos;
  DevBuf<uint32_t> pg_part_i, pg_cta_cnt, pg_ctl;
  int coop_blocks = -1;   // co-resident CTAs of pm_proximity_grid on this device (0: cooperative launch unavailable)
  bool any_max_zero = false;
  // extension (auction) state
  DevBuf<uint32_t> price_cap, auc_owner, auc_assigned, auc_withdrawn, auc_active, auc_bid_w, auc_winner, auc_flag, auc_gidx;
  DevBuf<long long> auc_price, auc_bid_p, auc_bid_max, auc_theta;
  DevBuf<uint32_t> auc_cand, auc_theta_w, auc_pool, auc_pool_bound_w;
  DevBuf<long long> auc_pool_bound_v;
  DevBuf<uint32_t> auc_class_of, auc_class_rep, auc_class_req, auc_class_list, auc_retry, auc_fallback;
  DevBuf<uint32_t> auc_walk_list, auc_split_w, auc_split_ticket;
  DevBuf<long long> auc_split_v;
  DevBuf<uint32_t> auc_perm, auc_pos_of, auc_idx, auc_sorted, auc_incl;
  DevBuf<uint64_t> auc_hash, auc_hash_out, auc_ckey, auc_ckey_s;
  DevBuf<uint4> auc_wa_s, auc_wb_s;
  DevBuf<long long> auc_price_s;
  DevBuf<pm::AuctionCtl> auc_ctl;
  PinBuf<pm::AuctionCtl> h_ctl;
  uint32_t auc_n_classes = 0;
  bool auc_classes_valid = false;
  bool have_caps = false;
  DevBuf<uint32_t> auc_split_first;
  DevBuf<uint64_t> auc_skip_key;
  DevBuf<uint32_t> reputation, ask_min_rep, auc_rep_s;   // extension: worker reputation column, per-ask floor, sorted copy
  bool have_rep = false, have_min_rep = false;
  uint64_t auc_scale = 1, auc_eps_start = 1;
  uint32_t auc_eps_div = 4;
  // Auction warm start (PM_AUCTION_WARM).  The stored state is auc_price / auc_owner / auc_assigned as the last auction
  // pass left them, over auc_state_w rows, with the caps and floors it ran with.  Rows and asks changed since are tracked
  // here, apart from the reference modes' dirty_rows / toggled (a reference-mode pass clears those): rows below auc_kept
  // one by one (auc_rows, each once; auc_rows_over past the cutoff), every row from auc_kept on as a range (rows a
  // shrink cut off, or a resize added), and the asks toggled since.  Changed caps and floors are found by a diff.
  bool auc_state = false;
  uint32_t auc_state_w = 0, auc_kept = 0;
  std::vector<uint8_t> auc_row_mark, auc_ask_mark;
  std::vector<uint32_t> auc_rows, auc_toggled;
  bool auc_rows_over = false;
  std::vector<uint32_t> cap_host, floor_host, auc_cap_stored, auc_floor_stored;
  bool auc_last_warm = false;   // pm_auction_state: the last pass
  uint32_t auc_last_released = 0;
  uint32_t auc_last_phases = 0, auc_last_rev_rounds = 0;   // pm_auction_reverse_stats: the last pass (0 without the bit)
  uint64_t auc_last_rev_bids = 0;
  DevBuf<uint32_t> auc_raised, auc_mark, auc_cmin, auc_chg;
  // reverse rounds (PM_AUCTION_REVERSE): bidder list and offers, per-ask profits and caps in class order, class runs
  DevBuf<uint32_t> auc_rev_bidders, auc_rev_offer_t, auc_rev_win, auc_rev_cap_s, auc_rev_cstart;
  DevBuf<long long> auc_rev_offer_p, auc_rev_best, auc_rev_pi_s;
  // pm_auction_certificate's own scratch: row minima, held-pair feasibility, ownership counts, row terms, accumulators
  DevBuf<uint64_t> cert_min, cert_acc;
  DevBuf<uint32_t> cert_ok, cert_own, cert_none;   // cert_none: [T] no holds, the per-ask sweep's view with demands
  DevBuf<long long> cert_bound;
  PinBuf<uint64_t> h_cert_acc;
  PinBuf<long long> h_cert_bound;
  // pm_auction_restore's staging: the caller's prices and assignment, the kept assignment (per slot with demands: D
  // entries), the rebuilt owners, the counts
  DevBuf<long long> rst_price;
  DevBuf<uint32_t> rst_assigned, rst_kept, rst_owner;
  DevBuf<uint64_t> rst_acc;
  PinBuf<uint64_t> h_rst_acc;
  // pm_resize_asks / pm_remove_asks / pm_insert_asks since the stored state: the removed asks that held a kept row
  // (those rows are unowned now, at their stored prices; they count against the cutoff), and whether rows were removed
  // or added at all (the certificate then waits for the next pass)
  uint32_t auc_removed_held = 0;
  bool auc_asks_resized = false;
  // pm_remove_workers / pm_insert_workers since the stored state (the certificate then waits for the next pass)
  bool auc_workers_spliced = false;
  // Ask demands (pm_set_ask_demand; the auction only): empty while every ask takes one worker, and the auction then runs
  // on the ask table itself.  Else the demands and their exclusive scan over T + 1 (host, and device in dem_off): ask t
  // is the auction's bidders (slots) dem_off[t] .. dem_off[t + 1] - 1, and the stored assignment is per slot.  The pass
  // builds the slot table (each slot's ask, and copies of its converted row, cap and floor) and runs on it.
  // auc_dem_kept[t]: the leading slots of ask t that can carry a stored hold since the last pass (empty: all of them);
  // a demand change lowers it, and the slots past it are in A0.
  std::vector<uint32_t> demand, dem_off_h, auc_dem_kept;
  DevBuf<uint32_t> dem_off, dem_off_old, slot_ask, slot_cap, slot_floor, auc_assigned_tmp, dem_members, dem_spos, dem_aflag;
  DevBuf<pm::DevAsk> slot_row;
  uint32_t n_slots() const { return demand.empty() ? n_asks : dem_off_h[n_asks]; }
  uint32_t slot0(uint32_t t) const { return demand.empty() ? t : dem_off_h[t]; }
  void auc_discard() {
    auc_state = false;
    auc_dem_kept.clear();
    auc_rows.clear();
    auc_toggled.clear();
    auc_row_mark.clear();
    auc_ask_mark.clear();
    auc_rows_over = false;
    auc_removed_held = 0;
    auc_asks_resized = false;
    auc_workers_spliced = false;
  }
  void auc_mark_ask(uint32_t t) {   // A0: toggled, replaced or appended since the stored state
    if (auc_state && !auc_ask_mark[t]) {
      auc_ask_mark[t] = 1;
      auc_toggled.push_back(t);
    }
  }
  void auc_mark_row(uint32_t i) {
    if (!auc_state || auc_rows_over || i >= auc_kept || auc_row_mark[i]) return;
    auc_row_mark[i] = 1;
    auc_rows.push_back(i);
    if (auc_rows.size() > tune_incr) auc_rows_over = true;
  }
  void auc_mark_rows(uint32_t first, uint32_t n) {
    if (!auc_state) return;
    const uint32_t hi = (uint32_t)std::min<uint64_t>((uint64_t)first + n, auc_kept);
    for (uint32_t i = first; i < hi && !auc_rows_over; ++i) auc_mark_row(i);
  }
  DevBuf<uint32_t> worker_group, worker_ask, group_ask, group_off, members;
  PinBuf<uint32_t> h_scalars;  // small D2H mailbox

  // result (pinned host)
  PinBuf<uint32_t> r_worker_group, r_worker_ask, r_group_ask, r_group_off, r_members, r_ask_count;
  PinBuf<long long> r_ask_best;
  uint32_t n_groups = 0, n_assigned = 0;
  bool matched = false, local_done = false;

  // multi-GPU: the communicator this engine exchanges through (not owned), and the packed exchange buffers
  pm_comm* comm = nullptr;
  DevBuf<unsigned char> xchg_send, xchg_recv;

  // The contiguous canonical-order range of workers this engine evaluates: the whole table, the range fixed by
  // pm_cfg / pm_set_shard, or — with a communicator attached — the rank's equal share.
  void shard(uint32_t* w0, uint32_t* nw) const {
    const uint32_t W = n_workers;
    if (comm) {
      const uint32_t per = (uint32_t)(((uint64_t)W + comm->n_ranks - 1) / comm->n_ranks);
      *w0 = (uint32_t)std::min<uint64_t>((uint64_t)comm->rank * per, W);
      *nw = std::min(per, W - *w0);
    } else {
      *w0 = cfg.shard_first;
      *nw = cfg.shard_count ? cfg.shard_count : (W > *w0 ? W - *w0 : 0);
    }
  }

  pm_stats stats{};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool own_stream = true;
  struct TimedRegion { cudaEvent_t a, b; float* acc; };
  std::vector<cudaEvent_t> ev_pool;     // grows on demand, reused across matches
  std::vector<TimedRegion> ev_pending;
  size_t ev_used = 0;
  cudaEvent_t take_event() {
    if (ev_used == ev_pool.size()) {
      cudaEvent_t ev = nullptr;
      if (cudaEventCreate(&ev) != cudaSuccess) return nullptr;
      ev_pool.push_back(ev);
    }
    return ev_pool[ev_used++];
  }
  void resolve_timers() {  // caller has synchronised the stream
    for (auto& r : ev_pending) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) *r.acc += ms;
    }
    ev_pending.clear();
    ev_used = 0;
  }

  int fail(pm_status st, const std::string& msg) {
    err = msg;
    return st;
  }
};

#define PM_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) {                                                            \
      return e->fail(PM_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e));    \
    }                                                                                   \
  } while (0)

#define PM_LAUNCH_CHECK(name)                                                           \
  do {                                                                                  \
    cudaError_t _e = cudaGetLastError();                                                \
    if (_e != cudaSuccess)                                                              \
      return e->fail(PM_E_CUDA, std::string("launch ") + name + ": " + cudaGetErrorString(_e)); \
    ++e->stats.n_launches;                                                              \
  } while (0)

namespace {

// Per-launch CUDA-event timing without host synchronisation: start/stop events
// are recorded around a region on the stream its kernels run on and resolved in
// one go at the end of the match (which synchronises anyway to read the group
// count).
struct Timer {
  pm_engine* e;
  float* acc;
  cudaStream_t st;
  bool on;
  size_t slot = 0;
  Timer(pm_engine* e_, float* acc_, cudaStream_t st_);
  void stop();
};

Timer::Timer(pm_engine* e_, float* acc_, cudaStream_t st_)
    : e(e_), acc(acc_), st(st_), on((e_->cfg.flags & PM_CFG_TIMING) != 0) {
  if (!on) return;
  cudaEvent_t a = e->take_event(), b = e->take_event();
  if (!a || !b) { on = false; return; }
  slot = e->ev_pending.size();
  e->ev_pending.push_back({a, b, acc});
  cudaEventRecord(a, st);
}
void Timer::stop() {
  if (!on) return;
  cudaEventRecord(e->ev_pending[slot].b, st);
  on = false;
}

pm::EvalParams eval_params(pm_engine* e) {
  pm::EvalParams p;
  p.wa = e->wa.p;
  p.wb = e->wb.p;
  p.asks = e->asks.p;
  p.opts = e->opts.p;
  p.opts_fast = e->opts_fast.p;
  p.frows = e->frows.p;
  p.bits = e->bits.p;
  p.nacc = nullptr;
  p.words = e->words;
  p.n_workers = e->n_workers;
  p.n_asks = e->n_asks;
  p.n_opts = e->n_opts;
  p.n_bits_rows = e->have_bits ? e->n_patterns + 1 : 1;
  p.sign_shift = 31;
  return p;
}

pm::AskTables ask_tables(pm_engine* e) {
  return pm::AskTables{e->asks.p, e->opts.p, e->opts_fast.p, e->frows.p, e->amin.p, e->amax.p};
}

// PM_MODE_AUCTION has no group sizes: its feasibility is candidate, compatible, cap and floor (prime_match.h), so an ask
// with max_group_size == 0, which the reference modes never fill, bids like any other there.  The converted rows carry
// the reference modes' clause; the auction and its certificate convert the enabled max_group_size == 0 asks again
// without it (auction = true), and the next call that reads the rows for a reference mode or toggles an ask converts
// them back.  Nothing else changes: a table without such asks is never converted again.
static int use_ask_form(pm_engine* e, bool auction) {
  if (e->rows_auction == auction) return PM_OK;
  std::vector<uint32_t> list;   // ask << 1 | enabled, as pm_ask_toggle takes it
  for (uint32_t t = 0; t < e->n_asks; ++t)
    if ((e->ask_kind[t] & pm_engine::kAskKindMaxZero) && e->ask_on[t]) list.push_back(t << 1 | 1u);
  if (!list.empty()) {
    PM_CUDA(cudaSetDevice(e->device));
    PM_CUDA(e->toggle_dev.ensure(list.size()));
    PM_CUDA(cudaMemcpyAsync(e->toggle_dev.p, list.data(), list.size() * 4, cudaMemcpyHostToDevice, e->stream));
    pm::pm_ask_toggle<<<blocks_for(list.size(), 256), 256, 0, e->stream>>>(e->raw_asks.p, e->raw_opts.p, e->ask_newoff.p,
                                                                         e->toggle_dev.p, (uint32_t)list.size(),
                                                                         ask_tables(e), !auction);
    PM_LAUNCH_CHECK("pm_ask_toggle");
    PM_CUDA(cudaStreamSynchronize(e->stream));   // `list` is a local
    e->rows_bound = false;
    e->auc_classes_valid = false;
  }
  e->rows_auction = auction;
  return PM_OK;
}

// The feature dictionary from the values pm_feature_collect left in h_feat: per kind the distinct values in increasing
// order, bit positions in kind order.  The candidate and never bits are always features (pm_kernels.cuh FeatDict).
static void build_feat_dict(pm_engine* e) {
  const uint32_t* h = e->h_feat.p;
  std::vector<uint32_t> vals[pm::kFeatKinds];
  const uint32_t pres = h[0] | pm::kKeyCandBit | pm::kKeyNeverBit;
  for (uint32_t j = 0; j < pm::kKeyPresence; ++j)
    if ((pres >> j) & 1u) vals[pm::kFeatKey].push_back(j);
  size_t n = vals[pm::kFeatKey].size();
  for (uint32_t k = 1; k < pm::kFeatKinds; ++k) {
    for (uint32_t i = 0; i < pm::kFeatSlots; ++i) {
      const uint32_t v = h[2 + (k - 1) * pm::kFeatSlots + i];
      if (v != pm::kNone) vals[k].push_back(v);
    }
    std::sort(vals[k].begin(), vals[k].end());
    n += vals[k].size();
  }
  e->feat_ok = h[1] == 0 && n <= pm::kFeatMax;
  e->feat = pm::FeatDict{};
  if (!e->feat_ok) return;
  uint32_t i = 0;
  for (uint32_t k = 0; k < pm::kFeatKinds; ++k) {
    e->feat.off[k] = i;
    for (uint32_t v : vals[k]) e->feat.val[i++] = v;
  }
  e->feat.off[pm::kFeatKinds] = i;
}

// The whole ask table converted from the resident raw rows, O(T + sum K) on the device: pm_ask_counts -> scan ->
// pm_ask_convert.  pm_set_asks and every delta of pm_update_asks / pm_resize_asks take this one path.  Every row comes
// out enabled, in the reference modes' form; *st gets the status bits.  Sets n_opts, max_pattern_row, asks_small and the
// feature dictionary (build_feat_dict).
static int convert_asks(pm_engine* e, uint32_t n_asks, uint32_t n_raw_opts, uint64_t opt_rows, uint32_t* st) {
  PM_CUDA(e->ask_counts.ensure((size_t)n_asks + 1)); PM_CUDA(e->ask_newoff.ensure((size_t)n_asks + 1));
  PM_CUDA(e->asks.ensure(n_asks)); PM_CUDA(e->amin.ensure(n_asks)); PM_CUDA(e->amax.ensure(n_asks));
  const size_t opt_cap = std::max<size_t>(n_raw_opts, (size_t)opt_rows);
  PM_CUDA(e->opts.ensure(opt_cap)); PM_CUDA(e->opts_fast.ensure(opt_cap)); PM_CUDA(e->frows.ensure(n_asks));
  e->rows_bound = false;
  e->rows_auction = false;
  e->auc_classes_valid = false;
  PM_CUDA(cudaMemsetAsync(e->counters.p + 12, 0, 8, e->stream));
  pm::pm_ask_counts<<<blocks_for((size_t)n_asks + 1, 256), 256, 0, e->stream>>>(e->raw_asks.p, n_asks, n_raw_opts, e->ask_counts.p,
                                                                                 e->counters.p + 12);
  PM_LAUNCH_CHECK("pm_ask_counts");
  {
    size_t tmp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp, e->ask_counts.p, e->ask_newoff.p, (int)(n_asks + 1), e->stream);
    PM_CUDA(e->cub_tmp.ensure(tmp));
    PM_CUDA(cub::DeviceScan::ExclusiveSum(e->cub_tmp.p, tmp, e->ask_counts.p, e->ask_newoff.p, (int)(n_asks + 1), e->stream));
  }
  if (n_asks) {
    pm::pm_ask_convert<<<blocks_for(n_asks, 256), 256, 0, e->stream>>>(e->raw_asks.p, e->raw_opts.p, n_asks, e->ask_newoff.p,
                                                                        ask_tables(e), e->counters.p + 12, e->counters.p + 13);
    PM_LAUNCH_CHECK("pm_ask_convert");
  }
  // the feature dictionary's values, collected from the converted rows and returned with this synchronisation
  const size_t feat_words = 2 + (pm::kFeatKinds - 1) * pm::kFeatSlots;
  PM_CUDA(e->feat_buf.ensure(feat_words));
  PM_CUDA(e->h_feat.ensure(feat_words));
  PM_CUDA(cudaMemsetAsync(e->feat_buf.p, 0, 8, e->stream));
  PM_CUDA(cudaMemsetAsync(e->feat_buf.p + 2, 0xFF, (feat_words - 2) * 4, e->stream));
  if (n_asks) {
    pm::pm_feature_collect<<<blocks_for(n_asks, 256), 256, 0, e->stream>>>(e->frows.p, e->opts_fast.p, n_asks, e->feat_buf.p);
    PM_LAUNCH_CHECK("pm_feature_collect");
  }
  PM_CUDA(cudaMemcpyAsync(e->h_feat.p, e->feat_buf.p, feat_words * 4, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 20, e->counters.p + 12, 8, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 22, e->ask_newoff.p + n_asks, 4, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  *st = e->h_scalars.p[20];
  e->n_opts = e->h_scalars.p[22];
  e->max_pattern_row = e->h_scalars.p[21];
  e->asks_small = (*st & pm::kAskNotSmall) == 0;
  build_feat_dict(e);
  return PM_OK;
}

// Per ask its kind, and the per-table facts over the enabled asks (asks_h and ask_on over n_asks)
static void recount_kinds(pm_engine* e) {
  const uint32_t T = e->n_asks;
  e->ask_kind.resize(T);
  e->n_off = e->n_on_not_solo = e->n_on_max_zero = 0;
  for (uint32_t t = 0; t < T; ++t) {
    const pm_ask& a = e->asks_h[t];
    e->ask_kind[t] = (uint8_t)((a.min_group_size == 1 && a.max_group_size == 1 ? 0 : pm_engine::kAskKindNotSolo) |
                               (a.max_group_size == 0 ? pm_engine::kAskKindMaxZero : 0));
    if (e->ask_on[t]) e->count_kind(t, +1);
    else ++e->n_off;
  }
  e->all_solo = e->n_on_not_solo == 0;
  e->any_max_zero = e->n_on_max_zero != 0;
}

// The caller's rows of pm_update_asks (idx given) or pm_resize_asks, checked on the host before anything changes: the
// indices, the group sizes and the option ranges within `opts` of every entry; then, over the distinct entries (the
// last one of an index decides), the converted option rows of the table they make.  The distinct entries go to
// uidx / urows (idx null: rows appended after the n_asks rows there are).
static int check_ask_rows(const pm_engine* e, const char* fn, const uint32_t* idx, const pm_ask* rows, uint32_t n,
                          uint32_t n_opts, std::vector<uint32_t>* uidx, std::vector<pm_ask>* urows, std::string* err) {
  for (uint32_t i = 0; i < n; ++i) {
    if (idx && idx[i] >= e->n_asks) { *err = std::string(fn) + ": ask index out of range"; return PM_E_INVALID; }
    if (rows[i].max_group_size < rows[i].min_group_size) {
      *err = std::string(fn) + ": max_group_size < min_group_size (Plugin configuration is invalid)";
      return PM_E_INVALID;
    }
    if ((uint64_t)rows[i].opt_off + rows[i].n_opts > n_opts) { *err = std::string(fn) + ": option range out of bounds"; return PM_E_INVALID; }
  }
  uidx->clear();
  urows->clear();
  uint64_t opt_rows = e->opt_rows;
  if (idx) {
    std::vector<uint32_t> ord(n);
    for (uint32_t i = 0; i < n; ++i) ord[i] = i;
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return idx[x] < idx[y]; });
    for (uint32_t j = 0; j < n; ++j) {
      if (j + 1 < n && idx[ord[j + 1]] == idx[ord[j]]) continue;
      const uint32_t t = idx[ord[j]];
      uidx->push_back(t);
      urows->push_back(rows[ord[j]]);
      opt_rows -= std::max<uint32_t>(e->asks_h[t].n_opts, 1u);
    }
  } else {
    for (uint32_t i = 0; i < n; ++i) {
      uidx->push_back(e->n_asks + i);
      urows->push_back(rows[i]);
    }
  }
  for (const pm_ask& a : *urows) opt_rows += std::max<uint32_t>(a.n_opts, 1u);
  if (opt_rows >= (1ull << 31)) { *err = std::string(fn) + ": too many option rows"; return PM_E_INVALID; }
  return PM_OK;
}

// Rows removed from and inserted into the ask table (pm_remove_asks, pm_insert_asks; pm_resize_asks is the tail case).
// removed: old indices, increasing and distinct; before: per inserted row the old row it goes before, non-decreasing.
// map: old index -> new index (kNone: removed); at: the new index of each inserted row; succ: per removed row the new
// index of the next kept row (n_new: none).
struct AskSplice {
  uint32_t n_old = 0, n_new = 0;
  std::vector<uint32_t> removed, before, map, at, succ;
  AskSplice(uint32_t n, std::vector<uint32_t> rm, std::vector<uint32_t> bf)
      : n_old(n), removed(std::move(rm)), before(std::move(bf)), map(n), at(before.size()), succ(removed.size()) {
    uint32_t r = 0, i = 0, j = 0;
    for (uint32_t t = 0; t <= n_old; ++t) {
      while (i < before.size() && before[i] == t) at[i++] = j++;
      if (t == n_old) break;
      if (r < removed.size() && removed[r] == t) {
        map[t] = pm::kNone;
        succ[r++] = j;   // a call removes or inserts, never both: the next index handed out is the next kept row's
      } else {
        map[t] = j++;
      }
    }
    n_new = j;
  }
  // every kept row keeps its index: a shrink or a grow (pm_resize_asks)
  bool tail() const {
    return (removed.empty() || removed[0] == n_old - removed.size()) && (before.empty() || before[0] == n_old);
  }
  // a per-ask vector moved with its rows, `fill` in the inserted rows; one of another length (empty: not in use) stays
  template <class V> void apply(std::vector<V>* v, V fill) const {
    if (v->size() != n_old) return;
    std::vector<V> out(n_new, fill);
    for (uint32_t t = 0; t < n_old; ++t)
      if (map[t] != pm::kNone) out[map[t]] = (*v)[t];
    v->swap(out);
  }
  // a list of asks renamed, the removed ones dropped
  void apply_list(std::vector<uint32_t>* list) const {
    size_t k = 0;
    for (uint32_t t : *list)
      if (map[t] != pm::kNone) (*list)[k++] = map[t];
    list->resize(k);
  }
};

// pm_update_asks / pm_resize_asks / pm_remove_asks / pm_insert_asks after their checks (the masks already moved to the
// new table): with a splice, asks_h is moved first and the raw rows go up again unless every kept row keeps its index;
// rows[i] goes to ask idx[i] (distinct, < n_asks), the option range it references in `opts` appended to raw_opts and its
// opt_off rebased onto that copy; raw_opts is compacted when its dead rows outnumber the live ones; then the whole table
// is converted again and the disabled asks are turned off (pm_ask_toggle).
static int commit_asks(pm_engine* e, uint32_t n_asks, const uint32_t* idx, const pm_ask* rows, uint32_t n,
                       const pm_gpu_opt* opts, const AskSplice* sp = nullptr) {
  const uint32_t base = e->raw_n_opts;
  // only the option ranges the new rows reference go up, each row's range after the last, opt_off rebased onto it:
  // a caller may pass its whole option table for one changed ask without leaving that table behind as dead rows
  std::vector<pm_ask> moved(rows, rows + n);
  std::vector<pm_gpu_opt> add;
  for (pm_ask& a : moved) {
    const uint32_t off = base + (uint32_t)add.size();
    add.insert(add.end(), opts + a.opt_off, opts + a.opt_off + a.n_opts);
    a.opt_off = off;
  }
  if (sp) sp->apply(&e->asks_h, pm_ask{});
  e->asks_h.resize(n_asks);
  for (uint32_t i = 0; i < n; ++i) e->asks_h[idx[i]] = moved[i];
  uint64_t opt_rows = 0, live = 0;
  for (const pm_ask& a : e->asks_h) {
    opt_rows += std::max<uint32_t>(a.n_opts, 1u);
    live += a.n_opts;
  }
  const uint64_t raw = (uint64_t)base + add.size();
  if (raw - std::min(raw, live) > live || raw >= (1ull << 31)) {
    // compaction: every ask's options copied once, in ask order, from the rows as they stand (old ones read back)
    std::vector<pm_gpu_opt> all(raw);
    if (base) {
      PM_CUDA(cudaMemcpyAsync(all.data(), e->raw_opts.p, (size_t)base * sizeof(pm_gpu_opt), cudaMemcpyDeviceToHost, e->stream));
      PM_CUDA(cudaStreamSynchronize(e->stream));
    }
    if (!add.empty()) std::memcpy(all.data() + base, add.data(), add.size() * sizeof(pm_gpu_opt));
    std::vector<pm_gpu_opt> packed;
    packed.reserve(live);
    for (pm_ask& a : e->asks_h) {
      const uint32_t off = (uint32_t)packed.size();
      packed.insert(packed.end(), all.begin() + a.opt_off, all.begin() + a.opt_off + a.n_opts);
      a.opt_off = off;
    }
    PM_CUDA(e->raw_asks.ensure(n_asks)); PM_CUDA(e->raw_opts.ensure(packed.size()));
    if (n_asks)
      PM_CUDA(cudaMemcpyAsync(e->raw_asks.p, e->asks_h.data(), (size_t)n_asks * sizeof(pm_ask), cudaMemcpyHostToDevice, e->stream));
    if (!packed.empty())
      PM_CUDA(cudaMemcpyAsync(e->raw_opts.p, packed.data(), packed.size() * sizeof(pm_gpu_opt), cudaMemcpyHostToDevice, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));   // `packed` is a local
    e->raw_n_opts = (uint32_t)packed.size();
  } else {
    if (!add.empty()) {
      PM_CUDA(e->raw_opts.grow_keep(raw, base, e->stream));
      PM_CUDA(cudaMemcpyAsync(e->raw_opts.p + base, add.data(), add.size() * sizeof(pm_gpu_opt), cudaMemcpyHostToDevice, e->stream));
    }
    const bool moved_rows = sp && !sp->tail();
    if (moved_rows) {   // the whole table goes up again (O(T), like the conversion that follows)
      PM_CUDA(e->raw_asks.ensure(std::max<uint32_t>(n_asks, 1)));
      if (n_asks)
        PM_CUDA(cudaMemcpyAsync(e->raw_asks.p, e->asks_h.data(), (size_t)n_asks * sizeof(pm_ask), cudaMemcpyHostToDevice, e->stream));
    } else {
      PM_CUDA(e->raw_asks.grow_keep(std::max<uint32_t>(n_asks, 1), std::min<size_t>(e->raw_asks.n, n_asks), e->stream));
    }
    if (n && !moved_rows) {
      PM_CUDA(e->scratch_idx.ensure(n)); PM_CUDA(e->upd_asks.ensure(n));
      PM_CUDA(cudaMemcpyAsync(e->scratch_idx.p, idx, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
      PM_CUDA(cudaMemcpyAsync(e->upd_asks.p, moved.data(), (size_t)n * sizeof(pm_ask), cudaMemcpyHostToDevice, e->stream));
      pm::pm_scatter_asks<<<blocks_for(n, 256), 256, 0, e->stream>>>(e->raw_asks.p, e->scratch_idx.p, e->upd_asks.p, n);
      PM_LAUNCH_CHECK("pm_scatter_asks");
    }
    e->raw_n_opts = (uint32_t)raw;
  }
  e->opt_rows = opt_rows;
  e->live_opts = live;
  uint32_t st = 0;
  {
    const int rc = convert_asks(e, n_asks, e->raw_n_opts, opt_rows, &st);   // (synchronises: `moved` and `add` are no longer read)
    if (rc != PM_OK) return rc;
  }
  if (st & (pm::kAskBadSizes | pm::kAskBadRange)) return e->fail(PM_E_INVALID, "ask table delta: rows out of bounds");
  e->n_asks = n_asks;
  std::vector<uint32_t> off;   // ask << 1 | 0, as pm_ask_toggle takes it
  for (uint32_t t = 0; t < n_asks; ++t)
    if (!e->ask_on[t]) off.push_back(t << 1);
  if (!off.empty()) {
    PM_CUDA(e->toggle_dev.ensure(off.size()));
    PM_CUDA(cudaMemcpyAsync(e->toggle_dev.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice, e->stream));
    pm::pm_ask_toggle<<<blocks_for(off.size(), 256), 256, 0, e->stream>>>(e->raw_asks.p, e->raw_opts.p, e->ask_newoff.p,
                                                                          e->toggle_dev.p, (uint32_t)off.size(), ask_tables(e), true);
    PM_LAUNCH_CHECK("pm_ask_toggle");
    PM_CUDA(cudaStreamSynchronize(e->stream));   // `off` is a local
  }
  recount_kinds(e);
  e->matched = e->local_done = false;
  return PM_OK;
}

}  // namespace

extern "C" {

void* pm_alloc_pinned(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void pm_free_pinned(void* p) {
  if (p) cudaFreeHost(p);
}

int pm_create(const pm_cfg* cfg, pm_engine** out) try {
  if (!cfg || !out) {
    g_create_error = "pm_create: null argument";
    return PM_E_INVALID;
  }
  *out = nullptr;
  if (cfg->abi_version != PM_ABI_VERSION) {
    g_create_error = "pm_create: ABI version mismatch";
    return PM_E_INVALID;
  }
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    g_create_error = "pm_create: no CUDA device visible (this engine has no CPU path)";
    return PM_E_NO_DEVICE;
  }
  if (cfg->device < 0 || cfg->device >= ndev) {
    g_create_error = "pm_create: device ordinal out of range";
    return PM_E_INVALID;
  }
  cudaDeviceProp prop{};
  // code built for sm_90a loads on compute capability 9.0 only
  if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
    cudaGetLastError();
    g_create_error = "pm_create: device is not sm_90 (kernels are built for sm_90a only)";
    return PM_E_NO_DEVICE;
  }
  pm_engine* e = new (std::nothrow) pm_engine;
  if (!e) return PM_E_NOMEM;
  e->cfg = *cfg;
  if (e->cfg.cost_tile_bytes == 0) e->cfg.cost_tile_bytes = 8ull << 30;
  e->device = cfg->device;
  e->sms = (unsigned)std::max(1, prop.multiProcessorCount);
  if (const char* t = std::getenv("PM_TUNE_GENERIC")) e->tune_generic = std::atoi(t);
  if (const char* t = std::getenv("PM_TUNE_BUILD")) e->tune_wide = std::atoi(t) == 8;
  if (const char* t = std::getenv("PM_TUNE_AUCTION")) e->tune_auction = std::atoi(t);
  if (const char* t = std::getenv("PM_TUNE_AUCTION_POOL")) std::sscanf(t, "%d,%d", &e->tune_auc_good, &e->tune_auc_extra);   // pool fill of a class walk
  if (const char* t = std::getenv("PM_TUNE_PROX")) e->tune_prox = std::atoi(t);   // 0: all-SM cooperative sweep; 2: single-CTA sweep
  if (const char* t = std::getenv("PM_TUNE_COMPRESS")) e->tune_compress = std::atoi(t);
  if (const char* t = std::getenv("PM_TUNE_INCR")) e->tune_incr = (uint32_t)std::strtoul(t, nullptr, 10);   // 0: always full
  bool ok = cudaSetDevice(e->device) == cudaSuccess;
  if (ok && cfg->stream) {
    e->stream = (cudaStream_t)cfg->stream;  // caller's stream (e.g. torch's current stream)
    e->own_stream = false;
  } else if (ok) {
    ok = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) == cudaSuccess;
  }
  ok = ok &&
            cudaEventCreate(&e->ev0) == cudaSuccess && cudaEventCreate(&e->ev1) == cudaSuccess &&
            e->h_scalars.ensure(64) == cudaSuccess && e->counters.ensure(32) == cudaSuccess;
  if (!ok) {
    g_create_error = std::string("pm_create: ") + cudaGetErrorString(cudaGetLastError());
    pm_destroy(e);
    return PM_E_CUDA;
  }
  *out = e;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

void pm_destroy(pm_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  e->wa.release(); e->wb.release(); e->lat.release(); e->lon.release(); e->addr_rank.release();
  e->asks.release(); e->opts.release(); e->opts_fast.release(); e->frows.release();
  e->raw_asks.release(); e->raw_opts.release(); e->upd_asks.release(); e->ask_counts.release(); e->ask_newoff.release(); e->amin.release(); e->amax.release(); e->bits.release();
  e->scratch_idx.release(); e->scratch_flags.release();
  e->upd_a.release(); e->upd_b.release(); e->upd_lat.release(); e->upd_lon.release();
  e->wa_alt.release(); e->wb_alt.release(); e->lat_alt.release(); e->lon_alt.release(); e->rank_alt.release();
  e->rep_alt.release(); e->nacc_alt.release(); e->first_alt.release(); e->owner_alt.release(); e->wsplice_dev.release();
  e->price_alt.release();
  e->cost.release(); e->first_ask.release(); e->ask_count.release(); e->ask_best.release();
  e->stripe_rank.release(); e->rank_best.release();
  e->feat_buf.release(); e->h_feat.release(); e->feat_w.release(); e->feat_a.release(); e->feat_o.release();
  e->sched_key.release(); e->sched_key_s.release(); e->sched_val.release(); e->sched_val_s.release();
  e->sched_ask.release(); e->sched_row.release();
  e->feat_key.release(); e->feat_key_s.release(); e->feat_val.release(); e->feat_perm.release();
  e->eval_first.release(); e->h_dirty.release(); e->dirty_dev.release(); e->incr_evals.release();
  e->walk_start.release(); e->toggle_dev.release(); e->splice_dev.release();
  e->keys.release(); e->keys_sorted.release(); e->iota.release(); e->order.release();
  e->hist.release(); e->seg_start.release(); e->ngroups.release(); e->group_base.release();
  e->base_len.release(); e->xhead.release(); e->xnext.release(); e->xcount.release();
  e->popped.release(); e->counters.release(); e->cub_tmp.release();
  e->prox_list.release(); e->prox_xs.release(); e->members_raw.release(); e->prox_dist.release();
  e->pg_part_d.release(); e->pg_part_i.release(); e->pg_cta_cnt.release(); e->pg_ctl.release();
  e->pg_clat.release(); e->pg_clon.release(); e->pg_ccos.release();
  e->nacc.release(); e->bits_wm.release();
  e->reputation.release(); e->ask_min_rep.release(); e->auc_rep_s.release(); e->auc_split_first.release(); e->auc_skip_key.release();
  e->dem_off.release(); e->dem_off_old.release(); e->slot_ask.release(); e->slot_cap.release(); e->slot_floor.release();
  e->auc_assigned_tmp.release(); e->cert_none.release(); e->dem_members.release(); e->dem_spos.release(); e->dem_aflag.release(); e->slot_row.release();
  e->price_cap.release(); e->auc_owner.release(); e->auc_assigned.release(); e->auc_withdrawn.release();
  e->auc_active.release(); e->auc_bid_w.release(); e->auc_winner.release(); e->auc_flag.release(); e->auc_gidx.release();
  e->auc_price.release(); e->auc_bid_p.release(); e->auc_bid_max.release();
  e->auc_theta.release(); e->auc_cand.release(); e->auc_theta_w.release();
  e->auc_walk_list.release(); e->auc_split_w.release(); e->auc_split_ticket.release(); e->auc_split_v.release();
  e->auc_pool.release(); e->auc_pool_bound_w.release(); e->auc_pool_bound_v.release(); e->auc_ckey.release(); e->auc_ckey_s.release();
  e->auc_class_of.release(); e->auc_class_rep.release(); e->auc_class_req.release(); e->auc_class_list.release();
  e->auc_retry.release(); e->auc_fallback.release(); e->auc_perm.release(); e->auc_pos_of.release();
  e->auc_idx.release(); e->auc_sorted.release(); e->auc_incl.release(); e->auc_hash.release();
  e->auc_hash_out.release(); e->auc_wa_s.release(); e->auc_wb_s.release(); e->auc_price_s.release(); e->auc_ctl.release();
  e->h_ctl.release();
  e->auc_raised.release(); e->auc_mark.release(); e->auc_cmin.release(); e->auc_chg.release();
  e->auc_rev_bidders.release(); e->auc_rev_offer_t.release(); e->auc_rev_win.release(); e->auc_rev_cap_s.release();
  e->auc_rev_cstart.release(); e->auc_rev_offer_p.release(); e->auc_rev_best.release(); e->auc_rev_pi_s.release();
  e->cert_min.release(); e->cert_acc.release(); e->cert_ok.release(); e->cert_own.release(); e->cert_bound.release();
  e->h_cert_acc.release(); e->h_cert_bound.release();
  e->rst_price.release(); e->rst_assigned.release(); e->rst_kept.release(); e->rst_owner.release(); e->rst_acc.release();
  e->h_rst_acc.release();
  e->worker_group.release(); e->worker_ask.release(); e->group_ask.release();
  e->group_off.release(); e->members.release(); e->h_scalars.release();
  e->xchg_send.release(); e->xchg_recv.release();
  e->r_worker_group.release(); e->r_worker_ask.release(); e->r_group_ask.release();
  e->r_group_off.release(); e->r_members.release(); e->r_ask_count.release(); e->r_ask_best.release();
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  for (cudaEvent_t ev : e->ev_pool) cudaEventDestroy(ev);
  if (e->stream && e->own_stream) cudaStreamDestroy(e->stream);
  delete e;
}

const char* pm_last_error(const pm_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int pm_set_asks(pm_engine* e, const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts,
                uint32_t n_opts) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  e->invalidate_eval();
  e->auc_discard();
  if ((n_asks && !asks) || (n_opts && !opts)) return e->fail(PM_E_INVALID, "pm_set_asks: null table");
  if (n_asks >= (1u << 30)) return e->fail(PM_E_INVALID, "pm_set_asks: too many asks");
  PM_CUDA(cudaSetDevice(e->device));
  // the caller's tables go up as they are; the device converts them (pm_ask_convert)
  PM_CUDA(e->raw_asks.ensure(n_asks)); PM_CUDA(e->raw_opts.ensure(n_opts));
  // asks may share or overlap option rows, so the converted table (one private range per ask) can be longer than
  // the caller's: size it by the sum of the per-ask counts
  uint64_t opt_rows = 0, live = 0;
  for (uint32_t i = 0; i < n_asks; ++i) {
    opt_rows += std::max<uint32_t>(asks[i].n_opts, 1u);   // an ask without options gets a neutral row
    live += asks[i].n_opts;
  }
  if (opt_rows >= (1ull << 31)) return e->fail(PM_E_INVALID, "pm_set_asks: too many option rows");
  if (n_asks) PM_CUDA(cudaMemcpyAsync(e->raw_asks.p, asks, (size_t)n_asks * sizeof(pm_ask), cudaMemcpyHostToDevice, e->stream));
  if (n_opts) PM_CUDA(cudaMemcpyAsync(e->raw_opts.p, opts, (size_t)n_opts * sizeof(pm_gpu_opt), cudaMemcpyHostToDevice, e->stream));
  e->have_asks = false;
  uint32_t st = 0;
  {
    const int rc = convert_asks(e, n_asks, n_opts, opt_rows, &st);   // also: the caller's tables are no longer read after return
    if (rc != PM_OK) return rc;
  }
  // NodeGroupConfiguration::is_valid, mod.rs:55-60 (the reference panics at construction)
  if (st & pm::kAskBadSizes)
    return e->fail(PM_E_INVALID, "pm_set_asks: max_group_size < min_group_size (Plugin configuration is invalid)");
  if (st & pm::kAskBadRange) return e->fail(PM_E_INVALID, "pm_set_asks: option range out of bounds");
  e->n_asks = n_asks;
  e->asks_h.assign(asks, asks + n_asks);
  e->raw_n_opts = n_opts;
  e->opt_rows = opt_rows;
  e->live_opts = live;
  // every ask enabled
  e->ask_on.assign(n_asks, 1);
  e->eval_on.assign(n_asks, 1);
  e->toggle_mark.assign(n_asks, 0);
  e->repl_mark.assign(n_asks, 0);
  e->orph_mark.assign(n_asks, 0);
  recount_kinds(e);
  e->have_caps = false;
  e->have_min_rep = false;
  e->demand.clear();
  e->dem_off_h.clear();
  e->auc_classes_valid = false;
  e->rows_auction = false;
  e->have_asks = true;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// Enabled configurations.  Only the asks whose state changes are converted again (pm_ask_toggle); the stored
// evaluation is kept, and the asks toggled since it are listed for the next incremental pass.
int pm_set_ask_enabled(pm_engine* e, const uint32_t* idx, const uint8_t* enabled, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks) return e->fail(PM_E_STATE, "pm_set_ask_enabled: no ask table");
  if (n == 0) return PM_OK;
  if (!idx || !enabled) return e->fail(PM_E_INVALID, "pm_set_ask_enabled: null");
  for (uint32_t i = 0; i < n; ++i)
    if (idx[i] >= e->n_asks) return e->fail(PM_E_INVALID, "pm_set_ask_enabled: ask index out of range");
  // the last entry for an ask decides its state
  std::vector<uint32_t> ord(n);
  for (uint32_t i = 0; i < n; ++i) ord[i] = i;
  std::stable_sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return idx[x] < idx[y]; });
  std::vector<uint32_t> changes;   // ask << 1 | enabled
  for (uint32_t j = 0; j < n; ++j) {
    if (j + 1 < n && idx[ord[j + 1]] == idx[ord[j]]) continue;
    const uint32_t t = idx[ord[j]];
    const uint8_t on = enabled[ord[j]] ? 1 : 0;
    if (on != e->ask_on[t]) changes.push_back(t << 1 | on);
  }
  if (changes.empty()) return PM_OK;
  ++e->table_version;
  {
    const int rc = use_ask_form(e, false);   // every row in one form: the toggled asks are converted in the reference one
    if (rc != PM_OK) return rc;
  }
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->toggle_dev.ensure(changes.size()));
  PM_CUDA(cudaMemcpyAsync(e->toggle_dev.p, changes.data(), changes.size() * 4, cudaMemcpyHostToDevice, e->stream));
  pm::pm_ask_toggle<<<blocks_for(changes.size(), 256), 256, 0, e->stream>>>(e->raw_asks.p, e->raw_opts.p, e->ask_newoff.p,
                                                                            e->toggle_dev.p, (uint32_t)changes.size(), ask_tables(e),
                                                                            true);
  PM_LAUNCH_CHECK("pm_ask_toggle");
  PM_CUDA(cudaStreamSynchronize(e->stream));   // `changes` is a local
  for (uint32_t v : changes) {
    const uint32_t t = v >> 1;
    const bool on = (v & 1u) != 0;
    e->ask_on[t] = on ? 1 : 0;
    e->n_off += on ? (uint32_t)-1 : 1u;
    e->count_kind(t, on ? +1 : -1);
    if (e->eval_valid && !e->toggle_mark[t]) {
      e->toggle_mark[t] = 1;
      e->toggled.push_back(t);
    }
    if (e->auc_state && !e->auc_ask_mark[t]) {
      e->auc_ask_mark[t] = 1;
      e->auc_toggled.push_back(t);
    }
  }
  e->rows_bound = false;           // the FastRows were converted again: pm_bind_rows binds them anew
  e->auc_classes_valid = false;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// Ask-table deltas.  Every call checks everything on the host first (a refusal changes nothing), then edit the raw rows
// and convert the whole table again (commit_asks).  The stored evaluation and the stored auction state are kept: the
// changed asks are listed for the next incremental pass (E / D) and the next warm pass (A0).  A failure after the
// checks (a CUDA error) leaves tables that are not trusted: the ask table is dropped, as a failed pm_set_asks does.
static int ask_delta_failed(pm_engine* e, int rc) {
  if (rc != PM_OK) {
    e->have_asks = false;
    e->invalidate_eval();
    e->auc_discard();
  }
  return rc;
}
// The part of a delta after its checks: any failure in it, a CUDA error or a host exception (an allocation the table
// size makes fail), leaves host bookkeeping and device tables that may disagree, so the ask table is dropped
extern "C++" {   // a template: C++ linkage inside the C block
template <class Body> static int ask_delta(pm_engine* e, Body&& body) {
  int rc;
  try {
    rc = body();
  } catch (...) {
    rc = pm_guard_rc();
    e->err = "ask table delta: host exception (the ask table was dropped)";
  }
  return ask_delta_failed(e, rc);
}
}

// The demands' offsets to the device; demands that are all 1 are dropped (the auction runs on the asks themselves).
static int upload_demand(pm_engine* e) {
  if (std::all_of(e->demand.begin(), e->demand.end(), [](uint32_t d) { return d == 1u; })) {
    e->demand.clear();
    e->dem_off_h.clear();
    return PM_OK;
  }
  PM_CUDA(e->dem_off.ensure(e->dem_off_h.size()));
  PM_CUDA(cudaMemcpyAsync(e->dem_off.p, e->dem_off_h.data(), e->dem_off_h.size() * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));   // dem_off_h may be reallocated by the next call
  return PM_OK;
}

int pm_update_asks(pm_engine* e, const uint32_t* idx, const pm_ask* asks, uint32_t n, const pm_gpu_opt* opts,
                   uint32_t n_opts) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks) return e->fail(PM_E_STATE, "pm_update_asks: no ask table");
  if ((n && (!idx || !asks)) || (n_opts && !opts)) return e->fail(PM_E_INVALID, "pm_update_asks: null");
  std::vector<uint32_t> uidx;
  std::vector<pm_ask> urows;
  {
    std::string err;
    const int rc = check_ask_rows(e, "pm_update_asks", idx, asks, n, n_opts, &uidx, &urows, &err);
    if (rc != PM_OK) return e->fail((pm_status)rc, err);
  }
  if (n == 0) return PM_OK;
  ++e->table_version;
  return ask_delta(e, [&]() -> int {
    PM_CUDA(cudaSetDevice(e->device));
    for (uint32_t t : uidx) {   // a replaced row counts as disabled and enabled again (split_toggles)
      if (e->eval_valid) e->repl_mark[t] = 1;
      e->mark_toggled(t);
      e->auc_mark_ask(t);
    }
    return commit_asks(e, e->n_asks, uidx.data(), urows.data(), (uint32_t)uidx.size(), opts);
  });
} catch (...) { return pm_guard_rc(); }

// The part of pm_resize_asks / pm_remove_asks / pm_insert_asks after their checks.  The stored evaluation's first asks
// and the stored auction state are remapped on the device and every per-ask host copy moves with its rows; then the
// rows are committed.  Removed rows take their enabled flag, cap, floor and demand with them; inserted rows are enabled,
// with cap 0, floor 0 and demand 1, in E (eval_on 0) and in A0, holding nothing; kept rows keep every mark.
static int splice_asks(pm_engine* e, const AskSplice& sp, const pm_ask* rows, const pm_gpu_opt* opts) {
  PM_CUDA(cudaSetDevice(e->device));
  const uint32_t n_old = sp.n_old, n_new = sp.n_new, nr = (uint32_t)sp.removed.size(), ni = (uint32_t)sp.before.size();
  const bool moves = nr || (ni && sp.before[0] < n_old);   // some kept row changes its index, or a row goes
  PM_CUDA(e->splice_dev.ensure(std::max<size_t>((size_t)nr + ni + n_old, 1)));
  uint32_t* rm_dev = e->splice_dev.p;
  uint32_t* bf_dev = rm_dev + nr;
  uint32_t* map_dev = bf_dev + ni;
  if (nr) PM_CUDA(cudaMemcpyAsync(rm_dev, sp.removed.data(), (size_t)nr * 4, cudaMemcpyHostToDevice, e->stream));
  if (ni) PM_CUDA(cudaMemcpyAsync(bf_dev, sp.before.data(), (size_t)ni * 4, cudaMemcpyHostToDevice, e->stream));
  // the stored evaluation: the workers of a removed ask land on its next kept row, which lists them as orphans
  std::vector<uint32_t> orphans_at;
  if (e->eval_valid) {
    for (uint32_t r = 0; r < nr; ++r) {
      const uint32_t t = sp.removed[r];
      if ((e->eval_on[t] || e->orph_mark[t]) && sp.succ[r] < n_new) orphans_at.push_back(sp.succ[r]);
    }
    uint32_t w0 = 0, nw = 0;
    e->shard(&w0, &nw);
    nw = w0 < e->n_workers ? std::min(nw, e->n_workers - w0) : 0u;
    if (moves && nw) {
      pm::pm_splice_first_asks<<<std::min(blocks_for(nw, 256), 8u * e->sms), 256, 0, e->stream>>>(e->eval_first.p, w0, nw, rm_dev, nr,
                                                                                                  bf_dev, ni, n_new);
      PM_LAUNCH_CHECK("pm_splice_first_asks");
    }
  }
  sp.apply(&e->ask_on, (uint8_t)1);
  sp.apply(&e->eval_on, (uint8_t)0);
  sp.apply(&e->toggle_mark, (uint8_t)0);
  sp.apply(&e->repl_mark, (uint8_t)0);
  sp.apply(&e->orph_mark, (uint8_t)0);
  sp.apply_list(&e->toggled);
  for (uint32_t s : sp.at) e->mark_toggled(s);
  for (uint32_t s : orphans_at) {
    e->orph_mark[s] = 1;
    e->mark_toggled(s);
  }
  // demands move with their rows (all 1 again: dropped, as pm_set_ask_demand drops them)
  const uint32_t old_slots = e->n_slots();
  const bool had_demand = !e->demand.empty();
  if (had_demand) {
    if (e->auc_state) {
      PM_CUDA(e->dem_off_old.ensure((size_t)n_old + 1));
      PM_CUDA(cudaMemcpyAsync(e->dem_off_old.p, e->dem_off_h.data(), ((size_t)n_old + 1) * 4, cudaMemcpyHostToDevice, e->stream));
      PM_CUDA(cudaStreamSynchronize(e->stream));   // dem_off_h is rebuilt below
    }
    sp.apply(&e->demand, 1u);
    e->dem_off_h.assign((size_t)n_new + 1, 0u);
    for (uint32_t t = 0; t < n_new; ++t) e->dem_off_h[t + 1] = e->dem_off_h[t] + e->demand[t];
    const int rc = upload_demand(e);
    if (rc != PM_OK) return rc;
  }
  // the stored auction state: each kept slot's hold moves to its row's new slots; a removed slot's kept row becomes
  // unowned at its stored price and counts against the cutoff; inserted slots hold nothing
  if (e->auc_state) {
    const uint32_t D_new = e->demand.empty() ? n_new : e->dem_off_h[n_new];
    PM_CUDA(e->auc_assigned_tmp.ensure(std::max<uint32_t>(D_new, 1)));
    PM_CUDA(cudaMemsetAsync(e->auc_assigned_tmp.p, 0xFF, (size_t)std::max<uint32_t>(D_new, 1) * 4, e->stream));
    PM_CUDA(cudaMemsetAsync(e->counters.p + 17, 0, 4, e->stream));
    if (old_slots) {
      if (n_old) PM_CUDA(cudaMemcpyAsync(map_dev, sp.map.data(), (size_t)n_old * 4, cudaMemcpyHostToDevice, e->stream));
      pm::pm_auction_slot_remap<<<std::min(blocks_for(old_slots, 256), 8u * e->sms), 256, 0, e->stream>>>(
          had_demand ? e->dem_off_old.p : nullptr, e->demand.empty() ? nullptr : e->dem_off.p, map_dev, n_old, old_slots,
          e->auc_assigned.p, e->auc_assigned_tmp.p, e->auc_owner.p, e->auc_kept, e->counters.p + 17);
      PM_LAUNCH_CHECK("pm_auction_slot_remap");
    }
    PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 17, e->counters.p + 17, 4, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));   // (the map is a host vector the caller owns)
    std::swap(e->auc_assigned, e->auc_assigned_tmp);
    e->auc_removed_held += e->h_scalars.p[17];
    sp.apply(&e->auc_ask_mark, (uint8_t)0);
    sp.apply(&e->auc_cap_stored, 0u);
    sp.apply(&e->auc_floor_stored, 0u);
    sp.apply(&e->auc_dem_kept, 0u);
    sp.apply_list(&e->auc_toggled);
    for (uint32_t s : sp.at) e->auc_mark_ask(s);
    e->auc_asks_resized = true;
  }
  if (e->have_caps) {
    sp.apply(&e->cap_host, 0u);
    PM_CUDA(e->price_cap.ensure(std::max<uint32_t>(n_new, 1)));
    if (n_new) PM_CUDA(cudaMemcpyAsync(e->price_cap.p, e->cap_host.data(), (size_t)n_new * 4, cudaMemcpyHostToDevice, e->stream));
  }
  if (e->have_min_rep) {
    sp.apply(&e->floor_host, 0u);
    PM_CUDA(e->ask_min_rep.ensure(std::max<uint32_t>(n_new, 1)));
    if (n_new) PM_CUDA(cudaMemcpyAsync(e->ask_min_rep.p, e->floor_host.data(), (size_t)n_new * 4, cudaMemcpyHostToDevice, e->stream));
  }
  return commit_asks(e, n_new, sp.at.data(), rows, ni, opts, &sp);   // (synchronises before the host copies change again)
}

// The checks of pm_remove_asks, on the host before anything changes: the distinct indices, increasing
static int check_remove(const pm_engine* e, const uint32_t* idx, uint32_t n, std::vector<uint32_t>* removed, std::string* err) {
  if (n && !idx) { *err = "pm_remove_asks: null"; return PM_E_INVALID; }
  removed->assign(idx, idx + n);
  for (uint32_t t : *removed)
    if (t >= e->n_asks) { *err = "pm_remove_asks: ask index out of range"; return PM_E_INVALID; }
  std::sort(removed->begin(), removed->end());
  removed->erase(std::unique(removed->begin(), removed->end()), removed->end());
  return PM_OK;
}

// The checks of pm_insert_asks and of pm_resize_asks' growth (before: every row at n_asks): the positions, the rows and
// their option ranges (check_ask_rows), the ask count and the slot total
static int check_insert(const pm_engine* e, const char* fn, const uint32_t* before, const pm_ask* asks, uint32_t n,
                        const pm_gpu_opt* opts, uint32_t n_opts, std::string* err) {
  if ((n && (!before || !asks)) || (n_opts && !opts)) { *err = std::string(fn) + ": null"; return PM_E_INVALID; }
  for (uint32_t i = 0; i < n; ++i)
    if (before[i] > e->n_asks || (i && before[i] < before[i - 1])) {
      *err = std::string(fn) + ": before[] decreases or exceeds n_asks";
      return PM_E_INVALID;
    }
  if ((uint64_t)e->n_asks + n >= (1u << 30)) { *err = std::string(fn) + ": too many asks"; return PM_E_INVALID; }
  std::vector<uint32_t> uidx;
  std::vector<pm_ask> urows;
  const int rc = check_ask_rows(e, fn, nullptr, asks, n, n_opts, &uidx, &urows, err);
  if (rc != PM_OK) return rc;
  // inserted asks take one slot each; the slots stay below the ask-count limit
  if ((uint64_t)e->n_slots() + n >= (1u << 30)) { *err = std::string(fn) + ": the ask demands' total reaches 2^30"; return PM_E_INVALID; }
  return PM_OK;
}

int pm_resize_asks(pm_engine* e, uint32_t n_asks, const pm_ask* added, const pm_gpu_opt* opts, uint32_t n_opts) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks) return e->fail(PM_E_STATE, "pm_resize_asks: no ask table");
  if (n_asks >= (1u << 30)) return e->fail(PM_E_INVALID, "pm_resize_asks: too many asks");
  const uint32_t old = e->n_asks;
  const uint32_t n_add = n_asks > old ? n_asks - old : 0u;
  // the tail case of pm_remove_asks / pm_insert_asks: drop [n_asks, old), or insert every added row at the end
  std::vector<uint32_t> removed, before(n_add, old);
  {
    std::string err;
    const int rc = check_insert(e, "pm_resize_asks", before.data(), added, n_add, opts, n_opts, &err);
    if (rc != PM_OK) return e->fail((pm_status)rc, err);
  }
  if (n_asks == old) return PM_OK;
  for (uint32_t t = n_asks; t < old; ++t) removed.push_back(t);
  ++e->table_version;
  return ask_delta(e, [&]() -> int {
    const AskSplice sp(old, std::move(removed), std::move(before));
    return splice_asks(e, sp, added, opts);
  });
} catch (...) { return pm_guard_rc(); }

int pm_remove_asks(pm_engine* e, const uint32_t* idx, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks) return e->fail(PM_E_STATE, "pm_remove_asks: no ask table");
  std::vector<uint32_t> removed;
  {
    std::string err;
    const int rc = check_remove(e, idx, n, &removed, &err);
    if (rc != PM_OK) return e->fail((pm_status)rc, err);
  }
  if (removed.empty()) return PM_OK;
  ++e->table_version;
  return ask_delta(e, [&]() -> int {
    const AskSplice sp(e->n_asks, std::move(removed), {});
    return splice_asks(e, sp, nullptr, nullptr);
  });
} catch (...) { return pm_guard_rc(); }

int pm_insert_asks(pm_engine* e, const uint32_t* before, const pm_ask* asks, uint32_t n, const pm_gpu_opt* opts,
                   uint32_t n_opts) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks) return e->fail(PM_E_STATE, "pm_insert_asks: no ask table");
  {
    std::string err;
    const int rc = check_insert(e, "pm_insert_asks", before, asks, n, opts, n_opts, &err);
    if (rc != PM_OK) return e->fail((pm_status)rc, err);
  }
  if (n == 0) return PM_OK;
  ++e->table_version;
  return ask_delta(e, [&]() -> int {
    const AskSplice sp(e->n_asks, {}, std::vector<uint32_t>(before, before + n));
    return splice_asks(e, sp, asks, opts);
  });
} catch (...) { return pm_guard_rc(); }

int pm_set_model_table(pm_engine* e, const uint32_t* bits, uint32_t n_patterns, uint32_t n_models,
                       uint32_t words) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  e->invalidate_eval();
  e->auc_discard();
  if (words == 0) words = 1;
  if (n_patterns && !bits) return e->fail(PM_E_INVALID, "pm_set_model_table: null table");
  if ((uint64_t)words * 32 < n_models) return e->fail(PM_E_INVALID, "pm_set_model_table: words too small");
  // device layout: 31 models per word (bit 31 stays clear: the fast predicate turns "non-zero" into a sign bit by
  // an addition, pm_device.cuh DevOptF), row 0 = no model clause = accepts everything
  const uint32_t dwords = std::max<uint32_t>((n_models + pm::kModelsPerWord - 1) / pm::kModelsPerWord, 1u);
  std::vector<uint32_t> tbl((size_t)(n_patterns + 1) * dwords, 0u);
  for (uint32_t i = 0; i < dwords; ++i) tbl[i] = 0x7FFFFFFFu;
  for (uint32_t p = 0; p < n_patterns; ++p) {
    const uint32_t* src = bits + (size_t)p * words;
    uint32_t* dst = tbl.data() + (size_t)(p + 1) * dwords;
    for (uint32_t wi = 0; wi < words; ++wi) {
      uint32_t v = src[wi];
      while (v) {
        const uint32_t m = wi * 32u + (uint32_t)__builtin_ctz(v);
        v &= v - 1;
        if (m < n_models) dst[m / pm::kModelsPerWord] |= 1u << (m % pm::kModelsPerWord);
      }
    }
  }
  words = dwords;
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->bits.ensure(tbl.size()));
  PM_CUDA(cudaMemcpyAsync(e->bits.p, tbl.data(), tbl.size() * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  e->n_patterns = n_patterns;
  e->n_models = n_models;
  e->words = words;
  e->have_bits = true;
  e->rows_bound = false;
  e->nacc_valid = false;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_set_worker_count(pm_engine* e, uint32_t n_workers) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  e->invalidate_eval();
  e->auc_discard();
  PM_CUDA(cudaSetDevice(e->device));
  // a full reload replaces the table: the second buffers of the worker splices go until the next splice needs them
  e->wa_alt.release(); e->wb_alt.release(); e->lat_alt.release(); e->lon_alt.release(); e->rank_alt.release();
  e->rep_alt.release(); e->nacc_alt.release(); e->first_alt.release(); e->owner_alt.release(); e->price_alt.release();
  if (n_workers > e->wa.n || !e->wa.p) {
    // grow, preserving nothing: callers upsert after (re)sizing
    PM_CUDA(e->wa.ensure(n_workers));
    PM_CUDA(e->wb.ensure(n_workers));
  }
  PM_CUDA(cudaMemsetAsync(e->wa.p, 0, (size_t)std::max<uint32_t>(n_workers, 1) * 16, e->stream));
  PM_CUDA(cudaMemsetAsync(e->wb.p, 0, (size_t)std::max<uint32_t>(n_workers, 1) * 16, e->stream));
  e->n_workers = n_workers;
  e->workers_checked = false;
  e->nacc_valid = false;
  e->have_workers = true;
  e->have_loc = e->have_rank = false;
  e->have_rep = false;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_upsert_workers(pm_engine* e, const pm_worker_a* a, const pm_worker_b* b, uint32_t first,
                      uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_upsert_workers: call pm_set_worker_count first");
  if ((uint64_t)first + n > e->n_workers) return e->fail(PM_E_INVALID, "pm_upsert_workers: range out of bounds");
  if (n && (!a || !b)) return e->fail(PM_E_INVALID, "pm_upsert_workers: null plane");
  e->mark_range_dirty(first, n);
  e->auc_mark_rows(first, n);
  PM_CUDA(cudaSetDevice(e->device));
  if (n) {
    PM_CUDA(cudaMemcpyAsync(e->wa.p + first, a, (size_t)n * 16, cudaMemcpyHostToDevice, e->stream));
    PM_CUDA(cudaMemcpyAsync(e->wb.p + first, b, (size_t)n * 16, cudaMemcpyHostToDevice, e->stream));
  }
  e->workers_checked = false;
  e->nacc_valid = false;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_set_worker_locations(pm_engine* e, const double* lat, const double* lon, uint32_t first,
                            uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_set_worker_locations: no worker table");
  if ((uint64_t)first + n > e->n_workers) return e->fail(PM_E_INVALID, "pm_set_worker_locations: range");
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->lat.ensure(e->n_workers));
  PM_CUDA(e->lon.ensure(e->n_workers));
  if (n) {
    PM_CUDA(cudaMemcpyAsync(e->lat.p + first, lat, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
    PM_CUDA(cudaMemcpyAsync(e->lon.p + first, lon, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  }
  e->have_loc = true;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_set_worker_addr_rank(pm_engine* e, const uint32_t* rank, uint32_t first, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_set_worker_addr_rank: no worker table");
  if ((uint64_t)first + n > e->n_workers) return e->fail(PM_E_INVALID, "pm_set_worker_addr_rank: range");
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->addr_rank.ensure(e->n_workers));
  if (n) PM_CUDA(cudaMemcpyAsync(e->addr_rank.p + first, rank, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  e->have_rank = true;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_set_flags(pm_engine* e, const uint32_t* idx, const uint32_t* flags, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_set_flags: no worker table");
  if (n == 0) return PM_OK;
  if (!idx || !flags) return e->fail(PM_E_INVALID, "pm_set_flags: null");
  for (uint32_t i = 0; i < n; ++i) {   // out-of-range indices are skipped, as the scatter does
    e->mark_dirty(idx[i]);
    e->auc_mark_row(idx[i]);
  }
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->scratch_idx.ensure(n));
  PM_CUDA(e->scratch_flags.ensure(n));
  PM_CUDA(cudaMemcpyAsync(e->scratch_idx.p, idx, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->scratch_flags.p, flags, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  pm::pm_scatter_flags<<<blocks_for(n, 256), 256, 0, e->stream>>>(e->wa.p, e->scratch_idx.p, e->scratch_flags.p, n, e->n_workers);
  PM_LAUNCH_CHECK("pm_scatter_flags");
  e->workers_checked = false;
  e->nacc_valid = false;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// Resident tables with deltas (the management pass of a long-running host: only rows that changed travel).
int pm_resize_workers(pm_engine* e, uint32_t n_workers) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  PM_CUDA(cudaSetDevice(e->device));
  const size_t keep = e->have_workers ? e->n_workers : 0;
  uint32_t a0 = 0, na = 0;   // the range before the resize
  e->shard(&a0, &na);
  if (e->eval_valid) {
    // the stored evaluation follows the table: kept rows keep their entries, rows past the old end are NONE and dirty
    PM_CUDA(e->eval_first.grow_keep(std::max<uint32_t>(n_workers, 1), keep, e->stream));
    if (n_workers > keep)
      PM_CUDA(cudaMemsetAsync(e->eval_first.p + keep, 0xFF, (size_t)(n_workers - keep) * 4, e->stream));
    if (n_workers < keep) {
      size_t j = 0;
      for (uint32_t i : e->dirty_rows) {
        if (i < n_workers) e->dirty_rows[j++] = i;
        else e->dirty_mark[i] = 0;
      }
      e->dirty_rows.resize(j);
    }
    e->dirty_mark.resize(n_workers, 0);
  }
  PM_CUDA(e->wa.grow_keep(std::max<uint32_t>(n_workers, 1), keep, e->stream));
  PM_CUDA(e->wb.grow_keep(std::max<uint32_t>(n_workers, 1), keep, e->stream));
  if (e->have_loc) {
    PM_CUDA(e->lat.grow_keep(std::max<uint32_t>(n_workers, 1), keep, e->stream));
    PM_CUDA(e->lon.grow_keep(std::max<uint32_t>(n_workers, 1), keep, e->stream));
  }
  if (e->have_rank) PM_CUDA(e->addr_rank.grow_keep(std::max<uint32_t>(n_workers, 1), keep, e->stream));
  if (e->have_rep) PM_CUDA(e->reputation.grow_keep(std::max<uint32_t>(n_workers, 1), keep, e->stream));
  if (n_workers > keep) {   // rows that were beyond the old table (or were cut off earlier) start empty
    PM_CUDA(cudaMemsetAsync(e->wa.p + keep, 0, (size_t)(n_workers - keep) * 16, e->stream));
    PM_CUDA(cudaMemsetAsync(e->wb.p + keep, 0, (size_t)(n_workers - keep) * 16, e->stream));
    if (e->have_loc) {
      PM_CUDA(cudaMemsetAsync(e->lat.p + keep, 0, (size_t)(n_workers - keep) * 8, e->stream));
      PM_CUDA(cudaMemsetAsync(e->lon.p + keep, 0, (size_t)(n_workers - keep) * 8, e->stream));
    }
    if (e->have_rank) PM_CUDA(cudaMemsetAsync(e->addr_rank.p + keep, 0, (size_t)(n_workers - keep) * 4, e->stream));
    if (e->have_rep) PM_CUDA(cudaMemsetAsync(e->reputation.p + keep, 0, (size_t)(n_workers - keep) * 4, e->stream));
  }
  e->n_workers = n_workers;
  if (e->auc_state && n_workers < e->auc_kept) {   // rows from the new end on count as changed from here on, as a range
    e->auc_kept = n_workers;
    size_t j = 0;
    for (uint32_t i : e->auc_rows) {
      if (i < n_workers) e->auc_rows[j++] = i;
      else e->auc_row_mark[i] = 0;
    }
    e->auc_rows.resize(j);
  }
  if (e->eval_valid) {
    // A communicator's equal share, or an open-ended pm_set_shard range, moves with W.  Rows that leave the range
    // return to NONE; rows that enter it were evaluated by another rank, or never: they are written.  Each is at most
    // two intervals.  The rows past the old end are written for the preludes wherever they lie.
    uint32_t b0 = 0, nb = 0;
    e->shard(&b0, &nb);
    const uint64_t a1 = std::min<uint64_t>((uint64_t)a0 + na, n_workers), b1 = (uint64_t)b0 + nb;
    auto none = [&](uint64_t lo, uint64_t hi) -> cudaError_t {
      return hi > lo ? cudaMemsetAsync(e->eval_first.p + lo, 0xFF, (size_t)(hi - lo) * 4, e->stream) : cudaSuccess;
    };
    PM_CUDA(none(a0, std::min<uint64_t>(a1, b0)));
    PM_CUDA(none(std::max<uint64_t>(a0, b1), a1));
    e->dirty_in = 0;
    for (uint32_t i : e->dirty_rows) e->dirty_in += e->in_range(i);
    if (e->dirty_in > e->tune_incr) e->mark_all_dirty();
    auto enter = [&](uint64_t lo, uint64_t hi) {
      if (hi > lo) e->mark_range_dirty((uint32_t)lo, (uint32_t)(hi - lo));
    };
    enter(b0, std::min<uint64_t>(b1, a0));
    enter(std::max<uint64_t>(b0, (uint64_t)a0 + na), b1);
    if (n_workers > keep) e->mark_range_dirty((uint32_t)keep, n_workers - (uint32_t)keep);
  }
  e->have_workers = true;
  e->workers_checked = false;
  e->nacc_valid = false;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_update_workers(pm_engine* e, const uint32_t* idx, const pm_worker_a* a, const pm_worker_b* b, const double* lat,
                      const double* lon, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_update_workers: no worker table");
  if (n == 0) return PM_OK;
  if (!idx || !a || !b || ((lat == nullptr) != (lon == nullptr))) return e->fail(PM_E_INVALID, "pm_update_workers: null");
  ++e->table_version;
  for (uint32_t i = 0; i < n; ++i) {   // out-of-range indices are skipped, as the scatter does
    e->mark_dirty(idx[i]);
    e->auc_mark_row(idx[i]);
  }
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->scratch_idx.ensure(n)); PM_CUDA(e->upd_a.ensure(n)); PM_CUDA(e->upd_b.ensure(n));
  PM_CUDA(cudaMemcpyAsync(e->scratch_idx.p, idx, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->upd_a.p, a, (size_t)n * 16, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->upd_b.p, b, (size_t)n * 16, cudaMemcpyHostToDevice, e->stream));
  if (lat) {
    if (!e->have_loc) {
      PM_CUDA(e->lat.ensure(e->wa.n)); PM_CUDA(e->lon.ensure(e->wa.n));
      PM_CUDA(cudaMemsetAsync(e->lat.p, 0, e->wa.n * 8, e->stream));
      PM_CUDA(cudaMemsetAsync(e->lon.p, 0, e->wa.n * 8, e->stream));
      e->have_loc = true;
    }
    PM_CUDA(e->upd_lat.ensure(n)); PM_CUDA(e->upd_lon.ensure(n));
    PM_CUDA(cudaMemcpyAsync(e->upd_lat.p, lat, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
    PM_CUDA(cudaMemcpyAsync(e->upd_lon.p, lon, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  }
  pm::pm_scatter_rows<<<blocks_for(n, 256), 256, 0, e->stream>>>(e->wa.p, e->wb.p, lat ? e->lat.p : nullptr, lat ? e->lon.p : nullptr,
                                                                 e->scratch_idx.p, e->upd_a.p, e->upd_b.p, e->upd_lat.p, e->upd_lon.p, n,
                                                                 e->n_workers);
  PM_LAUNCH_CHECK("pm_scatter_rows");
  e->workers_checked = false;
  e->nacc_valid = false;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// Rows removed from and inserted into the worker table (pm_remove_workers, pm_insert_workers).  removed: old rows,
// increasing and distinct; before: per inserted row the old row it goes before, non-decreasing.  There is no W-entry
// map: a row's new index is two binary searches away (pm_kernels.cuh WorkerSplice), here for the host's marked rows.
struct WorkerSpliceH {
  uint32_t n_old = 0, n_new = 0;
  std::vector<uint32_t> removed, before;
  WorkerSpliceH(uint32_t n, std::vector<uint32_t> rm, std::vector<uint32_t> bf)
      : n_old(n), n_new(n - (uint32_t)rm.size() + (uint32_t)bf.size()), removed(std::move(rm)), before(std::move(bf)) {}
  uint32_t rm_below(uint32_t x) const { return (uint32_t)(std::lower_bound(removed.begin(), removed.end(), x) - removed.begin()); }
  bool is_removed(uint32_t i) const { return std::binary_search(removed.begin(), removed.end(), i); }
  // the new index of kept old row i
  uint32_t map(uint32_t i) const {
    return i - rm_below(i) + (uint32_t)(std::upper_bound(before.begin(), before.end(), i) - before.begin());
  }
  // the new index of inserted row k
  uint32_t at(uint32_t k) const { return before[k] - rm_below(before[k]) + k; }
  // the new index of the boundary in front of old row x, ahead of the rows inserted before x: the new rows below it are
  // the kept rows below x and the rows inserted before a position < x
  uint32_t edge(uint32_t x) const {
    return x - rm_below(x) + (uint32_t)(std::lower_bound(before.begin(), before.end(), x) - before.begin());
  }
  // a list of rows renamed, the removed ones dropped (and their marks cleared)
  void apply_list(std::vector<uint32_t>* list, std::vector<uint8_t>* mark) const {
    size_t k = 0;
    for (uint32_t i : *list) {
      (*mark)[i] = 0;
      if (!is_removed(i)) (*list)[k++] = map(i);
    }
    list->resize(k);
  }
};

// The checks of pm_remove_workers, on the host before anything changes: the distinct indices, increasing
static int check_remove_workers(const pm_engine* e, const uint32_t* idx, uint32_t n, std::vector<uint32_t>* removed, std::string* err) {
  if (n && !idx) { *err = "pm_remove_workers: null"; return PM_E_INVALID; }
  removed->assign(idx, idx + n);
  for (uint32_t i : *removed)
    if (i >= e->n_workers) { *err = "pm_remove_workers: worker index out of range"; return PM_E_INVALID; }
  std::sort(removed->begin(), removed->end());
  removed->erase(std::unique(removed->begin(), removed->end()), removed->end());
  return PM_OK;
}

// The checks of pm_insert_workers: the pointers, the positions and the table size (it stays below PM_NONE rows)
static int check_insert_workers(const pm_engine* e, const uint32_t* before, const pm_worker_a* a, const pm_worker_b* b,
                                const double* lat, const double* lon, uint32_t n, std::string* err) {
  if ((n && (!before || !a || !b)) || ((lat == nullptr) != (lon == nullptr))) { *err = "pm_insert_workers: null"; return PM_E_INVALID; }
  if ((uint64_t)e->n_workers + n >= PM_NONE) { *err = "pm_insert_workers: the table would reach PM_NONE rows"; return PM_E_INVALID; }
  for (uint32_t i = 0; i < n; ++i)
    if (before[i] > e->n_workers || (i && before[i] < before[i - 1])) {
      *err = "pm_insert_workers: before[] decreases or exceeds n_workers";
      return PM_E_INVALID;
    }
  return PM_OK;
}

// The part of pm_remove_workers / pm_insert_workers after their checks.  One launch of pm_splice_workers moves every
// per-row column into its second buffer (the planes, location, address rank, reputation, the worker-major acceptance
// words while they hold, the stored first ask, the stored auction price and owner), the buffers are swapped, and one
// launch of pm_splice_worker_holds renames the stored assignment in place.  The host marks (dirty_rows, auc_rows) move
// with their rows.  Nothing else outlives a pass keyed by worker index: the cost tile's held-sentinel maps describe
// the tile buffer's contents, whatever rows they came from, and the auction's class caches, pools and sorted worker
// copy are rebuilt by every pass.
static int splice_workers(pm_engine* e, const WorkerSpliceH& sp, const pm_worker_a* a, const pm_worker_b* b,
                          const double* lat, const double* lon) {
  PM_CUDA(cudaSetDevice(e->device));
  const uint32_t n_old = sp.n_old, n_new = sp.n_new, nr = (uint32_t)sp.removed.size(), ni = (uint32_t)sp.before.size();
  uint32_t a0 = 0, na = 0;   // the range before the splice
  e->shard(&a0, &na);
  const uint32_t a1 = (uint32_t)std::min<uint64_t>((uint64_t)a0 + na, n_old);
  PM_CUDA(e->wsplice_dev.ensure(std::max<size_t>((size_t)nr + ni, 1)));
  const uint32_t* rm_dev = e->wsplice_dev.p;
  const uint32_t* bf_dev = e->wsplice_dev.p + nr;
  if (nr) PM_CUDA(cudaMemcpyAsync(e->wsplice_dev.p, sp.removed.data(), (size_t)nr * 4, cudaMemcpyHostToDevice, e->stream));
  if (ni) {
    PM_CUDA(cudaMemcpyAsync(e->wsplice_dev.p + nr, sp.before.data(), (size_t)ni * 4, cudaMemcpyHostToDevice, e->stream));
    PM_CUDA(e->upd_a.ensure(ni)); PM_CUDA(e->upd_b.ensure(ni));
    PM_CUDA(cudaMemcpyAsync(e->upd_a.p, a, (size_t)ni * 16, cudaMemcpyHostToDevice, e->stream));
    PM_CUDA(cudaMemcpyAsync(e->upd_b.p, b, (size_t)ni * 16, cudaMemcpyHostToDevice, e->stream));
    if (lat) {
      PM_CUDA(e->upd_lat.ensure(ni)); PM_CUDA(e->upd_lon.ensure(ni));
      PM_CUDA(cudaMemcpyAsync(e->upd_lat.p, lat, (size_t)ni * 8, cudaMemcpyHostToDevice, e->stream));
      PM_CUDA(cudaMemcpyAsync(e->upd_lon.p, lon, (size_t)ni * 8, cudaMemcpyHostToDevice, e->stream));
    }
  }
  if (lat && ni && !e->have_loc) {   // the first coordinates: every other row at (0, 0), as pm_update_workers does
    PM_CUDA(e->lat.ensure(e->wa.n)); PM_CUDA(e->lon.ensure(e->wa.n));
    PM_CUDA(cudaMemsetAsync(e->lat.p, 0, e->wa.n * 8, e->stream));
    PM_CUDA(cudaMemsetAsync(e->lon.p, 0, e->wa.n * 8, e->stream));
    e->have_loc = true;
  }
  const bool move_nacc = e->eval_valid && e->nacc_base;   // nacc holds every row outside dirty_rows
  const bool move_auc = e->auc_state;
  const uint32_t auc_kept = std::min(e->auc_kept, n_old);
  // the range after the splice (a communicator's share and an open-ended pm_set_shard range move with W)
  e->n_workers = n_new;
  uint32_t b0 = 0, nb = 0;
  e->shard(&b0, &nb);
  const uint32_t b1 = (uint32_t)std::min<uint64_t>((uint64_t)b0 + nb, n_new);
  // the second buffers, with room to grow
  const size_t want = std::max<size_t>(n_new, 1);
  auto room = [&](auto& buf, size_t need) -> cudaError_t { return buf.p && buf.n >= need ? cudaSuccess : buf.ensure(need + need / 8); };
  PM_CUDA(room(e->wa_alt, want)); PM_CUDA(room(e->wb_alt, want));
  if (e->have_loc) { PM_CUDA(room(e->lat_alt, want)); PM_CUDA(room(e->lon_alt, want)); }
  if (e->have_rank) PM_CUDA(room(e->rank_alt, want));
  if (e->have_rep) PM_CUDA(room(e->rep_alt, want));
  if (move_nacc) PM_CUDA(room(e->nacc_alt, want));
  if (e->eval_valid) PM_CUDA(room(e->first_alt, want));
  if (move_auc) { PM_CUDA(room(e->price_alt, want + 2)); PM_CUDA(room(e->owner_alt, want)); }
  pm::WorkerSplice s{};
  s.removed = rm_dev; s.before = bf_dev; s.nr = nr; s.ni = ni; s.n_old = n_old;
  s.wa = e->wa.p; s.wb = e->wb.p; s.ins_a = e->upd_a.p; s.ins_b = e->upd_b.p; s.wa_out = e->wa_alt.p; s.wb_out = e->wb_alt.p;
  if (e->have_loc) {
    s.lat = e->lat.p; s.lon = e->lon.p; s.lat_out = e->lat_alt.p; s.lon_out = e->lon_alt.p;
    s.ins_lat = lat ? e->upd_lat.p : nullptr; s.ins_lon = lat ? e->upd_lon.p : nullptr;
  }
  if (e->have_rank) { s.rank = e->addr_rank.p; s.rank_out = e->rank_alt.p; }
  if (e->have_rep) { s.rep = e->reputation.p; s.rep_out = e->rep_alt.p; }
  if (move_nacc) { s.nacc = e->nacc.p; s.nacc_out = e->nacc_alt.p; s.nacc_n = (uint32_t)std::min<size_t>(e->nacc.n, n_old); }
  if (e->eval_valid) { s.first = e->eval_first.p; s.first_out = e->first_alt.p; s.a0 = a0; s.a1 = std::max(a0, a1); s.b0 = b0; s.b1 = std::max(b0, b1); }
  if (move_auc) { s.price = e->auc_price.p; s.price_out = e->price_alt.p; s.owner = e->auc_owner.p; s.owner_out = e->owner_alt.p; s.auc_kept = auc_kept; }
  if (n_old + ni) {
    pm::pm_splice_workers<<<std::min(blocks_for((size_t)n_old + ni, 256), 8u * e->sms), 256, 0, e->stream>>>(s);
    PM_LAUNCH_CHECK("pm_splice_workers");
  }
  std::swap(e->wa, e->wa_alt); std::swap(e->wb, e->wb_alt);
  if (e->have_loc) { std::swap(e->lat, e->lat_alt); std::swap(e->lon, e->lon_alt); }
  if (e->have_rank) std::swap(e->addr_rank, e->rank_alt);
  if (e->have_rep) std::swap(e->reputation, e->rep_alt);
  if (move_nacc) std::swap(e->nacc, e->nacc_alt);
  if (e->eval_valid) std::swap(e->eval_first, e->first_alt);
  if (move_auc) {
    std::swap(e->auc_price, e->price_alt); std::swap(e->auc_owner, e->owner_alt);
    PM_CUDA(cudaMemsetAsync(e->auc_price.p + n_new, 0, 2 * 8, e->stream));
    const uint32_t D = e->n_slots();
    if (D) {
      pm::pm_splice_worker_holds<<<std::min(blocks_for(D, 256), 8u * e->sms), 256, 0, e->stream>>>(e->auc_assigned.p, D, rm_dev, nr, bf_dev,
                                                                                                  ni, auc_kept);
      PM_LAUNCH_CHECK("pm_splice_worker_holds");
    }
  }
  // the caller's arrays and the host vectors behind the staging copies are released once the copies are done
  PM_CUDA(cudaStreamSynchronize(e->stream));
  if (e->eval_valid) {
    // The written rows move with their rows.  Rows that enter the range (their old row was outside it, or they are
    // inserted) count as written; the rest of [L, U) are kept rows of the old range.  Inserted rows are written
    // wherever they lie, for the preludes.
    sp.apply_list(&e->dirty_rows, &e->dirty_mark);
    e->dirty_mark.assign(n_new, 0);
    for (uint32_t i : e->dirty_rows) e->dirty_mark[i] = 1;
    e->dirty_in = 0;
    for (uint32_t i : e->dirty_rows) e->dirty_in += e->in_range(i);
    if (e->dirty_in > e->tune_incr) e->mark_all_dirty();
    uint32_t lo = a0, hi = a1;   // the first and one past the last kept row of the old range
    while (lo < hi && sp.is_removed(lo)) ++lo;
    while (hi > lo && sp.is_removed(hi - 1)) --hi;
    const uint32_t L = lo < hi ? sp.map(lo) : n_new, U = lo < hi ? sp.map(hi - 1) + 1 : n_new;
    if (std::min(b1, L) > b0) e->mark_range_dirty(b0, std::min(b1, L) - b0);
    if (b1 > std::max(b0, U)) e->mark_range_dirty(std::max(b0, U), b1 - std::max(b0, U));
    for (uint32_t k = 0; k < ni; ++k) e->mark_dirty(sp.at(k));
  }
  if (move_auc) {
    // Rows below the new auc_kept are the kept rows below the old one and the rows inserted before them (listed, as
    // changed rows); every row from it on is the old range past auc_kept, and the rows inserted there.
    sp.apply_list(&e->auc_rows, &e->auc_row_mark);
    e->auc_kept = sp.edge(auc_kept);
    e->auc_state_w = n_new;
    e->auc_row_mark.assign(n_new, 0);
    for (uint32_t i : e->auc_rows) e->auc_row_mark[i] = 1;
    for (uint32_t k = 0; k < ni && sp.before[k] < auc_kept; ++k) e->auc_mark_row(sp.at(k));
    e->auc_workers_spliced = true;
  }
  e->workers_checked = false;
  e->nacc_valid = false;
  e->matched = e->local_done = false;
  return PM_OK;
}

// A failure after the checks (a CUDA error, a host exception) leaves tables that are not trusted: the worker table is
// dropped with the stored evaluation and auction state, and the next call that needs it is PM_E_STATE
static int worker_splice(pm_engine* e, const WorkerSpliceH& sp, const pm_worker_a* a, const pm_worker_b* b,
                         const double* lat, const double* lon) {
  int rc;
  try {
    rc = splice_workers(e, sp, a, b, lat, lon);
  } catch (...) {
    rc = pm_guard_rc();
    e->err = "worker table splice: host exception (the worker table was dropped)";
  }
  if (rc != PM_OK) {
    e->have_workers = false;
    e->invalidate_eval();
    e->auc_discard();
  }
  return rc;
}

int pm_remove_workers(pm_engine* e, const uint32_t* idx, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_remove_workers: no worker table");
  std::vector<uint32_t> removed;
  {
    std::string err;
    const int rc = check_remove_workers(e, idx, n, &removed, &err);
    if (rc != PM_OK) return e->fail((pm_status)rc, err);
  }
  if (removed.empty()) return PM_OK;
  ++e->table_version;
  return worker_splice(e, WorkerSpliceH(e->n_workers, std::move(removed), {}), nullptr, nullptr, nullptr, nullptr);
} catch (...) { return pm_guard_rc(); }

int pm_insert_workers(pm_engine* e, const uint32_t* before, const pm_worker_a* a, const pm_worker_b* b, const double* lat,
                      const double* lon, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_insert_workers: no worker table");
  {
    std::string err;
    const int rc = check_insert_workers(e, before, a, b, lat, lon, n, &err);
    if (rc != PM_OK) return e->fail((pm_status)rc, err);
  }
  if (n == 0) return PM_OK;
  ++e->table_version;
  return worker_splice(e, WorkerSpliceH(e->n_workers, {}, std::vector<uint32_t>(before, before + n)), a, b, lat, lon);
} catch (...) { return pm_guard_rc(); }

uint64_t pm_table_version(const pm_engine* e) { return e ? e->table_version : 0; }

// A second engine on the same device with the same configuration and its own stream and tables.
int pm_create_sibling(const pm_engine* e, pm_engine** out) try {
  if (!e || !out) return PM_E_INVALID;
  pm_cfg c = e->cfg;
  c.stream = nullptr;
  c.shard_first = c.shard_count = 0;
  return pm_create(&c, out);
} catch (...) { return pm_guard_rc(); }

// ------------------------------------------------------------------ evaluation
// Fast predicate only when both tables fit its operand limits; decided per match.  `rows` (an incremental pass, the
// device list of the n_rows rows written since the last evaluation): when every other row passed the last check, only
// these are checked, starting from that check's flags.
static int decide_fast(pm_engine* e, bool* fast, const uint32_t* rows = nullptr, uint32_t n_rows = 0) {
  *fast = false;
  if (e->tune_generic || !e->asks_small) return PM_OK;
  if (!e->workers_checked) {
    const bool partial = rows && e->workers_base;
    const uint32_t one[2] = {partial ? (uint32_t)e->workers_small : 1u, partial ? (uint32_t)e->prices_narrow : 1u};
    PM_CUDA(cudaMemcpyAsync(e->counters.p + 2, one, 8, cudaMemcpyHostToDevice, e->stream));
    if (partial) {
      if (n_rows) {
        pm::pm_check_worker_rows<<<blocks_for(n_rows, 256), 256, 0, e->stream>>>(e->wa.p, e->wb.p, rows, n_rows, e->counters.p + 2);
        PM_LAUNCH_CHECK("pm_check_worker_rows");
      }
    } else if (e->n_workers) {
      pm::pm_check_worker_ranges<<<blocks_for(e->n_workers, 256), 256, 0, e->stream>>>(e->wa.p, e->wb.p, e->n_workers, e->counters.p + 2);
      PM_LAUNCH_CHECK("pm_check_worker_ranges");
    }
    PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 4, e->counters.p + 2, 8, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));
    e->workers_small = e->h_scalars.p[4] != 0;
    e->prices_narrow = e->h_scalars.p[5] != 0;
    e->workers_checked = true;
  }
  *fast = e->workers_small;
  return PM_OK;
}

// FastRow.wp follows the model table: (re)bound after either table changed
static int bind_rows(pm_engine* e, bool wm) {
  if (e->rows_bound && e->rows_bound_wm == wm) return PM_OK;
  if (e->n_asks) {
    pm::pm_bind_rows<<<blocks_for(e->n_asks, 256), 256, 0, e->stream>>>(e->frows.p, e->opts_fast.p, wm ? e->bits_wm.p : e->bits.p,
                                                                        wm ? 1u : e->words, e->n_asks);
    PM_LAUNCH_CHECK("pm_bind_rows");
  }
  e->rows_bound = true;
  e->rows_bound_wm = wm;
  return PM_OK;
}

// More distinct model strings than the shared-memory acceptance table holds (BITS == 0: one global-memory lookup per
// (row, worker) pair, build kernel at 0.64 of the copy peak with 100k strings): turn the table around.  With at most 30
// patterns a worker's acceptance over ALL of them is one word, computed once per table change; the kernels then run
// their one-word form (BITS == 2) with the roles of row and worker swapped (EvalParams::nacc).  Fast predicate only.
// `rows` as in decide_fast: an incremental pass recomputes only the listed rows' words when the others still hold.
static int worker_major(pm_engine* e, pm::EvalParams* p, int* bits_mode, const uint32_t* rows = nullptr, uint32_t n_rows = 0) {
  if (!e->nacc_valid && rows && e->nacc_base) {
    PM_CUDA(e->nacc.grow_keep(std::max<uint32_t>(e->n_workers, 1), e->nacc.n, e->stream));   // new rows are listed
    if (n_rows) {
      pm::pm_worker_nacc_rows<<<blocks_for(n_rows, 256), 256, 0, e->stream>>>(e->wa.p, e->bits.p, e->words, p->n_bits_rows, rows, n_rows, e->nacc.p);
      PM_LAUNCH_CHECK("pm_worker_nacc_rows");
    }
    e->nacc_valid = true;
  }
  if (!e->nacc_valid) {
    PM_CUDA(e->nacc.ensure(std::max<uint32_t>(e->n_workers, 1)));
    PM_CUDA(e->bits_wm.ensure(32));
    uint32_t host[32];
    for (uint32_t r = 0; r < 32; ++r) host[r] = ~(1u << r);
    PM_CUDA(cudaMemcpyAsync(e->bits_wm.p, host, sizeof host, cudaMemcpyHostToDevice, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));   // `host` is a local
    if (e->n_workers) {
      pm::pm_worker_nacc<<<blocks_for(e->n_workers, 256), 256, 0, e->stream>>>(e->wa.p, e->bits.p, e->words, p->n_bits_rows, e->n_workers, e->nacc.p);
      PM_LAUNCH_CHECK("pm_worker_nacc");
    }
    e->nacc_valid = true;
  }
  p->bits = e->bits_wm.p;
  p->words = 1;
  p->nacc = e->nacc.p;
  *bits_mode = 2;
  return PM_OK;
}

// The predicate variant of every evaluation pass: `p` from eval_params, `bits_mode` from the acceptance table's size
// (2: one word per row, 1: the table in shared memory, 0: in global memory), the fast predicate when decide_fast
// allows it, and then the worker-major one-word table where the global-memory one would run (worker_major; p->nacc
// is set exactly then).  `rows` as in decide_fast.
static int pick_predicate(pm_engine* e, pm::EvalParams* p, int* bits_mode, bool* fast, const uint32_t* rows = nullptr,
                          uint32_t n_rows = 0) {
  *p = eval_params(e);
  *bits_mode = ((uint64_t)p->n_bits_rows * p->words <= (uint64_t)pm::kBitsCap) ? (p->words == 1 ? 2 : 1) : 0;
  const int rc = decide_fast(e, fast, rows, n_rows);
  if (rc != PM_OK) return rc;
  if (*fast && *bits_mode == 0 && p->n_bits_rows <= 31u) return worker_major(e, p, bits_mode, rows, n_rows);
  return PM_OK;
}

// The 32-bit cost tile, built and reduced in one launch per tile (pm_build_argmin, pm_build_argmin_feat): on the
// FastRow path, for tables whose every price is below 0x7FFFFFFF (decide_fast).  The generic predicate and other
// prices keep the int64 tile, built and reduced by separate launches; PM_TUNE_BUILD=8 keeps it on the FastRow path
// too, the 32-bit tile's reference.
static bool narrow_tile(const pm_engine* e, bool fast) {
  return fast && e->prices_narrow && !e->tune_wide;
}

// The int64 tile's build
static void launch_build(pm_engine* e, const pm::EvalParams& p, int bits_mode, bool fast, dim3 grid,
                         uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw, long long* tile, size_t ld) {
  e->cost.overwritten();   // tile is e->cost.p
#define PM_BUILD_CASE(B) pm::pm_build_cost<B><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, t0, nt, w0, nw, tile, ld)
#define PM_FAST_CASE(B)                                                                                                 \
  {                                                                                                                     \
    grid.y = blocks_for(nt, pm::kFastRows);                                                                             \
    pm::pm_build_cost_fast<B><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, t0, nt, w0, nw, tile, ld);                   \
  }
  if (fast) {   // the FastRow kernel
    // one-word acceptance rows are bound into the FastRows (pm_bind_rows) however many rows there are
    if (p.words == 1) bits_mode = 2;
    if (bits_mode == 2) PM_FAST_CASE(2)
    else if (bits_mode == 1) PM_FAST_CASE(1)
    else PM_FAST_CASE(0)
  } else {
    if (bits_mode == 2) PM_BUILD_CASE(2); else if (bits_mode == 1) PM_BUILD_CASE(1); else PM_BUILD_CASE(0);
  }
#undef PM_FAST_CASE
#undef PM_BUILD_CASE
}

static void launch_fused(pm_engine* e, const pm::EvalParams& p, int bits_mode, bool fast, bool stats, dim3 grid,
                         uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw) {
#define PM_FUSED_CASE(B, F, S) pm::pm_fused_eval<B, F, S><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, t0, nt, w0, nw, e->first_ask.p, e->ask_best.p, e->ask_count.p)
  // !stats (PM_NO_ASK_STATS) skips the per-ask outputs in every variant: they read INF / 0, as an incremental pass's do
#define PM_FUSED_BITS(F, S) { if (bits_mode == 2) PM_FUSED_CASE(2, F, S); else if (bits_mode == 1) PM_FUSED_CASE(1, F, S); else PM_FUSED_CASE(0, F, S); }
  if (fast && stats) PM_FUSED_BITS(true, true)
  else if (fast) PM_FUSED_BITS(true, false)
  else if (stats) PM_FUSED_BITS(false, true)
  else PM_FUSED_BITS(false, false)
#undef PM_FUSED_BITS
#undef PM_FUSED_CASE
}

// pm_build_argmin: the 32-bit tile's build and argmin in one launch (the stripe ranks of pm_stripe_rank in place).
// tile is e->cost.p; the feature kernel needs its maps prepared (TileBuf::prepare_held), and takes positions
// [t0, t0 + nt) of the pass's slot schedule (sched_row / sched_ask); pm_build_argmin takes asks [t0, t0 + nt).
static void launch_build_argmin(pm_engine* e, const pm::EvalParams& p, int bits_mode, uint32_t t0, uint32_t nt, uint32_t w0,
                                uint32_t nw, long long* tile, size_t ld) {
  const dim3 grid(blocks_for(ld, pm::kEvalCols), blocks_for(nt, pm::kFastRows));
  const pm::FoldOut fo{e->stripe_rank.p, e->rank_best.p, e->first_ask.p, e->ask_best.p, e->ask_count.p, e->feat_perm.p};
  uint32_t* t32 = reinterpret_cast<uint32_t*>(tile);
  if (e->feat_ok) {   // the feature rows of this pass (match_local)
    // Four CTAs per SM (__launch_bounds__: 64 registers, no spills, 12.75 KB of shared memory each), the fastest of 2, 3
    // and 4 with the slot schedule (pm::kFeatRows).  The grid's rows are pm::kFeatRows per CTA, half the FastRow
    // kernels'; t0 / nt are positions of the slot schedule.
    const dim3 fgrid(grid.x, blocks_for(nt, pm::kFeatRows));
    pm::pm_build_argmin_feat<<<fgrid, pm::kEvalThreads, 0, e->stream>>>(e->sched_row.p, e->sched_ask.p, e->feat_o.p,
                                                                      e->feat_w.p, t0, nt, w0, nw, t32, ld, e->cost.held,
                                                                      e->cost.priced, fo);
    return;
  }
  e->cost.overwritten();
  if (p.words == 1) bits_mode = 2;   // one-word acceptance rows are bound into the FastRows, as in launch_build
  if (bits_mode == 2) pm::pm_build_argmin<2><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, t0, nt, w0, nw, t32, ld, fo);
  else if (bits_mode == 1) pm::pm_build_argmin<1><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, t0, nt, w0, nw, t32, ld, fo);
  else pm::pm_build_argmin<0><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, t0, nt, w0, nw, t32, ld, fo);
}

// The int64 tile's argmin
static void launch_argmin(pm_engine* e, cudaStream_t st, const long long* tile, size_t ld, uint32_t nt, uint32_t t0,
                          uint32_t w0, uint32_t nw) {
  // 16 x 16 B in flight per lane: a warp's slice is 8 x 64 columns
  dim3 grid(blocks_for(ld, 8 * 64 * pm::kArgWarps), blocks_for(nt, pm::kArgRows));
  pm::pm_argmin<8, 2><<<grid, pm::kArgThreads, 0, st>>>(tile, ld, nt, t0, w0, nw, e->first_ask.p, e->ask_best.p,
                                                        e->ask_count.p);
}

// The incremental evaluation.  Three walks (pm_first_ask_rows) rewrite the stored per-worker first feasible ask; each
// merges with atomicMin after the resets, so their order does not matter:
//   * the rows written since it was taken: reset, and walked over every ask;
//   * after asks were disabled (`dis`, D): the orphans, workers whose stored first ask f is in D.  Only the device
//     holds the stored evaluation, so pm_collect_orphans finds them, resets them and lists them after the written rows,
//     each to be walked from f + 1; reading their count back is the pass's one extra host synchronisation, and only
//     D makes it;
//   * after asks were enabled (`en`, E): the E-pass, every worker against E only.  A worker whose f lies below every
//     ask of E is settled; the others gain min(f, first feasible ask of E).
// Then the stored copy goes to first_ask, the resolution's working copy.  Same predicate variant as the full pass
// would pick; the O(W) preludes (operand-range check, worker-major acceptance words) cover every written row, the walks
// the engine's range [w0, w0 + nw) only: written rows outside it are dropped, orphans are collected inside it and the
// E-pass walks its workers.
static int eval_incremental(pm_engine* e, const std::vector<uint32_t>& en, const std::vector<uint32_t>& dis) {
  const uint32_t W = e->n_workers, T = e->n_asks;
  uint32_t w0 = 0, nw = 0;
  e->shard(&w0, &nw);
  const uint32_t k = (uint32_t)e->dirty_rows.size(), kr = e->dirty_in;
  const uint32_t ne = (uint32_t)en.size(), nd = (uint32_t)dis.size();
  e->stats.n_tiles = kr;
  if (k || ne || nd) {
    // host staging [written rows (the preludes' list) | the range's written rows (the walk's list) | E | D]; the two
    // row lists are one when every written row lies in the range, and the preludes have none after rows_over.
    // Device: the row lists (then the orphans) in dirty_dev, E and D in toggle_dev
    const uint32_t kp = e->rows_over ? 0 : k;
    const bool one_list = kp == kr;
    const uint32_t kh = kp + (one_list ? 0 : kr);
    PM_CUDA(e->h_dirty.ensure((size_t)kh + ne + nd));
    uint32_t* h = e->h_dirty.p;
    if (one_list && kp) {
      std::memcpy(h, e->dirty_rows.data(), (size_t)k * 4);
    } else {
      std::memcpy(h, e->dirty_rows.data(), (size_t)kp * 4);
      uint32_t j = kp;
      for (uint32_t i : e->dirty_rows)
        if (i - w0 < nw) h[j++] = i;
    }
    std::memcpy(h + kh, en.data(), (size_t)ne * 4);
    std::memcpy(h + kh + ne, dis.data(), (size_t)nd * 4);
    PM_CUDA(e->dirty_dev.ensure(nd ? (size_t)kh + nw : std::max<size_t>(kh, 1)));
    PM_CUDA(e->toggle_dev.ensure((size_t)ne + nd));
    if (kh) PM_CUDA(cudaMemcpyAsync(e->dirty_dev.p, h, (size_t)kh * 4, cudaMemcpyHostToDevice, e->stream));
    if (ne + nd)
      PM_CUDA(cudaMemcpyAsync(e->toggle_dev.p, h + kh, ((size_t)ne + nd) * 4, cudaMemcpyHostToDevice, e->stream));
    const uint32_t* pre = e->rows_over ? nullptr : e->dirty_dev.p;   // null: the preludes check every row
    uint32_t* rows = e->dirty_dev.p + (one_list ? 0 : kp);
    PM_CUDA(e->incr_evals.ensure(1));
    PM_CUDA(cudaMemsetAsync(e->incr_evals.p, 0, 8, e->stream));
    pm::EvalParams p;
    int bits_mode = 0;
    bool fast = false;
    {
      const int rc = pick_predicate(e, &p, &bits_mode, &fast, pre, kp);
      if (rc != PM_OK) return rc;
    }
    auto walk = [&](const pm::AskWalk& a, dim3 grid) -> int {
#define PM_ROWS_CASE(B, F) pm::pm_first_ask_rows<B, F><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, a, e->eval_first.p, e->incr_evals.p)
      if (fast) {
        if (bits_mode == 2) PM_ROWS_CASE(2, true); else if (bits_mode == 1) PM_ROWS_CASE(1, true); else PM_ROWS_CASE(0, true);
      } else {
        if (bits_mode == 2) PM_ROWS_CASE(2, false); else if (bits_mode == 1) PM_ROWS_CASE(1, false); else PM_ROWS_CASE(0, false);
      }
#undef PM_ROWS_CASE
      PM_LAUNCH_CHECK("pm_first_ask_rows");
      return PM_OK;
    };
    Timer tm(e, &e->stats.ms_fused, e->stream);
    if (kr) {
      pm::pm_scatter_value<<<blocks_for(kr, 256), 256, 0, e->stream>>>(e->eval_first.p, rows, kr, pm::kNone);
      PM_LAUNCH_CHECK("pm_scatter_value");
    }
    uint32_t n_walk = kr;
    const uint32_t* starts = nullptr;
    if (nd && nw) {
      PM_CUDA(e->walk_start.ensure((size_t)kr + nw));
      if (kr) PM_CUDA(cudaMemsetAsync(e->walk_start.p, 0, (size_t)kr * 4, e->stream));   // written rows: every ask
      PM_CUDA(cudaMemsetAsync(e->counters.p + 16, 0, 4, e->stream));
      pm::pm_collect_orphans<<<blocks_for(nw, 256), 256, 0, e->stream>>>(e->eval_first.p, w0, nw, e->toggle_dev.p + ne, nd,
                                                                         rows + kr, e->walk_start.p + kr, e->counters.p + 16);
      PM_LAUNCH_CHECK("pm_collect_orphans");
      PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 16, e->counters.p + 16, 4, cudaMemcpyDeviceToHost, e->stream));
      PM_CUDA(cudaStreamSynchronize(e->stream));   // the orphan count sizes the walk's grid
      n_walk = kr + e->h_scalars.p[16];
      starts = e->walk_start.p;
      e->stats.n_tiles = n_walk;
    }
    if (n_walk) {
      // about four CTAs per SM in all: few listed workers split the asks into more chunks
      const uint32_t gx = blocks_for(n_walk, pm::kEvalCols);
      const uint32_t steps = blocks_for(T, pm::kEvalRows);
      const uint32_t want_y = std::max(1u, std::min(steps, blocks_for(4u * e->sms, gx)));
      const uint32_t chunk = blocks_for(steps, want_y) * pm::kEvalRows;
      const int rc = walk(pm::AskWalk{rows, starts, nullptr, n_walk, T, chunk, 0}, dim3(gx, blocks_for(T, chunk)));
      if (rc != PM_OK) return rc;
    }
    if (ne && nw) {   // every worker of the range against all of E: E is short, and nw / 1024 CTAs spread over the SMs
      const int rc = walk(pm::AskWalk{nullptr, nullptr, e->toggle_dev.p, nw, ne, ne, w0}, dim3(blocks_for(nw, pm::kEvalCols), 1));
      if (rc != PM_OK) return rc;
    }
    tm.stop();
    // read back with the pass's one host synchronisation (match_finish_locked)
    PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 30, e->incr_evals.p, 8, cudaMemcpyDeviceToHost, e->stream));
    e->incr_evals_pending = true;
  }
  PM_CUDA(cudaMemcpyAsync(e->first_ask.p, e->eval_first.p, (size_t)W * 4, cudaMemcpyDeviceToDevice, e->stream));
  e->clear_dirty();
  e->clear_toggled();
  return PM_OK;
}

static int match_local_locked(pm_engine* e, uint32_t mode) {
  if (!e->have_workers || !e->have_asks) return e->fail(PM_E_STATE, "pm_match: worker and ask tables must be set first");
  if (e->max_pattern_row > e->n_patterns || (e->max_pattern_row && !e->have_bits))
    return e->fail(PM_E_STATE, "pm_match: an ask references a model pattern missing from the model table");
  const uint32_t base_mode = mode & 0xFFu;
  if (base_mode == PM_MODE_AUCTION) return e->fail(PM_E_INVALID, "pm_match: auction mode goes through pm_match");
  if (base_mode != PM_MODE_FIRST_FIT && base_mode != PM_MODE_PROXIMITY && base_mode != PM_MODE_PROXIMITY_MERGE)
    return e->fail(PM_E_INVALID, "pm_match: unknown mode");
  if ((base_mode == PM_MODE_PROXIMITY && !e->all_solo) || base_mode == PM_MODE_PROXIMITY_MERGE) {
    if (!e->have_loc) return e->fail(PM_E_STATE, "pm_match: proximity mode needs pm_set_worker_locations");
    if (e->any_max_zero)
      return e->fail(PM_E_UNSUPPORTED, "pm_match: max_group_size == 0 is not supported in proximity mode");
  }
  {
    const int rc = use_ask_form(e, false);
    if (rc != PM_OK) return rc;
  }
  PM_CUDA(cudaSetDevice(e->device));
  const uint32_t W = e->n_workers, T = e->n_asks;
  uint32_t w0 = 0, nw = 0;
  e->shard(&w0, &nw);
  if ((uint64_t)w0 + nw > W) return e->fail(PM_E_INVALID, "pm_match: shard range exceeds the worker table");
  if (!e->have_bits) {  // tables without any model clause: a one-row all-ones table
    PM_CUDA(e->bits.ensure(1));
    PM_CUDA(cudaMemsetAsync(e->bits.p, 0xFF, 4, e->stream));
    e->words = 1;
  }

  e->stats = pm_stats{};
  e->incr_evals_pending = false;
  e->ev_pending.clear();
  e->ev_used = 0;
  const bool timing = (e->cfg.flags & PM_CFG_TIMING) != 0;
  if (timing) PM_CUDA(cudaEventRecord(e->ev0, e->stream));

  // PM_INCREMENTAL: re-evaluate the rows of this engine's range written since the stored evaluation when there is one
  // and few of them changed.  Each engine decides for itself: sharded ranks may differ (exchange_locked).
  const bool incr = (mode & PM_INCREMENTAL) != 0;
  std::vector<uint32_t> en, dis;   // asks enabled / disabled since the stored evaluation
  if (incr && e->eval_valid) e->split_toggles(&en, &dis);
  // The E-pass evaluates up to |E| x nw pairs, as many as |E| nw / T written rows walked in full: they count against
  // the same cutoff (DESIGN §5)
  const uint64_t e_rows = T ? ((uint64_t)en.size() * nw + T - 1) / T : 0;
  const bool use_incr = incr && e->eval_valid && !e->dirty_over && e->tune_incr != 0 &&
                        e->dirty_in + e_rows <= e->tune_incr && T && nw;

  PM_CUDA(e->first_ask.ensure(W));
  PM_CUDA(e->ask_best.ensure(T));
  PM_CUDA(e->ask_count.ensure(T));
  if (!use_incr) PM_CUDA(cudaMemsetAsync(e->first_ask.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
  PM_CUDA(cudaMemsetAsync(e->ask_count.p, 0, (size_t)std::max<uint32_t>(T, 1) * 4, e->stream));
  if (T) {
    pm::pm_fill_i64<<<std::min(blocks_for(T, 256), 8u * e->sms), 256, 0, e->stream>>>(e->ask_best.p, pm::kInf, T);
    PM_LAUNCH_CHECK("pm_fill_i64");
  }

  if (use_incr) {
    const int rc = eval_incremental(e, en, dis);
    if (rc != PM_OK) return rc;
  } else if (T && nw) {
    pm::EvalParams p;
    int bits_mode = 0;
    bool fast = false;
    {
      const int rc = pick_predicate(e, &p, &bits_mode, &fast);
      if (rc != PM_OK) return rc;
    }
    if (mode & PM_PATH_FUSED) {
      Timer tm(e, &e->stats.ms_fused, e->stream);
      const uint32_t rows_per_launch = 65535u * pm::kEvalRows;
      for (uint32_t t0 = 0; t0 < T; t0 += rows_per_launch) {
        const uint32_t nt = std::min(rows_per_launch, T - t0);
        dim3 grid(blocks_for(nw, pm::kEvalCols), blocks_for(nt, pm::kEvalRows));
        launch_fused(e, p, bits_mode, fast, (mode & PM_NO_ASK_STATS) == 0, grid, t0, nt, w0, nw);
        PM_LAUNCH_CHECK("pm_fused_eval");
        ++e->stats.n_fused_launches;
      }
      tm.stop();
      e->stats.n_tiles = 1;
    } else {
      // leading dimension = whole CTA stripes of the build kernel (1024 columns): its stores need no bounds test;
      // the columns past the shard hold "infeasible" and cost 0.05 % of a 1M-worker row
      const size_t ld = (((size_t)nw + pm::kEvalCols - 1) / pm::kEvalCols) * pm::kEvalCols;
      {
        const int rc = bind_rows(e, p.nacc != nullptr);
        if (rc != PM_OK) return rc;
      }
      // rows are sized by 8 B per element for both widths: the 32-bit tile covers the same asks in half the bytes, so
      // tiles and launches are the same whichever width runs
      const bool narrow = narrow_tile(e, fast);
      const uint32_t elem_bytes = narrow ? 4u : 8u;
      uint64_t rows = e->cfg.cost_tile_bytes / (ld * 8);
      if (rows == 0) rows = 1;
      rows = std::min<uint64_t>(rows, T);
      rows = std::min<uint64_t>(rows, 65535ull * pm::kArgRows);
      if (rows >= 1024) rows &= ~(uint64_t)511;   // whole row bands of the build kernel (no ragged last band in every tile)
      // pm_build_argmin_feat's launches follow the slot schedule: Ks = n_tiles - 1 scheduled launches before the final
      // writers' when there are three tiles or more, else the natural order (Ks = 0)
      const uint32_t n_tiles = (uint32_t)((T + rows - 1) / rows);
      const uint32_t sched_ks = narrow && e->feat_ok && n_tiles >= 3 ? n_tiles - 1 : 0u;
      const size_t tile_elems = (size_t)rows * ld * elem_bytes / 8;   // TileBuf elements; ld is a multiple of 1024
      if (e->cost.ensure(tile_elems, e->device, e->tune_compress != 0, e->stream) != cudaSuccess) {
        cudaGetLastError();
        return e->fail(PM_E_NOMEM, "pm_match: cannot allocate the cost tile; lower pm_cfg.cost_tile_bytes");
      }
      // One launch per tile (pm_build_argmin) wherever the 32-bit tile runs; the int64 tile takes a build and an
      // argmin launch
      if (narrow) {   // each column's rank within its stripe, from this pass's prices (ordered after any table update)
        PM_CUDA(e->stripe_rank.ensure(ld));
        PM_CUDA(e->rank_best.ensure(ld));
        const uint32_t* perm = nullptr;   // worker order
        if (e->feat_ok) {   // the feature predicate: this pass's R per ask and option row, F per worker, column order
          PM_CUDA(e->feat_w.ensure(ld));
          PM_CUDA(e->feat_a.ensure(T));
          PM_CUDA(e->feat_o.ensure(std::max<uint32_t>(e->n_opts, 1)));
          PM_CUDA(e->feat_key.ensure(ld));
          PM_CUDA(e->feat_key_s.ensure(ld));
          PM_CUDA(e->feat_val.ensure(ld));
          PM_CUDA(e->feat_perm.ensure(ld));
          pm::pm_feature_asks<<<blocks_for(T, 256), 256, 0, e->stream>>>(e->frows.p, e->opts_fast.p, T, e->feat, e->feat_a.p,
                                                                         e->feat_o.p);
          PM_LAUNCH_CHECK("pm_feature_asks");
          // the slot schedule (pm_kernels.cuh pm_sched_gather): the asks before the final writers sorted by R_0
          PM_CUDA(e->sched_row.ensure(T));
          PM_CUDA(e->sched_ask.ensure(T));
          const uint32_t* sorted = nullptr;
          if (sched_ks) {
            const uint32_t m = T - (uint32_t)rows;
            PM_CUDA(e->sched_key.ensure(m));
            PM_CUDA(e->sched_key_s.ensure(m));
            PM_CUDA(e->sched_val.ensure(m));
            PM_CUDA(e->sched_val_s.ensure(m));
            pm::pm_sched_keys<<<blocks_for(m, 256), 256, 0, e->stream>>>(e->feat_a.p, m, e->sched_key.p, e->sched_val.p);
            PM_LAUNCH_CHECK("pm_sched_keys");
            const int begin_bit = 64 - std::max<int>((int)e->feat.off[pm::kFeatKinds], 1);   // as the column sort's
            size_t tmp = 0;
            PM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, e->sched_key.p, e->sched_key_s.p, e->sched_val.p,
                                                    e->sched_val_s.p, (int)m, begin_bit, 64, e->stream));
            PM_CUDA(e->cub_tmp.ensure(tmp));
            PM_CUDA(cub::DeviceRadixSort::SortPairs(e->cub_tmp.p, tmp, e->sched_key.p, e->sched_key_s.p, e->sched_val.p,
                                                    e->sched_val_s.p, (int)m, begin_bit, 64, e->stream));
            sorted = e->sched_val_s.p;
          }
          pm::pm_sched_gather<<<blocks_for(T, 256), 256, 0, e->stream>>>(e->feat_a.p, sorted, T, (uint32_t)rows, sched_ks,
                                                                         e->sched_row.p, e->sched_ask.p);
          PM_LAUNCH_CHECK("pm_sched_gather");
          pm::pm_feature_keys<<<blocks_for(ld, 256), 256, 0, e->stream>>>(e->wa.p, e->wb.p, e->bits.p, e->words, w0, nw, ld,
                                                                          e->feat, e->feat_key.p, e->feat_val.p,
                                                                          e->feat_key_s.p, e->feat_perm.p);
          PM_LAUNCH_CHECK("pm_feature_keys");
          // stable (LSD) over the key's top n bits, where __brevll put the dictionary's n features
          const int begin_bit = 64 - std::max<int>((int)e->feat.off[pm::kFeatKinds], 1);
          size_t tmp = 0;
          PM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, e->feat_key.p, e->feat_key_s.p, e->feat_val.p, e->feat_perm.p,
                                                  (int)nw, begin_bit, 64, e->stream));
          PM_CUDA(e->cub_tmp.ensure(tmp));
          PM_CUDA(cub::DeviceRadixSort::SortPairs(e->cub_tmp.p, tmp, e->feat_key.p, e->feat_key_s.p, e->feat_val.p,
                                                  e->feat_perm.p, (int)nw, begin_bit, 64, e->stream));
          perm = e->feat_perm.p;
        }
        pm::pm_stripe_rank<<<(unsigned)(ld / pm::kEvalCols), pm::kEvalThreads, 0, e->stream>>>(e->wb.p, perm, w0, nw,
                                                                                               e->stripe_rank.p, e->rank_best.p);
        PM_LAUNCH_CHECK("pm_stripe_rank");
        if (e->feat_ok) {
          pm::pm_feature_gather<<<blocks_for(ld, 256), 256, 0, e->stream>>>(e->wb.p, e->feat_key_s.p, e->feat_perm.p,
                                                                            e->stripe_rank.p, w0, nw, ld, e->feat_w.p);
          PM_LAUNCH_CHECK("pm_feature_gather");
        }
      }
      if (narrow && e->feat_ok) PM_CUDA(e->cost.prepare_held(e->stream));
      e->cost_tile_used = (size_t)rows * ld * elem_bytes;
      long long* tile = e->cost.p;
      for (uint32_t k = 0; k < n_tiles; ++k) {
        uint32_t t0 = k * (uint32_t)rows;
        uint32_t nt = (uint32_t)std::min<uint64_t>(rows, T - t0);
        if (sched_ks) {   // launch k of the schedule: positions [base_k, base_k + nt_k), the last one the final writers
          const uint32_t m = T - (uint32_t)rows, a = m / sched_ks, b = m % sched_ks;
          t0 = k < sched_ks ? k * a + std::min(k, b) : m;
          nt = k < sched_ks ? a + (k < b ? 1u : 0u) : (uint32_t)rows;
        }
        if (narrow) {
          // one launch that is both: its time counts in ms_build and in ms_argmin
          Timer tb(e, &e->stats.ms_build, e->stream);
          Timer ta(e, &e->stats.ms_argmin, e->stream);
          launch_build_argmin(e, p, bits_mode, t0, nt, w0, nw, tile, ld);
          PM_LAUNCH_CHECK("pm_build_argmin");
          ta.stop();
          tb.stop();
          ++e->stats.n_build_launches;
          ++e->stats.n_argmin_launches;
        } else {
          {
            Timer tm(e, &e->stats.ms_build, e->stream);
            dim3 grid(blocks_for(ld, pm::kEvalCols), blocks_for(nt, pm::kEvalRows));
            launch_build(e, p, bits_mode, fast, grid, t0, nt, w0, nw, tile, ld);
            PM_LAUNCH_CHECK("pm_build_cost");
            tm.stop();
            ++e->stats.n_build_launches;
          }
          {
            Timer tm(e, &e->stats.ms_argmin, e->stream);
            launch_argmin(e, e->stream, tile, ld, nt, t0, w0, nw);
            PM_LAUNCH_CHECK("pm_argmin");
            tm.stop();
            ++e->stats.n_argmin_launches;
          }
        }
        ++e->stats.n_tiles;
        // algorithmic: 4 or 8 B per evaluation, the tile's element (padding columns not counted)
        e->stats.cost_bytes_written += (uint64_t)nt * nw * elem_bytes;
        e->stats.cost_bytes_read += (uint64_t)nt * nw * elem_bytes;
      }
    }
    e->stats.evals = (uint64_t)T * nw;
  }
  if (!use_incr) {
    // every full evaluation refreshes the stored one: one 4 B-per-worker copy of the range's entries and NONE outside
    // it, taken before a communicator's exchange fills the rest of first_ask
    PM_CUDA(e->eval_first.ensure(std::max<uint32_t>(W, 1)));
    PM_CUDA(cudaMemcpyAsync(e->eval_first.p, e->first_ask.p, (size_t)W * 4, cudaMemcpyDeviceToDevice, e->stream));
    e->clear_dirty();
    e->dirty_mark.resize(W, 0);   // every mark is clear after clear_dirty
    e->clear_toggled();
    e->eval_on = e->ask_on;       // the mask this evaluation was taken under
    e->eval_valid = true;
    if (incr) e->stats.n_tiles = nw;   // rows re-evaluated
  }
  e->workers_base = e->eval_valid && e->workers_checked;
  e->nacc_base = e->eval_valid && e->nacc_valid;
  e->local_done = true;
  e->matched = false;
  return PM_OK;
}

// ------------------------------------------------------------------ resolution
static int sort_and_scan(pm_engine* e, uint32_t n_bins, uint32_t shift) {
  const uint32_t W = e->n_workers;
  PM_CUDA(cudaMemsetAsync(e->hist.p, 0, ((size_t)n_bins + 1) * 4, e->stream));
  if (W) {
    pm::pm_make_keys<<<blocks_for(W, 256), 256, 0, e->stream>>>(e->first_ask.p, e->wa.p, W, shift, e->keys.p, e->hist.p);
    PM_LAUNCH_CHECK("pm_make_keys");
  }
  size_t tmp_scan = 0, tmp_sort = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, e->hist.p, e->seg_start.p, (int)(n_bins + 1), e->stream);
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, e->keys.p, e->keys_sorted.p, e->iota.p, e->order.p, (int)W, 0, 32, e->stream);
  size_t tmp = std::max(tmp_scan, tmp_sort);
  PM_CUDA(e->cub_tmp.ensure(tmp));
  PM_CUDA(cub::DeviceScan::ExclusiveSum(e->cub_tmp.p, tmp, e->hist.p, e->seg_start.p, (int)(n_bins + 1), e->stream));
  if (W) PM_CUDA(cub::DeviceRadixSort::SortPairs(e->cub_tmp.p, tmp, e->keys.p, e->keys_sorted.p, e->iota.p, e->order.p, (int)W, 0, 32, e->stream));
  return PM_OK;
}

// The O(W + T) resolution sweep.  Everything between the sort and the last kernel stays on the device (counts are
// read through device pointers, tables are sized for the worst case), so a pass has exactly ONE host synchronisation:
// the one at the end that brings back {groups, members, bumped} (and resolves the event timers).
static int match_finish_locked(pm_engine* e, uint32_t mode) {
  if (!e->local_done) return e->fail(PM_E_STATE, "pm_match_finish: pm_match_local has not run");
  PM_CUDA(cudaSetDevice(e->device));
  const uint32_t base_mode = mode & 0xFFu;
  const uint32_t W = e->n_workers, T = e->n_asks;
  const bool merge_mode = base_mode == PM_MODE_PROXIMITY_MERGE;
  const bool prox_general = (base_mode == PM_MODE_PROXIMITY && !e->all_solo) || merge_mode;
  const uint32_t shift = (base_mode == PM_MODE_PROXIMITY && !prox_general) ? 1u : 0u;
  const uint32_t n_bins = T << shift;
  Timer tm(e, &e->stats.ms_resolve, e->stream);

  PM_CUDA(e->keys.ensure(W)); PM_CUDA(e->keys_sorted.ensure(W)); PM_CUDA(e->iota.ensure(W));
  PM_CUDA(e->order.ensure(W)); PM_CUDA(e->hist.ensure((size_t)n_bins + 1));
  PM_CUDA(e->seg_start.ensure((size_t)n_bins + 1)); PM_CUDA(e->ngroups.ensure((size_t)n_bins + 1));
  PM_CUDA(e->group_base.ensure((size_t)n_bins + 1));
  PM_CUDA(e->worker_group.ensure(W)); PM_CUDA(e->worker_ask.ensure(W)); PM_CUDA(e->members.ensure(W));
  PM_CUDA(cudaMemsetAsync(e->counters.p, 0, 12 * 4, e->stream));   // [12..13] belong to pm_set_asks
  if (W) {
    pm::pm_iota_u32<<<std::min(blocks_for(W, 256), 8u * e->sms), 256, 0, e->stream>>>(e->iota.p, W);
    PM_LAUNCH_CHECK("pm_iota_u32");
  }
  int rc = sort_and_scan(e, n_bins, shift);
  if (rc != PM_OK) return rc;
  uint32_t* const scal = e->counters.p + 8;   // device mailbox {groups, members, bumped, overflow}
  bool prox_grid_ran = false;

  if (prox_general) {
    // sequential-per-group nearest-neighbour formation (pm_proximity.cuh)
    uint32_t P = 1;
    while (P < std::max<uint32_t>(W, 1)) P <<= 1;
    const uint32_t cap = W + T + 1;
    PM_CUDA(e->base_len.ensure(T)); PM_CUDA(e->xhead.ensure(T)); PM_CUDA(e->xcount.ensure(T));
    PM_CUDA(e->xnext.ensure(W)); PM_CUDA(e->popped.ensure(W));
    PM_CUDA(e->prox_list.ensure(W)); PM_CUDA(e->prox_xs.ensure(P)); PM_CUDA(e->prox_dist.ensure(W));
    PM_CUDA(e->members_raw.ensure(W));
    PM_CUDA(e->group_ask.ensure((size_t)cap + 1)); PM_CUDA(e->group_off.ensure((size_t)cap + 1));
    PM_CUDA(cudaMemcpyAsync(e->base_len.p, e->hist.p, (size_t)T * 4, cudaMemcpyDeviceToDevice, e->stream));
    PM_CUDA(cudaMemsetAsync(e->xhead.p, 0xFF, (size_t)T * 4, e->stream));
    PM_CUDA(cudaMemsetAsync(e->xcount.p, 0, (size_t)T * 4, e->stream));
    PM_CUDA(cudaMemsetAsync(e->worker_group.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
    PM_CUDA(cudaMemsetAsync(e->worker_ask.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
    pm::ProxParams pp;
    pp.ev = eval_params(e);
    pp.lat = e->lat.p; pp.lon = e->lon.p;
    pp.cur = e->first_ask.p; pp.base_len = e->base_len.p; pp.seg_start = e->seg_start.p; pp.order = e->order.p;
    pp.xhead = e->xhead.p; pp.xnext = e->xnext.p; pp.xcount = e->xcount.p; pp.amin = e->amin.p; pp.amax = e->amax.p;
    pp.list = e->prox_list.p; pp.xs = e->prox_xs.p; pp.dist = e->prox_dist.p; pp.popped = e->popped.p;
    pp.worker_group = e->worker_group.p; pp.worker_ask = e->worker_ask.p; pp.group_ask = e->group_ask.p;
    pp.group_off = e->group_off.p; pp.members = e->members_raw.p; pp.out_counts = scal;   // {G, M, bumped, overflow}
    pp.group_cap = cap;
    if (e->coop_blocks < 0) {   // once per engine: can the whole-chip sweep be launched cooperatively, and how wide?
      int coop = 0, per_sm = 0, sms = 0;
      cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, e->device);
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->device);
      if (coop && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pm::pm_proximity_grid, pm::kPgThreads, 0) == cudaSuccess)
        e->coop_blocks = per_sm * sms;
      else
        e->coop_blocks = 0;
      (void)cudaGetLastError();
    }
    if (merge_mode) pm::pm_merge_sweep<<<1, pm::kProxThreads, 0, e->stream>>>(pp);
    else if (e->tune_prox == 0 && e->coop_blocks > 0) {
      // all SMs: one grid barrier per group instead of one CTA doing everything (pm_proximity_grid.cuh)
      const unsigned grid = std::max(1u, std::min<unsigned>((unsigned)e->coop_blocks, blocks_for(std::max<uint32_t>(W, 1), pm::kPgThreads)));
      PM_CUDA(e->pg_part_d.ensure((size_t)2 * grid * pm::kPgTopK)); PM_CUDA(e->pg_part_i.ensure((size_t)2 * grid * pm::kPgTopK));
      PM_CUDA(e->pg_cta_cnt.ensure((size_t)2 * grid)); PM_CUDA(e->pg_ctl.ensure(8));
      PM_CUDA(e->pg_clat.ensure(W)); PM_CUDA(e->pg_clon.ensure(W)); PM_CUDA(e->pg_ccos.ensure(W));
      PM_CUDA(cudaMemsetAsync(e->pg_ctl.p, 0, 32, e->stream));
      pm::GridProxParams gp;
      gp.p = pp;
      gp.part_d = e->pg_part_d.p; gp.part_i = e->pg_part_i.p; gp.cta_cnt = e->pg_cta_cnt.p; gp.gctl = e->pg_ctl.p;
      gp.clat = e->pg_clat.p; gp.clon = e->pg_clon.p; gp.ccos = e->pg_ccos.p;
      gp.n_workers = W;
      void* args[] = {&gp};
      PM_CUDA(cudaLaunchCooperativeKernel((const void*)pm::pm_proximity_grid, dim3(grid), dim3(pm::kPgThreads), args, 0, e->stream));
      PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 24, e->pg_ctl.p + 4, 12, cudaMemcpyDeviceToHost, e->stream));
      prox_grid_ran = true;
    }
    else pm::pm_proximity_sweep<<<1, pm::kProxThreads, 0, e->stream>>>(pp);
    PM_LAUNCH_CHECK("pm_proximity_sweep");
    if (W) {
      pm::pm_order_members<<<blocks_for(W, 256), 256, 0, e->stream>>>(
          e->members_raw.p, scal + 1, e->worker_group.p, e->group_off.p, e->have_rank ? e->addr_rank.p : nullptr, e->members.p);
      PM_LAUNCH_CHECK("pm_order_members");
    }
  } else {
    if (shift == 0 && T && !e->all_solo) {
      // under-filled tails: flagged on the device; the single-CTA sweep returns at once when there is none
      pm::pm_check_tails<<<blocks_for(T, 256), 256, 0, e->stream>>>(e->hist.p, e->amin.p, e->amax.p, T, e->counters.p);
      PM_LAUNCH_CHECK("pm_check_tails");
      PM_CUDA(e->base_len.ensure(T)); PM_CUDA(e->xhead.ensure(T)); PM_CUDA(e->xcount.ensure(T));
      PM_CUDA(e->xnext.ensure(W)); PM_CUDA(e->popped.ensure(W));
      PM_CUDA(cudaMemcpyAsync(e->base_len.p, e->hist.p, (size_t)T * 4, cudaMemcpyDeviceToDevice, e->stream));
      PM_CUDA(cudaMemsetAsync(e->xhead.p, 0xFF, (size_t)T * 4, e->stream));
      PM_CUDA(cudaMemsetAsync(e->xcount.p, 0, (size_t)T * 4, e->stream));
      pm::SweepParams sp;
      sp.ev = eval_params(e);
      sp.cur = e->first_ask.p; sp.base_len = e->base_len.p; sp.seg_start = e->seg_start.p;
      sp.order = e->order.p; sp.xhead = e->xhead.p; sp.xnext = e->xnext.p; sp.xcount = e->xcount.p;
      sp.amin = e->amin.p; sp.amax = e->amax.p; sp.popped = e->popped.p; sp.n_bumped = e->counters.p + 1;
      sp.any_bad = e->counters.p;
      pm::pm_sweep<<<1, 1024, 0, e->stream>>>(sp);
      PM_LAUNCH_CHECK("pm_sweep");
      rc = sort_and_scan(e, n_bins, shift);   // owners may have moved
      if (rc != PM_OK) return rc;
    }

    if (n_bins) {
      pm::pm_count_groups<<<blocks_for(n_bins, 256), 256, 0, e->stream>>>(e->hist.p, e->amin.p, e->amax.p, n_bins, shift, e->ngroups.p);
      PM_LAUNCH_CHECK("pm_count_groups");
    }
    PM_CUDA(cudaMemsetAsync(e->ngroups.p + n_bins, 0, 4, e->stream));
    {
      size_t tmp = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, tmp, e->ngroups.p, e->group_base.p, (int)(n_bins + 1), e->stream);
      PM_CUDA(e->cub_tmp.ensure(tmp));
      PM_CUDA(cub::DeviceScan::ExclusiveSum(e->cub_tmp.p, tmp, e->ngroups.p, e->group_base.p, (int)(n_bins + 1), e->stream));
    }
    // groups <= members + one empty group per bin; sized for that so the count never has to visit the host first
    const size_t gcap = (size_t)W + n_bins + 1;
    PM_CUDA(e->group_ask.ensure(gcap + 1));
    PM_CUDA(e->group_off.ensure(gcap + 1));
    const uint32_t* n_assigned_dev = e->seg_start.p + n_bins;
    PM_CUDA(cudaMemsetAsync(e->worker_group.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
    PM_CUDA(cudaMemsetAsync(e->worker_ask.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
    if (W) {
      pm::pm_emit_workers<<<blocks_for(W, 256), 256, 0, e->stream>>>(
          e->keys_sorted.p, e->order.p, n_assigned_dev, e->hist.p, e->seg_start.p, e->group_base.p, e->amin.p,
          e->amax.p, shift, e->worker_group.p, e->worker_ask.p, e->group_ask.p, e->group_off.p);
      PM_LAUNCH_CHECK("pm_emit_workers");
    }
    if (n_bins && !e->all_solo) {
      pm::pm_emit_empty_groups<<<blocks_for(n_bins, 256), 256, 0, e->stream>>>(
          e->hist.p, e->seg_start.p, e->group_base.p, e->ngroups.p, e->amin.p, n_bins, shift, e->group_ask.p, e->group_off.p);
      PM_LAUNCH_CHECK("pm_emit_empty_groups");
    }
    pm::pm_close_groups<<<1, 1, 0, e->stream>>>(e->group_base.p + n_bins, n_assigned_dev, e->counters.p + 1, e->group_off.p, scal);
    PM_LAUNCH_CHECK("pm_close_groups");
    if (W) {
      pm::pm_order_members<<<blocks_for(W, 256), 256, 0, e->stream>>>(
          e->order.p, n_assigned_dev, e->worker_group.p, e->group_off.p, e->have_rank ? e->addr_rank.p : nullptr, e->members.p);
      PM_LAUNCH_CHECK("pm_order_members");
    }
  }
  tm.stop();
  PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 8, scal, 16, cudaMemcpyDeviceToHost, e->stream));
  if (e->cfg.flags & PM_CFG_TIMING) PM_CUDA(cudaEventRecord(e->ev1, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));   // the pass's one host synchronisation
  if (prox_general && e->h_scalars.p[11]) return e->fail(PM_E_CUDA, "pm_match: proximity group table overflow");
  e->n_groups = e->h_scalars.p[8];
  e->n_assigned = e->h_scalars.p[9];
  e->stats.n_bumped = e->h_scalars.p[10];
  if (e->incr_evals_pending) {
    std::memcpy(&e->stats.evals, e->h_scalars.p + 30, 8);
    e->incr_evals_pending = false;
  }
  if (prox_grid_ran && !(mode & PM_INCREMENTAL)) {   // with PM_INCREMENTAL n_tiles keeps the rows re-evaluated   // cooperative proximity sweep: seed-parallel batches, groups formed in them, groups formed one at a time
    e->stats.n_tiles = e->h_scalars.p[24];
    e->stats.n_rounds = e->h_scalars.p[25];
    e->stats.n_build_launches = e->h_scalars.p[26];
  }
  if (e->cfg.flags & PM_CFG_TIMING) {
    PM_CUDA(cudaEventElapsedTime(&e->stats.ms_total, e->ev0, e->ev1));
    e->resolve_timers();
  }
  e->matched = true;
  return PM_OK;
}

// ------------------------------------------------------------------ extension: auction
// Ask classes for the auction: asks with identical requirement rows (pm_auction.cuh), over the T rows and floors given
// (the ask table, or with demands the slot table).
static int auction_build_classes(pm_engine* e, const pm::DevAsk* rows, const uint32_t* floor, uint32_t T) {
  e->auc_n_classes = 0;
  PM_CUDA(e->auc_class_of.ensure(T)); PM_CUDA(e->auc_class_rep.ensure(T)); PM_CUDA(e->auc_hash.ensure(T));
  PM_CUDA(e->auc_hash_out.ensure(T)); PM_CUDA(e->auc_idx.ensure(T)); PM_CUDA(e->auc_sorted.ensure(T));
  PM_CUDA(e->auc_flag.ensure((size_t)T + 1)); PM_CUDA(e->auc_incl.ensure(T));
  if (T == 0) { e->auc_classes_valid = true; return PM_OK; }
  pm::pm_auction_ask_hash<<<blocks_for(T, 256), 256, 0, e->stream>>>(rows, e->opts.p, floor, T, e->auc_hash.p, e->auc_idx.p);
  PM_LAUNCH_CHECK("pm_auction_ask_hash");
  size_t tmp_sort = 0, tmp_scan = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, e->auc_hash.p, e->auc_hash_out.p, e->auc_idx.p, e->auc_sorted.p, (int)T, 0, 64, e->stream);
  cub::DeviceScan::InclusiveSum(nullptr, tmp_scan, e->auc_flag.p, e->auc_incl.p, (int)T, e->stream);
  size_t tmp = std::max(tmp_sort, tmp_scan);
  PM_CUDA(e->cub_tmp.ensure(tmp));
  PM_CUDA(cub::DeviceRadixSort::SortPairs(e->cub_tmp.p, tmp, e->auc_hash.p, e->auc_hash_out.p, e->auc_idx.p, e->auc_sorted.p, (int)T, 0, 64, e->stream));
  pm::pm_auction_class_flags<<<blocks_for(T, 256), 256, 0, e->stream>>>(rows, e->opts.p, floor, e->auc_sorted.p, T, e->auc_flag.p);
  PM_LAUNCH_CHECK("pm_auction_class_flags");
  PM_CUDA(cub::DeviceScan::InclusiveSum(e->cub_tmp.p, tmp, e->auc_flag.p, e->auc_incl.p, (int)T, e->stream));
  pm::pm_auction_class_assign<<<blocks_for(T, 256), 256, 0, e->stream>>>(e->auc_sorted.p, e->auc_flag.p, e->auc_incl.p, T,
                                                                          e->auc_class_of.p, e->auc_class_rep.p);
  PM_LAUNCH_CHECK("pm_auction_class_assign");
  PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 16, e->auc_incl.p + (T - 1), 4, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  e->auc_n_classes = e->h_scalars.p[16];
  e->auc_classes_valid = true;
  return PM_OK;
}

// The auction's integer domain (prime_match.h, DESIGN 4): with P the largest ask price of the worker table, K the largest
// cap, S = cost_scale and E = eps_start, (P + K + 2) * S + E < 2^61 keeps every value, outside option, bid, profit and
// sort key strictly between -2^61 (kAucNeg, "no worker") and 2^61.  Evaluated in 128 bits: no product can wrap.
static bool auction_in_domain(uint32_t P, uint32_t K, uint64_t S, uint64_t E) {
  return ((unsigned __int128)P + K + 2u) * S + E < ((unsigned __int128)1 << 61);
}

static int auction_pass(pm_engine* e, bool want_warm, bool want_repair, bool reverse, bool* refused);

// The grouped result of a pass with demands (prime_match.h "Auction demands"): the slots' held flags and their scan give
// each ask's held count and its members' place; one group per ask holding a worker, in ask order; then each group's
// members sorted by worker index (one segmented sort).  *G groups, *M members.
static int auction_emit_groups(pm_engine* e, uint32_t* G, uint32_t* M) {
  const uint32_t W = e->n_workers, T = e->n_asks, D = e->n_slots();
  PM_CUDA(e->auc_flag.ensure((size_t)D + 1)); PM_CUDA(e->dem_spos.ensure((size_t)D + 1));
  PM_CUDA(e->dem_aflag.ensure((size_t)T + 1)); PM_CUDA(e->auc_gidx.ensure((size_t)T + 1));
  PM_CUDA(e->dem_members.ensure(std::max<uint32_t>(W, 1)));
  pm::pm_auction_slot_flags<<<blocks_for((size_t)D + 1, 256), 256, 0, e->stream>>>(e->auc_assigned.p, D, e->auc_flag.p);
  PM_LAUNCH_CHECK("pm_auction_slot_flags");
  size_t tmp = 0, tmp2 = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp, e->auc_flag.p, e->dem_spos.p, (int)(D + 1), e->stream);
  cub::DeviceScan::ExclusiveSum(nullptr, tmp2, e->dem_aflag.p, e->auc_gidx.p, (int)(T + 1), e->stream);
  PM_CUDA(e->cub_tmp.ensure(std::max(tmp, tmp2)));
  tmp = e->cub_tmp.n;
  PM_CUDA(cub::DeviceScan::ExclusiveSum(e->cub_tmp.p, tmp, e->auc_flag.p, e->dem_spos.p, (int)(D + 1), e->stream));
  pm::pm_auction_group_counts<<<blocks_for((size_t)T + 1, 256), 256, 0, e->stream>>>(e->dem_off.p, e->dem_spos.p, e->auc_assigned.p, e->wb.p,
                                                                                     T, e->dem_aflag.p, e->ask_best.p, e->ask_count.p);
  PM_LAUNCH_CHECK("pm_auction_group_counts");
  tmp = e->cub_tmp.n;
  PM_CUDA(cub::DeviceScan::ExclusiveSum(e->cub_tmp.p, tmp, e->dem_aflag.p, e->auc_gidx.p, (int)(T + 1), e->stream));
  PM_CUDA(cudaMemsetAsync(e->worker_group.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
  PM_CUDA(cudaMemsetAsync(e->worker_ask.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
  if (T) {
    pm::pm_auction_group_emit<<<blocks_for(T, 256), 256, 0, e->stream>>>(e->dem_off.p, e->dem_spos.p, e->auc_gidx.p, e->auc_assigned.p, T,
                                                                          e->worker_group.p, e->worker_ask.p, e->group_ask.p,
                                                                          e->group_off.p, e->dem_members.p);
    PM_LAUNCH_CHECK("pm_auction_group_emit");
  }
  PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 17, e->auc_gidx.p + T, 4, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 18, e->dem_spos.p + D, 4, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  *G = e->h_scalars.p[17];
  *M = e->h_scalars.p[18];
  PM_CUDA(cudaMemcpyAsync(e->group_off.p + *G, e->h_scalars.p + 18, 4, cudaMemcpyHostToDevice, e->stream));
  if (*G) {
    tmp = 0;
    cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp, e->dem_members.p, e->members.p, (int)*M, (int)*G, e->group_off.p,
                                            e->group_off.p + 1, 0, 32, e->stream);
    PM_CUDA(e->cub_tmp.ensure(tmp));
    PM_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(e->cub_tmp.p, tmp, e->dem_members.p, e->members.p, (int)*M, (int)*G, e->group_off.p,
                                                    e->group_off.p + 1, 0, 32, e->stream));
  }
  PM_CUDA(cudaStreamSynchronize(e->stream));   // (h_scalars is the copy's source)
  return PM_OK;
}
static int match_auction_locked(pm_engine* e, uint32_t mode) {
  if (!e->have_workers || !e->have_asks) return e->fail(PM_E_STATE, "pm_match: worker and ask tables must be set first");
  if (!e->have_caps) return e->fail(PM_E_STATE, "pm_match: auction mode needs pm_set_ask_price_caps");
  if (e->max_pattern_row > e->n_patterns || (e->max_pattern_row && !e->have_bits))
    return e->fail(PM_E_STATE, "pm_match: an ask references a model pattern missing from the model table");
  if (e->cfg.shard_count || e->comm) return e->fail(PM_E_UNSUPPORTED, "pm_match: auction mode is single-GPU");
  // the class cache is keyed on requirement rows, which a disabled ask's no longer are
  if (e->n_off) return e->fail(PM_E_UNSUPPORTED, "pm_match: auction mode with disabled asks");
  {
    const int rc = use_ask_form(e, true);
    if (rc != PM_OK) return rc;
  }
  bool refused = false;
  const int rc = auction_pass(e, (mode & PM_AUCTION_WARM) != 0, (mode & PM_AUCTION_REPAIR) != 0, (mode & PM_AUCTION_REVERSE) != 0,
                              &refused);
  // the stored state may be half released or half bid: it is not trusted again (a refused pass touched none of it)
  if (rc != PM_OK && !refused) e->auc_discard();
  return rc;
}

static int auction_pass(pm_engine* e, bool want_warm, bool want_repair, bool reverse, bool* refused) {
  PM_CUDA(cudaSetDevice(e->device));
  const uint32_t W = e->n_workers, T = e->n_asks;
  // the bidders: with demands the slots (pm_auction.cuh, "ask demands"), each ask t its own single bidder without
  const bool dem = !e->demand.empty();
  const uint32_t D = e->n_slots();
  if (!e->have_bits) {
    PM_CUDA(e->bits.ensure(1));
    PM_CUDA(cudaMemsetAsync(e->bits.p, 0xFF, 4, e->stream));
    e->words = 1;
  }
  e->stats = pm_stats{};
  e->ev_pending.clear();
  e->ev_used = 0;
  if (e->cfg.flags & PM_CFG_TIMING) PM_CUDA(cudaEventRecord(e->ev0, e->stream));
  Timer tm(e, &e->stats.ms_fused, e->stream);
  const bool use_rep = e->have_min_rep;   // `reputation` clause: only when a floor was given
  if (dem) {   // the slot table, from the current caps and floors: the auction's ask table
    PM_CUDA(e->slot_ask.ensure(D)); PM_CUDA(e->slot_row.ensure(D)); PM_CUDA(e->slot_cap.ensure(D));
    if (use_rep) PM_CUDA(e->slot_floor.ensure(D));
    pm::pm_auction_slot_table<<<std::min(blocks_for(D, 256), 8u * e->sms), 256, 0, e->stream>>>(
        e->dem_off.p, T, D, e->asks.p, e->price_cap.p, use_rep ? e->ask_min_rep.p : nullptr, e->slot_ask.p, e->slot_row.p,
        e->slot_cap.p, use_rep ? e->slot_floor.p : nullptr);
    PM_LAUNCH_CHECK("pm_auction_slot_table");
  }
  const uint32_t* cap_b = dem ? e->slot_cap.p : e->price_cap.p;   // per bidder
  const uint32_t* floor_b = use_rep ? (dem ? e->slot_floor.p : e->ask_min_rep.p) : nullptr;
  if (!e->auc_classes_valid) {
    const int rc = auction_build_classes(e, dem ? e->slot_row.p : e->asks.p, floor_b, D);
    if (rc != PM_OK) return rc;
  }
  const uint32_t C = e->auc_n_classes;
  const unsigned kScanGrid = 2u * e->sms;   // two scanning CTAs per SM (shared memory)
  // Warm start from the stored state when there is one and the changed rows R0 plus the changed asks A0 stay within the
  // cutoff.  A0: caps or floors that differ from the stored ones (a diff of the host copies), and asks toggled since,
  // as bidders: every slot of such an ask, and the slots a demand change added to any other.
  std::vector<uint32_t> changed;   // the listed rows of R0, then A0
  bool warm = false;
  uint32_t n_kept = 0;
  if (want_warm && e->auc_state && !e->auc_rows_over) {
    changed = e->auc_rows;
    for (uint32_t t = 0; t < T; ++t) {
      const uint32_t fl = e->have_min_rep ? e->floor_host[t] : 0u;
      const bool a0 = e->cap_host[t] != e->auc_cap_stored[t] || fl != e->auc_floor_stored[t] || e->auc_ask_mark[t];
      const uint32_t s0 = e->slot0(t), s1 = e->slot0(t + 1);
      const uint32_t kept = a0 ? 0u : e->auc_dem_kept.empty() ? s1 - s0 : std::min(e->auc_dem_kept[t], s1 - s0);
      for (uint32_t s = s0 + kept; s < s1; ++s) changed.push_back(s);
    }
    n_kept = std::min(e->auc_kept, W);
    warm = (uint64_t)changed.size() + (W - n_kept) + e->auc_removed_held <= e->tune_incr;
  }
  const uint32_t n_rows = warm ? (uint32_t)e->auc_rows.size() : 0u, n_chg = warm ? (uint32_t)changed.size() - n_rows : 0u;
  const bool repair = want_repair && warm;   // PM_AUCTION_REPAIR: the same warm start, repaired by raising instead of releasing
  // the stored state survives the buffers' growth (a resize since the last pass); a cold pass overwrites it below
  PM_CUDA(e->auc_price.grow_keep((size_t)W + 2, e->auc_price.n, e->stream)); PM_CUDA(e->auc_owner.grow_keep(W, e->auc_owner.n, e->stream));
  PM_CUDA(e->auc_assigned.grow_keep(D, e->auc_assigned.n, e->stream));
  PM_CUDA(e->auc_bid_max.ensure(W)); PM_CUDA(e->auc_winner.ensure(W)); PM_CUDA(e->auc_withdrawn.ensure(D));
  PM_CUDA(e->auc_active.ensure((size_t)2 * std::max<uint32_t>(D, 1))); PM_CUDA(e->auc_bid_w.ensure(D)); PM_CUDA(e->auc_bid_p.ensure(D));
  PM_CUDA(e->auc_flag.ensure((size_t)T + 1)); PM_CUDA(e->auc_gidx.ensure((size_t)T + 1));
  PM_CUDA(e->auc_theta.ensure(C)); PM_CUDA(e->auc_theta_w.ensure(C)); PM_CUDA(e->auc_cand.ensure((size_t)C * pm::kAucCache));
  PM_CUDA(e->auc_pool.ensure((size_t)C * pm::kAucPool)); PM_CUDA(e->auc_pool_bound_v.ensure(C)); PM_CUDA(e->auc_pool_bound_w.ensure(C));
  PM_CUDA(e->auc_walk_list.ensure(C)); PM_CUDA(e->auc_split_v.ensure(kScanGrid * 16)); PM_CUDA(e->auc_split_w.ensure(kScanGrid * 16));
  PM_CUDA(e->auc_split_ticket.ensure(kScanGrid));
  PM_CUDA(cudaMemsetAsync(e->auc_split_ticket.p, 0, kScanGrid * 4, e->stream));
  PM_CUDA(e->auc_split_first.ensure(kScanGrid)); PM_CUDA(e->auc_skip_key.ensure(std::max<uint32_t>(C, 1)));
  PM_CUDA(cudaMemsetAsync(e->auc_split_first.p, 0xFF, kScanGrid * 4, e->stream));
  PM_CUDA(cudaMemsetAsync(e->auc_skip_key.p, 0, (size_t)std::max<uint32_t>(C, 1) * 8, e->stream));
  PM_CUDA(e->auc_class_req.ensure(C)); PM_CUDA(e->auc_class_list.ensure(C)); PM_CUDA(e->auc_retry.ensure(D)); PM_CUDA(e->auc_fallback.ensure(D));
  PM_CUDA(e->auc_perm.ensure((size_t)W + 4)); PM_CUDA(e->auc_pos_of.ensure(W));
  PM_CUDA(e->auc_idx.ensure(std::max(W, D))); PM_CUDA(e->auc_wa_s.ensure(W)); PM_CUDA(e->auc_wb_s.ensure(W)); PM_CUDA(e->auc_price_s.ensure((size_t)W + 2));
  PM_CUDA(e->auc_ctl.ensure(1)); PM_CUDA(e->h_ctl.ensure(1));
  PM_CUDA(e->worker_group.ensure(W)); PM_CUDA(e->worker_ask.ensure(W)); PM_CUDA(e->members.ensure(std::max(W, T)));
  PM_CUDA(e->group_ask.ensure((size_t)T + 1)); PM_CUDA(e->group_off.ensure((size_t)T + 2));
  PM_CUDA(e->ask_best.ensure(T)); PM_CUDA(e->ask_count.ensure(T)); PM_CUDA(e->first_ask.ensure(W));
  PM_CUDA(cudaMemsetAsync(e->auc_ctl.p, 0, sizeof(pm::AuctionCtl), e->stream));
  // The table limits, read back before anything of the stored state is touched: a pass outside the integer domain is
  // refused and leaves the stored state as it was.  The same read-back tells whether (value, worker) sorts as one packed
  // 64-bit key (decided on the device, read by the kernels).
  pm::pm_auction_limits<<<std::max(1u, std::min(blocks_for(std::max(W, D), 256), 4u * e->sms)), 256, 0, e->stream>>>(e->wb.p, W, cap_b, D, e->auc_ctl.p);
  PM_LAUNCH_CHECK("pm_auction_limits");
  // (a warm pass: every price an ask kept was bid under its unchanged cap at eps = 1, every other price is 0, so the
  // bound on reachable costs is the cold one at eps = 1.  A warm repair keeps the stored prices of unowned workers too,
  // which an eps-scaled pass may have left at up to (K + 1) * S + eps_start: it is decided with eps_start.)
  pm::pm_auction_decide_packed<<<1, 1, 0, e->stream>>>(e->auc_ctl.p, W, D, e->auc_scale, warm && !repair ? 1 : e->auc_eps_start,
                                                       (uint32_t)e->tune_auction);
  PM_LAUNCH_CHECK("pm_auction_decide_packed");
  PM_CUDA(cudaMemcpyAsync(e->h_ctl.p, e->auc_ctl.p, sizeof(pm::AuctionCtl), cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  if (!auction_in_domain(e->h_ctl.p->max_ask_price, e->h_ctl.p->max_cap, e->auc_scale, e->auc_eps_start)) {
    *refused = true;
    return e->fail(PM_E_INVALID, "pm_match: (max ask_price + max cap + 2) * cost_scale + eps_start must stay below 2^61");
  }
  const bool packed_claim = e->h_ctl.p->packed_claim != 0;   // then no round launches pm_auction_claim at all
  const bool cost_packed = e->h_ctl.p->packed != 0;
  if (warm) {   // rows from n_kept on were cut off or added since the stored state: unowned, price 0
    if (W > n_kept) PM_CUDA(cudaMemsetAsync(e->auc_owner.p + n_kept, 0xFF, (size_t)(W - n_kept) * 4, e->stream));
    PM_CUDA(cudaMemsetAsync(e->auc_price.p + n_kept, 0, ((size_t)W + 2 - n_kept) * 8, e->stream));
  } else {
    PM_CUDA(cudaMemsetAsync(e->auc_price.p, 0, ((size_t)W + 2) * 8, e->stream));
  }
  PM_CUDA(cudaMemsetAsync(e->auc_price_s.p, 0, ((size_t)W + 2) * 8, e->stream));
  PM_CUDA(cudaMemsetAsync(e->auc_class_req.p, 0, (size_t)std::max<uint32_t>(C, 1) * 4, e->stream));
  PM_CUDA(e->auc_ckey.ensure(W)); PM_CUDA(e->auc_ckey_s.ensure(W));
  // a missing worker column is a column of zeros
  if (use_rep) {
    if (!e->have_rep) {
      PM_CUDA(e->reputation.ensure(std::max<size_t>(e->wa.n, 1)));
      PM_CUDA(cudaMemsetAsync(e->reputation.p, 0, std::max<size_t>(e->wa.n, 1) * 4, e->stream));
      e->have_rep = true;
    }
    PM_CUDA(e->auc_rep_s.ensure((size_t)W + 4));
    PM_CUDA(cudaMemsetAsync(e->auc_rep_s.p, 0, ((size_t)W + 4) * 4, e->stream));
  }
  pm::AuctionParams ap;
  ap.ev = eval_params(e);
  if (dem) ap.ev.asks = e->slot_row.p;
  ap.wa_s = e->auc_wa_s.p; ap.wb_s = e->auc_wb_s.p; ap.perm = e->auc_perm.p; ap.pos_of = e->auc_pos_of.p; ap.price_s = e->auc_price_s.p;
  ap.csort_s = reinterpret_cast<const unsigned long long*>(e->auc_ckey_s.p);
  ap.rep_s = use_rep ? e->auc_rep_s.p : nullptr; ap.min_rep = floor_b;
  ap.price_cap = cap_b; ap.price = e->auc_price.p; ap.owner = e->auc_owner.p; ap.assigned = e->auc_assigned.p;
  ap.withdrawn = e->auc_withdrawn.p; ap.active = e->auc_active.p; ap.n_asks = D; ap.bid_w = e->auc_bid_w.p; ap.bid_p = e->auc_bid_p.p;
  ap.bid_max = e->auc_bid_max.p; ap.winner = e->auc_winner.p; ap.scale = (long long)e->auc_scale;
  ap.class_of = e->auc_class_of.p; ap.class_rep = e->auc_class_rep.p; ap.class_req = e->auc_class_req.p;
  ap.cand = e->auc_cand.p; ap.theta = e->auc_theta.p; ap.theta_w = e->auc_theta_w.p;
  ap.pool = e->auc_pool.p; ap.pool_bound_v = e->auc_pool_bound_v.p; ap.pool_bound_w = e->auc_pool_bound_w.p;
  ap.walk_list = e->auc_walk_list.p; ap.split_bound_v = e->auc_split_v.p; ap.split_bound_w = e->auc_split_w.p; ap.split_ticket = e->auc_split_ticket.p; ap.split_first = e->auc_split_first.p;
  ap.skip_key = reinterpret_cast<unsigned long long*>(e->auc_skip_key.p);
  ap.class_list = e->auc_class_list.p; ap.retry = e->auc_retry.p; ap.fallback = e->auc_fallback.p; ap.ctl = e->auc_ctl.p;
  ap.dbg = (uint32_t)e->tune_auction;
  ap.pool_good = e->tune_auc_good > 0 ? (uint32_t)e->tune_auc_good : (uint32_t)pm::kAucPoolGood;
  ap.pool_extra = e->tune_auc_extra > 0 ? (uint32_t)e->tune_auc_extra : (uint32_t)pm::kAucPoolExtra;
  if (W) {
    pm::pm_fill_i64<<<std::min(blocks_for(W, 256), 8u * e->sms), 256, 0, e->stream>>>(e->auc_bid_max.p, pm::kAucNeg, W);
    PM_LAUNCH_CHECK("pm_fill_i64");
  }
  // Reverse rounds (PM_AUCTION_REVERSE, and the last stage of a warm repair): per round collect the bidders and the asks'
  // profits, one CTA per bid, (claim), apply, advance; batched into one CUDA graph per phase like the forward rounds, one
  // poll of the control block per batch.  (Set up here: a warm repair's raise runs on the same buffers before the rounds.)
  const bool rev_on = (reverse || repair) && T && W;
  pm::AuctionRev rv{};
  if (rev_on) {
    PM_CUDA(e->auc_rev_bidders.ensure(W)); PM_CUDA(e->auc_rev_offer_t.ensure(W)); PM_CUDA(e->auc_rev_offer_p.ensure(W));
    PM_CUDA(e->auc_rev_best.ensure(D)); PM_CUDA(e->auc_rev_win.ensure(D)); PM_CUDA(e->auc_rev_pi_s.ensure(D));
    PM_CUDA(e->auc_rev_cap_s.ensure(D)); PM_CUDA(e->auc_rev_cstart.ensure((size_t)C + 1));
    rv.bidders = e->auc_rev_bidders.p; rv.offer_t = e->auc_rev_offer_t.p; rv.offer_p = e->auc_rev_offer_p.p;
    rv.best = e->auc_rev_best.p; rv.win = e->auc_rev_win.p; rv.pi_s = e->auc_rev_pi_s.p; rv.cap_s = e->auc_rev_cap_s.p;
    rv.sorted = e->auc_sorted.p; rv.cls_s = e->auc_incl.p; rv.cstart = e->auc_rev_cstart.p;
    rv.rep = use_rep ? e->reputation.p : nullptr; rv.n_classes = C;
    pm::pm_auction_rev_classes<<<blocks_for(D, 256), 256, 0, e->stream>>>(e->auc_sorted.p, e->auc_incl.p, cap_b, D, C,
                                                                          e->auc_rev_cstart.p, e->auc_rev_cap_s.p);
    PM_LAUNCH_CHECK("pm_auction_rev_classes");
  }
  const bool rev_packed = cost_packed && !(e->tune_auction & 128);   // then no round launches pm_auction_rev_claim
  const unsigned g_rev = std::max(1u, std::min(blocks_for(std::max(W, D), 256), 8u * e->sms));
  const unsigned g_rev_bid = 4u * e->sms;   // 64 registers per thread (no spills): four resident CTAs per SM
  // Release (warm start, steps 2 and 3 of DESIGN 4): the initial release and price reset, then the closure — per
  // iteration C x |R_new| predicate evaluations and one compare per still-assigned ask, one poll of the control block.
  // A warm repair instead keeps every stored price and raises the changed rows (below).
  // Every reset happens here, before the first sort of the worker copy: within the rounds sort keys still only rise.
  uint64_t closure_evals = 0;
  uint32_t n_released = 0;
  if (repair) {
    // 1. the warm start's initial release, no price reset: a released worker is unowned at its stored price;
    // 2. R = the changed rows (R0, and every row from n_kept on), each raised to max(0, beta - 1) against the asks that
    //    still hold a worker, with their profits as the release left them (the collect writes them into pi_s; the
    //    bidder list it also makes is dropped: the reverse stage collects its own).  A raised price may be lower than
    //    the stored one, but it comes before the first sort of the worker copy, so sort keys still only rise within
    //    the forward rounds.
    PM_CUDA(e->auc_raised.ensure(std::max<uint32_t>(W, 1))); PM_CUDA(e->auc_mark.ensure(std::max<uint32_t>(W, 1)));
    PM_CUDA(e->auc_chg.ensure(std::max<size_t>(changed.size(), 1)));
    if (!changed.empty()) PM_CUDA(cudaMemcpyAsync(e->auc_chg.p, changed.data(), changed.size() * 4, cudaMemcpyHostToDevice, e->stream));
    ap.eps = 1;
    const unsigned g_seed = std::max(1u, std::min(blocks_for((size_t)D + changed.size(), 256), 8u * e->sms));
    pm::pm_auction_warm_seed<<<g_seed, 256, 0, e->stream>>>(ap, e->auc_chg.p, n_rows, e->auc_chg.p + n_rows, n_chg, n_kept);
    PM_LAUNCH_CHECK("pm_auction_warm_seed");
    if (rev_on) {
      const unsigned g_w = std::max(1u, std::min(blocks_for(W, 256), 8u * e->sms));
      PM_CUDA(cudaMemsetAsync(e->auc_mark.p, 0, (size_t)W * 4, e->stream));
      pm::pm_auction_warm_rows<<<g_w, 256, 0, e->stream>>>(ap, e->auc_chg.p, n_rows, n_kept, e->auc_raised.p, e->auc_mark.p);
      PM_LAUNCH_CHECK("pm_auction_warm_rows");
      pm::pm_auction_rev_collect<<<g_rev, 256, 0, e->stream>>>(ap, rv);
      PM_LAUNCH_CHECK("pm_auction_rev_collect");
      pm::pm_auction_repair_raise<<<g_rev_bid, pm::kAucThreads, 0, e->stream>>>(ap, rv, e->auc_raised.p);
      PM_LAUNCH_CHECK("pm_auction_repair_raise");
      PM_CUDA(cudaMemsetAsync(&e->auc_ctl.p->n_bid, 0, sizeof(uint32_t), e->stream));
    } else if (W) {   // no asks: nobody holds a worker, so every price ends at 0
      PM_CUDA(cudaMemsetAsync(e->auc_price.p, 0, (size_t)W * 8, e->stream));
    }
  } else if (warm) {
    PM_CUDA(e->auc_raised.ensure(std::max<uint32_t>(W, 1))); PM_CUDA(e->auc_mark.ensure(std::max<uint32_t>(W, 1)));
    PM_CUDA(e->auc_cmin.ensure(std::max<uint32_t>(C, 1))); PM_CUDA(e->auc_chg.ensure(std::max<size_t>(changed.size(), 1)));
    if (!changed.empty()) PM_CUDA(cudaMemcpyAsync(e->auc_chg.p, changed.data(), changed.size() * 4, cudaMemcpyHostToDevice, e->stream));
    ap.eps = 1;
    const unsigned g_seed = std::max(1u, std::min(blocks_for((size_t)D + changed.size(), 256), 8u * e->sms));
    pm::pm_auction_warm_seed<<<g_seed, 256, 0, e->stream>>>(ap, e->auc_chg.p, n_rows, e->auc_chg.p + n_rows, n_chg, n_kept);
    PM_LAUNCH_CHECK("pm_auction_warm_seed");
    if (W) {
      const unsigned g_w = std::max(1u, std::min(blocks_for(W, 256), 8u * e->sms));
      pm::pm_auction_warm_reset<<<g_w, 256, 0, e->stream>>>(ap, e->auc_raised.p, e->auc_mark.p);
      PM_LAUNCH_CHECK("pm_auction_warm_reset");
      pm::pm_auction_warm_rows<<<g_w, 256, 0, e->stream>>>(ap, e->auc_chg.p, n_rows, n_kept, e->auc_raised.p, e->auc_mark.p);
      PM_LAUNCH_CHECK("pm_auction_warm_rows");
    }
    const unsigned g_t = std::max(1u, std::min(blocks_for(D, 256), 8u * e->sms));
    const uint32_t kYChunk = 65535u * 256u;   // raised workers per launch of pm_auction_release_classes (grid.y limit)
    uint32_t lo = 0;
    for (;;) {
      PM_CUDA(cudaMemcpyAsync(e->h_ctl.p, e->auc_ctl.p, sizeof(pm::AuctionCtl), cudaMemcpyDeviceToHost, e->stream));
      PM_CUDA(cudaStreamSynchronize(e->stream));
      const uint32_t hi = e->h_ctl.p->n_raised;
      if (hi == lo || C == 0) break;
      PM_CUDA(cudaMemsetAsync(e->auc_cmin.p, 0xFF, (size_t)C * 4, e->stream));
      for (uint32_t s0 = lo; s0 < hi; s0 += kYChunk) {
        const uint32_t s1 = std::min(hi, s0 + kYChunk);
        pm::pm_auction_release_classes<<<dim3(C, (s1 - s0 + 255) / 256), 256, 0, e->stream>>>(
            ap, e->auc_raised.p, s0, s1, use_rep ? e->reputation.p : nullptr, e->auc_cmin.p);
        PM_LAUNCH_CHECK("pm_auction_release_classes");
      }
      pm::pm_auction_release_asks<<<g_t, 256, 0, e->stream>>>(ap, e->auc_cmin.p, e->auc_raised.p);
      PM_LAUNCH_CHECK("pm_auction_release_asks");
      closure_evals += (uint64_t)C * (hi - lo);
      lo = hi;
    }
    n_released = e->h_ctl.p->n_released;
  }
  // worker planes sorted by (ask_price * S + price, index): stable radix sort; redone as prices move (below)
  auto sort_workers = [&]() -> int {
    if (!W) return PM_OK;
    pm::pm_auction_cost_keys<<<blocks_for(W, 256), 256, 0, e->stream>>>(e->wb.p, e->auc_price.p, (long long)e->auc_scale, W, reinterpret_cast<unsigned long long*>(e->auc_ckey.p), e->auc_idx.p);
    PM_LAUNCH_CHECK("pm_auction_cost_keys");
    size_t tmp = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp, e->auc_ckey.p, e->auc_ckey_s.p, e->auc_idx.p, e->auc_perm.p, (int)W, 0, 64, e->stream);
    PM_CUDA(e->cub_tmp.ensure(tmp));
    PM_CUDA(cub::DeviceRadixSort::SortPairs(e->cub_tmp.p, tmp, e->auc_ckey.p, e->auc_ckey_s.p, e->auc_idx.p, e->auc_perm.p, (int)W, 0, 64, e->stream));
    pm::pm_auction_gather_sorted<<<blocks_for(W, 256), 256, 0, e->stream>>>(e->wa.p, e->wb.p, e->auc_perm.p, e->auc_price.p, W, e->auc_wa_s.p,
                                                                            e->auc_wb_s.p, e->auc_pos_of.p, e->auc_price_s.p,
                                                                            use_rep ? e->reputation.p : nullptr, use_rep ? e->auc_rep_s.p : nullptr);
    PM_LAUNCH_CHECK("pm_auction_gather_sorted");
    return PM_OK;
  };
  {
    const int rc = sort_workers();
    if (rc != PM_OK) return rc;
  }
  PM_CUDA(cudaMemsetAsync(e->auc_winner.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));

  const size_t smem = pm::kAucStages * sizeof(pm::AuctionStage) + sizeof(pm::AuctionMerge);
  PM_CUDA(cudaFuncSetAttribute(pm::pm_auction_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // fixed grids: every kernel strides over a list whose length it reads from the control block
  const unsigned g_scan = kScanGrid;
  const unsigned g_apply = std::max(1u, std::min(blocks_for(D, 256), e->sms));   // every CTA pays a fence + the ticket: one per SM at most
  const unsigned g_refill = std::max(1u, std::min(C, 8u * e->sms));   // 12 KB of shared memory per CTA: eight per SM
  const unsigned g_warp = std::max(1u, std::min(blocks_for(D, pm::kAucWarps), 8u * e->sms));
  const unsigned g_thr = std::max(1u, std::min(blocks_for(D, 256), 4u * e->sms));
  const uint32_t kBatch = 32;  // rounds launched between polls of the control block
  const uint32_t kResort = (e->tune_auction >> 8) ? (uint32_t)(e->tune_auction >> 8) : 4u;   // batches between re-sorts of the worker copy
  uint64_t eps = warm ? 1 : (e->auc_eps_start ? e->auc_eps_start : 1);   // a warm pass is one phase at eps = 1
  const uint32_t div = e->auc_eps_div < 2 ? 2 : e->auc_eps_div;
  const uint32_t kRevBatch = 16;   // reverse rounds launched between polls of the control block
  uint32_t n_phases = 0;
  auto reverse_stage = [&]() -> int {
    auto launch_rev = [&]() {
      for (uint32_t r = 0; r < kRevBatch; ++r) {
        pm::pm_auction_rev_collect<<<g_rev, 256, 0, e->stream>>>(ap, rv);
        pm::pm_auction_rev_bid<<<g_rev_bid, pm::kAucThreads, 0, e->stream>>>(ap, rv);
        if (!rev_packed) pm::pm_auction_rev_claim<<<g_rev, 256, 0, e->stream>>>(ap, rv);
        pm::pm_auction_rev_apply<<<g_rev, 256, 0, e->stream>>>(ap, rv);
        pm::pm_auction_rev_advance<<<1, 1, 0, e->stream>>>(e->auc_ctl.p);
      }
    };
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t graph_exec = nullptr;
    if (cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      launch_rev();
      if (cudaStreamEndCapture(e->stream, &graph) != cudaSuccess || cudaGraphInstantiate(&graph_exec, graph, 0) != cudaSuccess) {
        if (graph) cudaGraphDestroy(graph);
        graph = nullptr;
        graph_exec = nullptr;
      }
    }
    (void)cudaGetLastError();
    int rc = PM_OK;
    for (;;) {
      cudaError_t ce;
      if (graph_exec) ce = cudaGraphLaunch(graph_exec, e->stream);
      else { launch_rev(); ce = cudaGetLastError(); }
      if (ce == cudaSuccess) ce = cudaMemcpyAsync(e->h_ctl.p, e->auc_ctl.p, sizeof(pm::AuctionCtl), cudaMemcpyDeviceToHost, e->stream);
      if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
      if (ce != cudaSuccess) { rc = e->fail(PM_E_CUDA, std::string("pm_match: auction reverse rounds: ") + cudaGetErrorString(ce)); break; }
      if (e->h_ctl.p->rev_last == 0) break;
      if (e->h_ctl.p->rev_rounds > 50u * 1000u * 1000u) { rc = e->fail(PM_E_CUDA, "pm_match: auction reverse rounds did not terminate"); break; }
    }
    if (graph_exec) cudaGraphExecDestroy(graph_exec);
    if (graph) cudaGraphDestroy(graph);
    return rc;
  };
  bool first_phase = true;
  for (;;) {  // eps phases: assignment cleared, prices (and so the class caches' bounds) kept
    if (!warm) {   // a warm pass starts from the released state: every unassigned ask is active (withdrawn ones too)
      PM_CUDA(cudaMemsetAsync(e->auc_owner.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
      PM_CUDA(cudaMemsetAsync(e->auc_assigned.p, 0xFF, (size_t)std::max<uint32_t>(D, 1) * 4, e->stream));
    }
    PM_CUDA(cudaMemsetAsync(e->auc_withdrawn.p, 0, (size_t)std::max<uint32_t>(D, 1) * 4, e->stream));
    if (C && first_phase) {  // no cache yet (on every pass, warm or cold): "invalid" sends every class to a scan
      pm::pm_fill_i64<<<std::min(blocks_for(C, 256), 8u * e->sms), 256, 0, e->stream>>>(e->auc_theta.p, pm::kThetaInvalid, C);
      pm::pm_fill_i64<<<std::min(blocks_for(C, 256), 8u * e->sms), 256, 0, e->stream>>>(e->auc_pool_bound_v.p, pm::kThetaInvalid, C);
      PM_LAUNCH_CHECK("pm_fill_i64");
    }
    first_phase = false;
    ap.eps = (long long)eps;
    if (D) {
      pm::pm_auction_compact<<<blocks_for(D, 256), 256, 0, e->stream>>>(ap, D);
      PM_LAUNCH_CHECK("pm_auction_compact");
    }
    pm::pm_auction_advance<<<1, 1, 0, e->stream>>>(e->auc_ctl.p, 1);
    PM_LAUNCH_CHECK("pm_auction_advance");
    auto launch_rounds = [&]() {
      for (uint32_t r = 0; r < kBatch; ++r) {
        pm::pm_auction_bid_cached<<<g_warp, pm::kAucThreads, 0, e->stream>>>(ap, 0);
        pm::pm_auction_refill<<<g_refill, pm::kAucThreads, 0, e->stream>>>(ap);
        pm::pm_auction_scan<<<g_scan, pm::kAucThreads, smem, e->stream>>>(ap, 1);
        pm::pm_auction_bid_cached<<<g_warp, pm::kAucThreads, 0, e->stream>>>(ap, 1);
        pm::pm_auction_scan<<<g_scan, pm::kAucThreads, smem, e->stream>>>(ap, 0);
        if (!packed_claim) pm::pm_auction_claim<<<g_thr, 256, 0, e->stream>>>(ap);
        pm::pm_auction_apply<<<g_apply, 256, 0, e->stream>>>(ap);   // ... and the next round's active list, and the advance
      }
    };
    // a batch of rounds is one CUDA graph (the kernels are a few microseconds each: launch-bound otherwise);
    // a stream that cannot be captured (the legacy default stream) gets plain launches
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t graph_exec = nullptr;
    if (T && cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      launch_rounds();
      if (cudaStreamEndCapture(e->stream, &graph) != cudaSuccess || cudaGraphInstantiate(&graph_exec, graph, 0) != cudaSuccess) {
        if (graph) cudaGraphDestroy(graph);
        graph = nullptr;
        graph_exec = nullptr;
      }
    }
    (void)cudaGetLastError();
    int rc_rounds = PM_OK;
    uint32_t n_batches = 0;
    for (;;) {
      cudaError_t ce = cudaMemcpyAsync(e->h_ctl.p, e->auc_ctl.p, sizeof(pm::AuctionCtl), cudaMemcpyDeviceToHost, e->stream);
      if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
      if (ce != cudaSuccess) { rc_rounds = e->fail(PM_E_CUDA, std::string("pm_match: auction rounds: ") + cudaGetErrorString(ce)); break; }
      if (e->tune_auction & 4) {   // PM_TUNE_AUCTION=4: one line per batch of rounds
        static thread_local double t_prev = 0;
        timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
        const double now = ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
        std::fprintf(stderr, "auction batch: rounds=%u active=%u refills=%llu class_scans=%llu ask_scans=%llu evals=%llu dt_ms=%.2f\n", e->h_ctl.p->rounds,
                     e->h_ctl.p->n_active, e->h_ctl.p->n_refills, e->h_ctl.p->n_class_scans, e->h_ctl.p->n_ask_scans, e->h_ctl.p->evals, t_prev ? now - t_prev : 0.0);
        t_prev = now;
      }
      if (e->h_ctl.p->n_active == 0) break;
      if (e->h_ctl.p->rounds > 50u * 1000u * 1000u) { rc_rounds = e->fail(PM_E_CUDA, "pm_match: auction did not terminate"); break; }
      if (n_batches && n_batches % kResort == 0) {   // bid-up workers move back in the walk order
        const int rc = sort_workers();
        if (rc != PM_OK) { rc_rounds = rc; break; }
      }
      ++n_batches;
      if (graph_exec) ce = cudaGraphLaunch(graph_exec, e->stream);
      else { launch_rounds(); ce = cudaGetLastError(); }
      if (ce != cudaSuccess) { rc_rounds = e->fail(PM_E_CUDA, std::string("pm_match: auction rounds: ") + cudaGetErrorString(ce)); break; }
    }
    if (graph_exec) cudaGraphExecDestroy(graph_exec);
    if (graph) cudaGraphDestroy(graph);
    if (rc_rounds != PM_OK) return rc_rounds;
    ++n_phases;
    if (rev_on) {
      Timer trv(e, &e->stats.ms_build, e->stream);   // (auction mode builds no cost tile: ms_build is the reverse rounds)
      const int rc = reverse_stage();
      trv.stop();
      if (rc != PM_OK) return rc;
      // The class caches, pool bounds, skip keys and the worker copy's order rest on "prices only rise": a stage that
      // lowered a price leaves them to be rebuilt before the next phase's forward rounds (after the last phase nothing
      // reads them, and the next pass starts them afresh).
      if (e->h_ctl.p->rev_lowered && eps != 1) {
        if (C) {
          pm::pm_fill_i64<<<std::min(blocks_for(C, 256), 8u * e->sms), 256, 0, e->stream>>>(e->auc_theta.p, pm::kThetaInvalid, C);
          pm::pm_fill_i64<<<std::min(blocks_for(C, 256), 8u * e->sms), 256, 0, e->stream>>>(e->auc_pool_bound_v.p, pm::kThetaInvalid, C);
          PM_LAUNCH_CHECK("pm_fill_i64");
          PM_CUDA(cudaMemsetAsync(e->auc_skip_key.p, 0, (size_t)C * 8, e->stream));
        }
        PM_CUDA(cudaMemsetAsync(&e->auc_ctl.p->rev_lowered, 0, sizeof(uint32_t), e->stream));
        const int rs = sort_workers();
        if (rs != PM_OK) return rs;
      }
    }
    if (eps == 1) break;
    eps = std::max<uint64_t>(1, eps / div);
  }
  e->stats.n_rounds = e->h_ctl.p->rounds;
  if (repair) {   // (nothing after the seed counts releases or raised rows: the last poll has them)
    n_released = e->h_ctl.p->n_released;
    closure_evals = (uint64_t)C * e->h_ctl.p->n_raised;   // the raise: one bid's class evaluations per raised row
  }
  e->stats.evals = e->h_ctl.p->evals + closure_evals + (uint64_t)C * e->h_ctl.p->rev_bids;
  e->stats.n_tiles = (uint32_t)std::min<unsigned long long>(e->h_ctl.p->n_class_scans, 0xFFFFFFFFull);
  e->stats.n_fused_launches = (uint32_t)std::min<unsigned long long>(e->h_ctl.p->n_ask_scans, 0xFFFFFFFFull);
  e->stats.n_launches = e->h_ctl.p->rounds * (packed_claim ? 6u : 7u);
  e->stats.n_build_launches = (uint32_t)std::min<unsigned long long>(e->h_ctl.p->n_refills, 0xFFFFFFFFull);
  tm.stop();
  Timer tr(e, &e->stats.ms_resolve, e->stream);
  uint32_t G = 0, M = 0;
  if (dem) {
    const int rc = auction_emit_groups(e, &G, &M);
    if (rc != PM_OK) return rc;
  } else {
    // result: one solo group per assigned ask, ask order
    pm::pm_auction_flags<<<blocks_for((size_t)T + 1, 256), 256, 0, e->stream>>>(e->auc_assigned.p, T, e->auc_flag.p);
    PM_LAUNCH_CHECK("pm_auction_flags");
    {
      size_t tmp = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, tmp, e->auc_flag.p, e->auc_gidx.p, (int)(T + 1), e->stream);
      PM_CUDA(e->cub_tmp.ensure(tmp));
      PM_CUDA(cub::DeviceScan::ExclusiveSum(e->cub_tmp.p, tmp, e->auc_flag.p, e->auc_gidx.p, (int)(T + 1), e->stream));
    }
    PM_CUDA(cudaMemsetAsync(e->worker_group.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
    PM_CUDA(cudaMemsetAsync(e->worker_ask.p, 0xFF, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
    if (T) {
      pm::pm_auction_emit<<<blocks_for(T, 256), 256, 0, e->stream>>>(e->auc_assigned.p, e->auc_gidx.p, e->wb.p, T, e->worker_group.p,
                                                                      e->worker_ask.p, e->group_ask.p, e->group_off.p, e->members.p,
                                                                      e->ask_best.p, e->ask_count.p);
      PM_LAUNCH_CHECK("pm_auction_emit");
    }
    PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 17, e->auc_gidx.p + T, 4, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));
    G = M = e->h_scalars.p[17];
    PM_CUDA(cudaMemcpyAsync(e->group_off.p + G, e->h_scalars.p + 17, 4, cudaMemcpyHostToDevice, e->stream));
  }
  tr.stop();
  e->n_groups = G;
  e->n_assigned = M;
  if (e->cfg.flags & PM_CFG_TIMING) {
    PM_CUDA(cudaEventRecord(e->ev1, e->stream));
    PM_CUDA(cudaEventSynchronize(e->ev1));
    PM_CUDA(cudaEventElapsedTime(&e->stats.ms_total, e->ev0, e->ev1));
    e->resolve_timers();
  }
  // the stored state for the next warm start: prices, owners and assignment stay in their buffers
  e->auc_discard();
  e->auc_state = true;
  e->auc_state_w = e->auc_kept = W;
  e->auc_row_mark.assign(W, 0);
  e->auc_ask_mark.assign(T, 0);
  e->auc_cap_stored = e->cap_host;
  if (e->have_min_rep) e->auc_floor_stored = e->floor_host;
  else e->auc_floor_stored.assign(T, 0u);
  e->auc_last_warm = warm;
  e->auc_last_released = n_released;
  e->auc_last_phases = reverse || repair ? n_phases : 0u;
  e->auc_last_rev_rounds = reverse || repair ? e->h_ctl.p->rev_rounds : 0u;
  e->auc_last_rev_bids = reverse || repair ? e->h_ctl.p->rev_bids : 0u;
  e->matched = true;
  e->local_done = false;
  return PM_OK;
}

// The last auction pass: its prices, whether it started warm, how many asks its warm start released.
int pm_auction_state(pm_engine* e, int64_t* price, uint32_t* warm, uint32_t* n_released) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->auc_state) return e->fail(PM_E_STATE, "pm_auction_state: no auction pass since the engine's tables were last replaced");
  PM_CUDA(cudaSetDevice(e->device));
  if (price && e->auc_state_w) {
    PM_CUDA(cudaMemcpyAsync(price, e->auc_price.p, (size_t)e->auc_state_w * 8, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));
  }
  if (warm) *warm = e->auc_last_warm ? 1u : 0u;
  if (n_released) *n_released = e->auc_last_released;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// The last auction pass's eps phases, reverse rounds and reverse bids (all 0 for a pass without PM_AUCTION_REVERSE).
int pm_auction_reverse_stats(pm_engine* e, uint32_t* n_phases, uint32_t* n_reverse_rounds, uint64_t* n_reverse_bids) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->auc_state) return e->fail(PM_E_STATE, "pm_auction_reverse_stats: no auction pass since the engine's tables were last replaced");
  if (n_phases) *n_phases = e->auc_last_phases;
  if (n_reverse_rounds) *n_reverse_rounds = e->auc_last_rev_rounds;
  if (n_reverse_bids) *n_reverse_bids = e->auc_last_rev_bids;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// pm_get_stats keeps reporting the last pass: the launch checks of a certificate or a restore count into e->stats,
// which is put back on return
struct KeepStats {
  pm_engine* e;
  pm_stats saved;
  ~KeepStats() { e->stats = saved; }
};

// The certificate's kernels (pm_auction_cert.cuh) over the prices and assignment given (device, [W] and [D]), into the
// certificate's private scratch: one sweep over every pair, then one pass over the asks and one over the workers.
// Enqueued only; *c gets the parameters the launches took.
static int cert_launch(pm_engine* e, const long long* price, const uint32_t* assigned, pm::CertParams* out) {
  const uint32_t W = e->n_workers, T = e->n_asks;
  if (!e->have_bits) {   // as an auction pass: no model table is one all-ones word
    PM_CUDA(e->bits.ensure(1));
    PM_CUDA(cudaMemsetAsync(e->bits.p, 0xFF, 4, e->stream));
    e->words = 1;
  }
  const bool dem = !e->demand.empty();
  const uint32_t D = e->n_slots();
  PM_CUDA(e->cert_min.ensure(std::max<uint32_t>(T, 1))); PM_CUDA(e->cert_ok.ensure(std::max<uint32_t>(std::max(T, D), 1)));
  PM_CUDA(e->cert_bound.ensure(std::max<uint32_t>(T, 1))); PM_CUDA(e->cert_own.ensure(std::max<uint32_t>(W, 1)));
  PM_CUDA(e->cert_acc.ensure(pm::kCertAccWords)); PM_CUDA(e->h_cert_acc.ensure(pm::kCertAccWords));
  PM_CUDA(cudaMemsetAsync(e->cert_min.p, 0xFF, (size_t)std::max<uint32_t>(T, 1) * 8, e->stream));
  PM_CUDA(cudaMemsetAsync(e->cert_own.p, 0, (size_t)std::max<uint32_t>(W, 1) * 4, e->stream));
  PM_CUDA(cudaMemsetAsync(e->cert_acc.p, 0, pm::kCertAccWords * 8, e->stream));
  pm::CertParams& c = *out;
  c.price = price;
  c.rep = e->have_min_rep && e->have_rep ? e->reputation.p : nullptr;
  c.cap = e->price_cap.p;
  c.floor = e->have_min_rep ? e->ask_min_rep.p : nullptr;
  c.assigned = assigned;
  c.row_min = reinterpret_cast<unsigned long long*>(e->cert_min.p);
  c.held_ok = e->cert_ok.p;
  c.own = e->cert_own.p;
  c.ask_bound = e->cert_bound.p;
  c.acc = reinterpret_cast<unsigned long long*>(e->cert_acc.p);
  c.scale = e->auc_scale;
  c.n_workers = W;
  c.n_asks = T;
  // With demands the assignment is per slot: the sweep runs per ask with no holds, and pm_auction_cert_slots checks
  // them instead of pm_auction_cert_asks (held_ok then per slot).  The slot table it builds stays in slot_ask.
  pm::CertParams cs = c;
  if (dem) {
    PM_CUDA(e->cert_none.ensure(std::max<uint32_t>(T, 1)));
    PM_CUDA(cudaMemsetAsync(e->cert_none.p, 0xFF, (size_t)std::max<uint32_t>(T, 1) * 4, e->stream));
    cs.assigned = e->cert_none.p;
  }
  if (T && W) {   // the fused pass's predicate variant (pm_match, PM_PATH_FUSED)
    pm::EvalParams p;
    int bits_mode = 0;
    bool fast = false;
    const int rc = pick_predicate(e, &p, &bits_mode, &fast);
    if (rc != PM_OK) return rc;
    const uint32_t rows_per_launch = 65535u * pm::kEvalRows;
    for (uint32_t t0 = 0; t0 < T; t0 += rows_per_launch) {
      const uint32_t nt = std::min(rows_per_launch, T - t0);
      const dim3 grid(blocks_for(W, pm::kEvalCols), blocks_for(nt, pm::kEvalRows));
#define PM_CERT_CASE(B, F) pm::pm_auction_cert_sweep<B, F><<<grid, pm::kEvalThreads, 0, e->stream>>>(p, cs, t0, nt)
      if (fast) { if (bits_mode == 2) PM_CERT_CASE(2, true); else if (bits_mode == 1) PM_CERT_CASE(1, true); else PM_CERT_CASE(0, true); }
      else { if (bits_mode == 2) PM_CERT_CASE(2, false); else if (bits_mode == 1) PM_CERT_CASE(1, false); else PM_CERT_CASE(0, false); }
#undef PM_CERT_CASE
      PM_LAUNCH_CHECK("pm_auction_cert_sweep");
    }
  }
  if (dem && T) {
    PM_CUDA(e->slot_ask.ensure(D)); PM_CUDA(e->slot_row.ensure(D)); PM_CUDA(e->slot_cap.ensure(D));
    pm::pm_auction_slot_table<<<std::min(blocks_for(D, 256), 8u * e->sms), 256, 0, e->stream>>>(
        e->dem_off.p, T, D, e->asks.p, e->price_cap.p, nullptr, e->slot_ask.p, e->slot_row.p, e->slot_cap.p, nullptr);
    PM_LAUNCH_CHECK("pm_auction_slot_table");
    pm::pm_auction_cert_slots<<<std::min(blocks_for(D, 256), 4u * e->sms), 256, 0, e->stream>>>(c, eval_params(e), e->slot_ask.p, D);
    PM_LAUNCH_CHECK("pm_auction_cert_slots");
  } else if (T) {
    pm::pm_auction_cert_asks<<<std::min(blocks_for(T, 256), 4u * e->sms), 256, 0, e->stream>>>(c, e->wb.p);
    PM_LAUNCH_CHECK("pm_auction_cert_asks");
  }
  if (W) {
    pm::pm_auction_cert_workers<<<std::min(blocks_for(W, 256), 4u * e->sms), 256, 0, e->stream>>>(c, e->wb.p);
    PM_LAUNCH_CHECK("pm_auction_cert_workers");
  }
  return PM_OK;
}

// The certificate of the stored auction state (pm_auction_cert.cuh) on private buffers; one synchronisation.  Reads the
// stored state and the tables only: the result buffers, pm_stats, the table version and the warm-start bookkeeping stay
// as they are.
int pm_auction_certificate(pm_engine* e, pm_auction_cert* out, int64_t* ask_bound) try {
  if (!e || !out) return e ? e->fail(PM_E_INVALID, "pm_auction_certificate: null output") : PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->auc_state) return e->fail(PM_E_STATE, "pm_auction_certificate: no auction pass since the engine's tables were last replaced");
  const uint32_t W = e->n_workers, T = e->n_asks;
  if (W != e->auc_state_w) return e->fail(PM_E_STATE, "pm_auction_certificate: the worker table was resized since the last auction pass");
  if (e->auc_asks_resized) return e->fail(PM_E_STATE, "pm_auction_certificate: the ask table was resized since the last auction pass");
  if (e->auc_workers_spliced)
    return e->fail(PM_E_STATE, "pm_auction_certificate: workers were removed or inserted since the last auction pass");
  if (e->max_pattern_row > e->n_patterns || (e->max_pattern_row && !e->have_bits))
    return e->fail(PM_E_STATE, "pm_auction_certificate: an ask references a model pattern missing from the model table");
  if (e->n_off) return e->fail(PM_E_UNSUPPORTED, "pm_auction_certificate: disabled asks");
  KeepStats keep_stats{e, e->stats};   // before the rows go to the auction's form: that launch is no pass's either
  {
    const int rc = use_ask_form(e, true);
    if (rc != PM_OK) return rc;
  }
  PM_CUDA(cudaSetDevice(e->device));
  if (ask_bound) PM_CUDA(e->h_cert_bound.ensure(std::max<uint32_t>(T, 1)));
  pm::CertParams c;
  {
    const int rc = cert_launch(e, e->auc_price.p, e->auc_assigned.p, &c);
    if (rc != PM_OK) return rc;
  }
  PM_CUDA(cudaMemcpyAsync(e->h_cert_acc.p, e->cert_acc.p, pm::kCertAccWords * 8, cudaMemcpyDeviceToHost, e->stream));
  if (ask_bound && T) PM_CUDA(cudaMemcpyAsync(e->h_cert_bound.p, e->cert_bound.p, (size_t)T * 8, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  const uint64_t* h = e->h_cert_acc.p;
  uint32_t K = 0;
  for (uint32_t t = 0; t < T; ++t) K = std::max(K, e->cap_host[t]);
  if (!auction_in_domain((uint32_t)h[pm::kCertMaxAskPrice], K, e->auc_scale, e->auc_eps_start))
    return e->fail(PM_E_INVALID, "pm_auction_certificate: (max ask_price + max cap + 2) * cost_scale + eps_start must stay below 2^61");
  using i128 = __int128;
  auto join = [&](int i) { return (i128)h[i] + ((i128)h[i + 1] << 32); };
  const i128 cost = join(pm::kCertCostLo), bound = join(pm::kCertRowLo) - join(pm::kCertPriceLo), gap = cost - bound;
  const i128 free_sum = join(pm::kCertFreeLo);
  pm_auction_cert r{};
  r.cost_hi = (int64_t)(cost >> 64); r.cost_lo = (uint64_t)cost;
  r.bound_hi = (int64_t)(bound >> 64); r.bound_lo = (uint64_t)bound;
  r.gap_hi = (int64_t)(gap >> 64); r.gap_lo = (uint64_t)gap;
  r.n_held = (uint32_t)h[pm::kCertHeld];
  r.n_bad_holds = (uint32_t)h[pm::kCertBadHolds];
  r.n_shared = (uint32_t)h[pm::kCertShared];
  r.n_priced_unowned = (uint32_t)h[pm::kCertFree];
  r.n_slack_over = (uint32_t)h[pm::kCertSlackOver];
  r.max_slack = T ? (int64_t)(h[pm::kCertMaxSlack] ^ 0x8000000000000000ull) : 0;
  r.priced_unowned_lo = (uint64_t)free_sum;
  r.priced_unowned_hi = (uint64_t)(free_sum >> 64);
  r.evals = (uint64_t)T * W;
  *out = r;
  if (ask_bound && T) std::memcpy(ask_bound, e->h_cert_bound.p, (size_t)T * 8);
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// After a worker splice the stored assignment marks a hold on a removed row kCutHold (pm_splice_worker_holds): it
// is released by the next warm pass, and exported as PM_NONE
static void cut_holds_read_none(uint32_t* assigned, uint32_t n) {
  for (uint32_t s = 0; s < n; ++s)
    if (assigned[s] == pm::kCutHold) assigned[s] = PM_NONE;
}

// The stored state's assignment over the current asks (remapped by pm_update_asks / pm_resize_asks like the state itself)
int pm_auction_assignment(pm_engine* e, uint32_t* assigned) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->auc_state) return e->fail(PM_E_STATE, "pm_auction_assignment: no auction pass since the engine's tables were last replaced");
  if (e->n_asks && !assigned) return e->fail(PM_E_INVALID, "pm_auction_assignment: null output");
  if (!e->demand.empty()) return e->fail(PM_E_UNSUPPORTED, "pm_auction_assignment: an ask demand above 1 (the format is one worker per ask)");
  PM_CUDA(cudaSetDevice(e->device));
  if (e->n_asks) {
    PM_CUDA(cudaMemcpyAsync(assigned, e->auc_assigned.p, (size_t)e->n_asks * 4, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));
    if (e->auc_workers_spliced) cut_holds_read_none(assigned, e->n_asks);
  }
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// The stored state's assignment per slot over the current slot table (prime_match.h "Auction state restore per
// slot"): the stored array itself, which every remap of the asks and demands keeps per slot.  *n_slots in/out; a size
// query with assigned NULL.
int pm_auction_slot_assignment(pm_engine* e, uint32_t* assigned, uint32_t* n_slots) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!n_slots) return e->fail(PM_E_INVALID, "pm_auction_slot_assignment: null n_slots");
  if (!e->auc_state) return e->fail(PM_E_STATE, "pm_auction_slot_assignment: no auction pass since the engine's tables were last replaced");
  const uint32_t D = e->n_slots();
  if (!assigned) {
    *n_slots = D;
    return PM_OK;
  }
  if (*n_slots != D) {
    *n_slots = D;
    return e->fail(PM_E_INVALID, "pm_auction_slot_assignment: n_slots is not the number of slots (written back)");
  }
  PM_CUDA(cudaSetDevice(e->device));
  if (D) {
    PM_CUDA(cudaMemcpyAsync(assigned, e->auc_assigned.p, (size_t)D * 4, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaStreamSynchronize(e->stream));
    if (e->auc_workers_spliced) cut_holds_read_none(assigned, D);
  }
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// A caller's auction state, audited on the device and made the stored state (prime_match.h "Auction state restore"),
// for pm_auction_restore (per_slot false: one entry per ask, refused under demands) and pm_auction_restore_slots (one
// entry per slot; without demands the slots are the asks).  Called with the engine's lock held.  Every host check
// first, then the caller's arrays go to staging buffers and the certificate's kernels run over them (with demands
// cert_launch builds the slot table and checks the holds per slot); the audit (pm_auction_restore_asks over the asks or
// the slots, pm_auction_restore_workers) writes staging buffers too.  One synchronisation, the domain check on the
// sweep's largest ask price, and only then the stored state is overwritten, by device copies.
static int auction_restore(pm_engine* e, const char* fn, bool per_slot, const int64_t* price, uint32_t n_workers,
                           const uint32_t* assigned, uint32_t n, pm_auction_restore_report* report) {
  auto refuse = [&](pm_status st, const char* why) { return e->fail(st, std::string(fn) + ": " + why); };
  if ((n_workers && !price) || (n && !assigned)) return refuse(PM_E_INVALID, "null");
  if (!e->have_workers || !e->have_asks) return refuse(PM_E_STATE, "worker and ask tables must be set first");
  if (!e->have_caps) return refuse(PM_E_STATE, "no price caps (pm_set_ask_price_caps)");
  if (e->max_pattern_row > e->n_patterns || (e->max_pattern_row && !e->have_bits))
    return refuse(PM_E_STATE, "an ask references a model pattern missing from the model table");
  if (e->cfg.shard_count || e->comm) return refuse(PM_E_UNSUPPORTED, "auction mode is single-GPU");
  if (e->n_off) return refuse(PM_E_UNSUPPORTED, "disabled asks");
  if (!per_slot && !e->demand.empty()) return refuse(PM_E_UNSUPPORTED, "an ask demand above 1 (the format is one worker per ask)");
  const bool dem = !e->demand.empty();
  const uint32_t W = e->n_workers, T = e->n_asks, D = e->n_slots();
  if (n_workers != W || n != D)
    return refuse(PM_E_INVALID, per_slot ? "one price per worker and one entry per slot" : "one price per worker and one entry per ask");
  for (uint32_t s = 0; s < D; ++s)
    if (assigned[s] != PM_NONE && assigned[s] >= W) return refuse(PM_E_INVALID, "assigned worker out of range");
  // every price the warm pass and the repair can start from: (K + 1) * S + max(E, 1), in 128 bits
  uint32_t K = 0;
  for (uint32_t t = 0; t < T; ++t) K = std::max(K, e->cap_host[t]);
  const unsigned __int128 p_max = ((unsigned __int128)K + 1u) * e->auc_scale + std::max<uint64_t>(e->auc_eps_start, 1);
  for (uint32_t w = 0; w < W; ++w)
    if (price[w] < 0 || (unsigned __int128)price[w] > p_max)
      return refuse(PM_E_INVALID, "price outside [0, (max cap + 1) * cost_scale + eps_start]");
  KeepStats keep_stats{e, e->stats};   // before the rows go to the auction's form: that launch is no pass's either
  {
    const int rc = use_ask_form(e, true);
    if (rc != PM_OK) return rc;
  }
  PM_CUDA(cudaSetDevice(e->device));
  // the stored buffers at their pass sizes, their contents kept (a refusal below leaves the stored state as it was)
  PM_CUDA(e->auc_price.grow_keep((size_t)W + 2, e->auc_price.n, e->stream)); PM_CUDA(e->auc_owner.grow_keep(W, e->auc_owner.n, e->stream));
  PM_CUDA(e->auc_assigned.grow_keep(D, e->auc_assigned.n, e->stream));
  PM_CUDA(e->rst_price.ensure(std::max<uint32_t>(W, 1))); PM_CUDA(e->rst_owner.ensure(std::max<uint32_t>(W, 1)));
  PM_CUDA(e->rst_assigned.ensure(std::max<uint32_t>(D, 1))); PM_CUDA(e->rst_kept.ensure(std::max<uint32_t>(D, 1)));
  PM_CUDA(e->rst_acc.ensure(pm::kRstAccWords)); PM_CUDA(e->h_rst_acc.ensure(pm::kRstAccWords));
  if (W) PM_CUDA(cudaMemcpyAsync(e->rst_price.p, price, (size_t)W * 8, cudaMemcpyHostToDevice, e->stream));
  if (D) PM_CUDA(cudaMemcpyAsync(e->rst_assigned.p, assigned, (size_t)D * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaMemsetAsync(e->rst_acc.p, 0, pm::kRstAccWords * 8, e->stream));
  pm::CertParams c;
  {
    const int rc = cert_launch(e, e->rst_price.p, e->rst_assigned.p, &c);
    if (rc != PM_OK) return rc;
  }
  if (D) {
    pm::pm_auction_restore_asks<<<std::min(blocks_for(D, 256), 4u * e->sms), 256, 0, e->stream>>>(
        c, e->wb.p, dem ? e->slot_ask.p : nullptr, D, e->rst_kept.p, reinterpret_cast<unsigned long long*>(e->rst_acc.p));
    PM_LAUNCH_CHECK("pm_auction_restore_asks");
  }
  if (W) {
    pm::pm_auction_restore_workers<<<std::min(blocks_for(W, 256), 8u * e->sms), 256, 0, e->stream>>>(e->cert_own.p, W, e->rst_owner.p);
    PM_LAUNCH_CHECK("pm_auction_restore_workers");
  }
  PM_CUDA(cudaMemcpyAsync(e->h_cert_acc.p, e->cert_acc.p, pm::kCertAccWords * 8, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->h_rst_acc.p, e->rst_acc.p, pm::kRstAccWords * 8, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  if (!auction_in_domain((uint32_t)e->h_cert_acc.p[pm::kCertMaxAskPrice], K, e->auc_scale, e->auc_eps_start))
    return refuse(PM_E_INVALID, "(max ask_price + max cap + 2) * cost_scale + eps_start must stay below 2^61");
  // commit: from here a failure leaves a half-copied state, which is dropped.  auc_discard also clears the demand
  // bookkeeping (auc_dem_kept): every slot of the restored state may carry a hold.
  e->auc_discard();
  if (W) {
    PM_CUDA(cudaMemcpyAsync(e->auc_price.p, e->rst_price.p, (size_t)W * 8, cudaMemcpyDeviceToDevice, e->stream));
    PM_CUDA(cudaMemcpyAsync(e->auc_owner.p, e->rst_owner.p, (size_t)W * 4, cudaMemcpyDeviceToDevice, e->stream));
  }
  PM_CUDA(cudaMemsetAsync(e->auc_price.p + W, 0, 2 * 8, e->stream));
  if (D) PM_CUDA(cudaMemcpyAsync(e->auc_assigned.p, e->rst_kept.p, (size_t)D * 4, cudaMemcpyDeviceToDevice, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  // the bookkeeping of a pass that just ran on the current tables: nothing changed since, nothing to report
  e->auc_state = true;
  e->auc_state_w = e->auc_kept = W;
  e->auc_row_mark.assign(W, 0);
  e->auc_ask_mark.assign(T, 0);
  e->auc_cap_stored = e->cap_host;
  if (e->have_min_rep) e->auc_floor_stored = e->floor_host;
  else e->auc_floor_stored.assign(T, 0u);
  e->auc_last_warm = false;
  e->auc_last_released = 0;
  e->auc_last_phases = e->auc_last_rev_rounds = 0;
  e->auc_last_rev_bids = 0;
  if (report) {
    const uint64_t* h = e->h_rst_acc.p;
    report->n_held = (uint32_t)h[pm::kRstHeld];
    report->n_dropped_bad = (uint32_t)h[pm::kRstBad];
    report->n_dropped_shared = (uint32_t)h[pm::kRstShared];
    report->n_dropped_slack = (uint32_t)h[pm::kRstSlack];
    report->evals = (uint64_t)T * W;   // the sweep is per ask with demands too
  }
  return PM_OK;
}

int pm_auction_restore(pm_engine* e, const int64_t* price, uint32_t n_workers, const uint32_t* assigned, uint32_t n_asks,
                       pm_auction_restore_report* report) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  return auction_restore(e, "pm_auction_restore", false, price, n_workers, assigned, n_asks, report);
} catch (...) { return pm_guard_rc(); }

// With demands d: what pm_auction_restore does on the twin engine (row t repeated d[t] times), `assigned` the twin's
// per-ask assignment; without demands exactly pm_auction_restore.
int pm_auction_restore_slots(pm_engine* e, const int64_t* price, uint32_t n_workers, const uint32_t* assigned, uint32_t n_slots,
                             pm_auction_restore_report* report) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  return auction_restore(e, "pm_auction_restore_slots", true, price, n_workers, assigned, n_slots, report);
} catch (...) { return pm_guard_rc(); }

int pm_set_ask_price_caps(pm_engine* e, const uint32_t* price_cap, uint32_t n_asks) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks || n_asks != e->n_asks) return e->fail(PM_E_INVALID, "pm_set_ask_price_caps: one cap per ask, after pm_set_asks");
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->price_cap.ensure(n_asks));
  if (n_asks) PM_CUDA(cudaMemcpyAsync(e->price_cap.p, price_cap, (size_t)n_asks * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  e->cap_host.assign(price_cap, price_cap + n_asks);   // a warm start finds the changed caps by a diff
  e->have_caps = true;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// `reputation` worker column and the per-ask floor on it (north-star extension; PM_MODE_AUCTION only)
int pm_set_worker_reputation(pm_engine* e, const uint32_t* reputation, uint32_t first, uint32_t n) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  ++e->table_version;
  if (!e->have_workers) return e->fail(PM_E_STATE, "pm_set_worker_reputation: no worker table");
  if ((uint64_t)first + n > e->n_workers) return e->fail(PM_E_INVALID, "pm_set_worker_reputation: range");
  if (n && !reputation) return e->fail(PM_E_INVALID, "pm_set_worker_reputation: null");
  PM_CUDA(cudaSetDevice(e->device));
  if (!e->have_rep) {
    PM_CUDA(e->reputation.ensure(std::max<size_t>(e->wa.n, 1)));
    PM_CUDA(cudaMemsetAsync(e->reputation.p, 0, std::max<size_t>(e->wa.n, 1) * 4, e->stream));
  }
  e->auc_mark_rows(first, n);   // the auction reads reputation: for its warm start these rows changed
  if (n) PM_CUDA(cudaMemcpyAsync(e->reputation.p + first, reputation, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  e->have_rep = true;
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_set_ask_min_reputation(pm_engine* e, const uint32_t* min_reputation, uint32_t n_asks) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks || n_asks != e->n_asks) return e->fail(PM_E_INVALID, "pm_set_ask_min_reputation: one floor per ask, after pm_set_asks");
  if (n_asks && !min_reputation) return e->fail(PM_E_INVALID, "pm_set_ask_min_reputation: null");
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(e->ask_min_rep.ensure(std::max<uint32_t>(n_asks, 1)));
  if (n_asks) PM_CUDA(cudaMemcpyAsync(e->ask_min_rep.p, min_reputation, (size_t)n_asks * 4, cudaMemcpyHostToDevice, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  e->floor_host.assign(min_reputation, min_reputation + n_asks);
  e->have_min_rep = true;
  e->auc_classes_valid = false;   // the floor is part of an ask's class
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// Ask demands (north-star extension; PM_MODE_AUCTION only, prime_match.h "Auction demands").  Every check comes first
// (a refusal changes nothing); a stored auction state is then remapped slot by slot on the device.
int pm_set_ask_demand(pm_engine* e, const uint32_t* demand, uint32_t n_asks) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_asks) return e->fail(PM_E_STATE, "pm_set_ask_demand: no ask table");
  if (n_asks != e->n_asks) return e->fail(PM_E_INVALID, "pm_set_ask_demand: one demand per ask");
  if (n_asks && !demand) return e->fail(PM_E_INVALID, "pm_set_ask_demand: null");
  const uint32_t T = n_asks;
  std::vector<uint32_t> off((size_t)T + 1, 0u);
  bool same = true;
  for (uint32_t t = 0; t < T; ++t) {
    if (demand[t] == 0) return e->fail(PM_E_INVALID, "pm_set_ask_demand: a demand of 0");
    const uint64_t s = (uint64_t)off[t] + demand[t];
    if (s >= (1u << 30)) return e->fail(PM_E_INVALID, "pm_set_ask_demand: the demands' total reaches 2^30");
    off[t + 1] = (uint32_t)s;
    same = same && demand[t] == (e->demand.empty() ? 1u : e->demand[t]);
  }
  if (same) return PM_OK;
  ++e->table_version;
  PM_CUDA(cudaSetDevice(e->device));
  if (e->auc_state) {
    const int rc = [&]() -> int {
      const uint32_t D_old = e->n_slots(), D_new = off[T];
      std::vector<uint32_t> old_off((size_t)T + 1);
      for (uint32_t t = 0; t <= T; ++t) old_off[t] = e->slot0(t);
      PM_CUDA(e->dem_off_old.ensure((size_t)T + 1)); PM_CUDA(e->dem_off.ensure((size_t)T + 1));
      PM_CUDA(e->auc_assigned_tmp.ensure(std::max<uint32_t>(D_new, 1)));
      PM_CUDA(cudaMemcpyAsync(e->dem_off_old.p, old_off.data(), old_off.size() * 4, cudaMemcpyHostToDevice, e->stream));
      PM_CUDA(cudaMemcpyAsync(e->dem_off.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice, e->stream));
      PM_CUDA(cudaMemsetAsync(e->auc_assigned_tmp.p, 0xFF, (size_t)std::max<uint32_t>(D_new, 1) * 4, e->stream));
      PM_CUDA(cudaMemsetAsync(e->counters.p + 17, 0, 4, e->stream));
      if (D_old) {
        pm::pm_auction_slot_remap<<<std::min(blocks_for(D_old, 256), 8u * e->sms), 256, 0, e->stream>>>(
            e->dem_off_old.p, e->dem_off.p, nullptr, T, D_old, e->auc_assigned.p, e->auc_assigned_tmp.p, e->auc_owner.p,
            e->auc_kept, e->counters.p + 17);
        PM_LAUNCH_CHECK("pm_auction_slot_remap");
      }
      PM_CUDA(cudaMemcpyAsync(e->h_scalars.p + 17, e->counters.p + 17, 4, cudaMemcpyDeviceToHost, e->stream));
      PM_CUDA(cudaStreamSynchronize(e->stream));   // (old_off and off are locals)
      std::swap(e->auc_assigned, e->auc_assigned_tmp);
      e->auc_removed_held += e->h_scalars.p[17];
      if (e->auc_dem_kept.empty())
        for (uint32_t t = 0; t < T; ++t) e->auc_dem_kept.push_back(old_off[t + 1] - old_off[t]);
      for (uint32_t t = 0; t < T; ++t) e->auc_dem_kept[t] = std::min(e->auc_dem_kept[t], demand[t]);
      return PM_OK;
    }();
    if (rc != PM_OK) {
      e->auc_discard();
      return rc;
    }
  }
  e->demand.assign(demand, demand + T);
  e->dem_off_h = std::move(off);
  e->auc_classes_valid = false;   // the auction's classes are built over the slots
  e->matched = e->local_done = false;
  return upload_demand(e);
} catch (...) { return pm_guard_rc(); }

int pm_set_auction_params(pm_engine* e, uint64_t cost_scale, uint64_t eps_start, uint32_t eps_div) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (cost_scale >= (1ull << 61) || eps_start >= (1ull << 61))   // outside the domain whatever the tables; changes nothing
    return e->fail(PM_E_INVALID, "pm_set_auction_params: cost_scale and eps_start must stay below 2^61");
  e->auc_discard();
  e->auc_scale = cost_scale ? cost_scale : 1;
  e->auc_eps_start = eps_start ? eps_start : 1;
  e->auc_eps_div = eps_div < 2 ? 2 : eps_div;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// The one data-path exchange of a sharded pass (SURVEY 8e): every rank packs {per-ask (min cost, argmin) and feasible
// count over its workers, first feasible ask of its own workers} into one buffer, ONE all-gather over NVLink moves
// them, and every rank folds the contributions into the same global arrays.  Enqueued on the engine's stream: no host
// synchronisation, nothing but NCCL's kernel between the evaluation and the resolution sweep.
// Under PM_INCREMENTAL every rank decides full or incremental for its own range (match_local_locked: its own written
// rows against the cutoff), so in one pass some ranks may evaluate their range in full while others walk a few rows.
// Either way each rank's range of first_ask is exact, and every rank makes this same single all-gather, so the
// collective sequence of the ranks never diverges.  Under PM_NO_ASK_STATS ask_best / ask_count are INF / 0 on every
// rank and the fold keeps them so.
static int exchange_locked(pm_engine* e) {
  const NcclApi& nccl = nccl_api();
  if (!nccl.ok) return e->fail(PM_E_UNSUPPORTED, nccl.err);
  const uint32_t W = e->n_workers, T = e->n_asks, n = e->comm->n_ranks;
  uint32_t w0 = 0, nw = 0;
  e->shard(&w0, &nw);
  const uint32_t per = (uint32_t)(((uint64_t)W + n - 1) / n);
  const size_t stride = (((size_t)T * 12 + (size_t)per * 4) + 15) & ~(size_t)15;
  PM_CUDA(e->xchg_send.ensure(stride));
  PM_CUDA(e->xchg_recv.ensure(stride * n));
  Timer tm(e, &e->stats.ms_exchange, e->stream);
  const size_t work = std::max<size_t>(std::max<size_t>(T, W), 1);
  pm::pm_xchg_pack<<<std::min(blocks_for(work, 256), 8u * e->sms), 256, 0, e->stream>>>(e->first_ask.p + w0, nw, per, e->ask_best.p, e->ask_count.p, T,
                                                                                  e->xchg_send.p);
  PM_LAUNCH_CHECK("pm_xchg_pack");
  const ncclResult_t nr = nccl.AllGather(e->xchg_send.p, e->xchg_recv.p, stride, ncclUint8, e->comm->nccl, e->stream);
  if (nr != ncclSuccess) return e->fail(PM_E_CUDA, std::string("ncclAllGather: ") + nccl.GetErrorString(nr));
  pm::pm_xchg_unpack<<<std::min(blocks_for(work, 256), 8u * e->sms), 256, 0, e->stream>>>(e->xchg_recv.p, n, stride, std::max(per, 1u), W, T, e->first_ask.p,
                                                                                    e->ask_best.p, e->ask_count.p);
  PM_LAUNCH_CHECK("pm_xchg_unpack");
  tm.stop();
  e->stats.exchange_bytes = (uint64_t)stride * n;
  return PM_OK;
}

// PM_INCREMENTAL: a reference mode on the fused lean path.  pm_match_local takes it on any engine (the host moves the
// three arrays); pm_match on a shard engine without a communicator refuses it: that call resolves one range as if it
// were the table, so there is no whole-table result to keep incremental.
static int check_incremental(pm_engine* e, uint32_t mode, bool local) {
  if ((mode & PM_AUCTION_WARM) && (mode & 0xFFu) != PM_MODE_AUCTION)
    return e->fail(PM_E_INVALID, "pm_match: PM_AUCTION_WARM is for the auction only");
  if ((mode & PM_AUCTION_REVERSE) && (mode & 0xFFu) != PM_MODE_AUCTION)
    return e->fail(PM_E_INVALID, "pm_match: PM_AUCTION_REVERSE is for the auction only");
  // a warm pass is one eps = 1 phase whose release already leaves every unowned worker at price 0
  if ((mode & PM_AUCTION_REVERSE) && (mode & PM_AUCTION_WARM))
    return e->fail(PM_E_INVALID, "pm_match: PM_AUCTION_REVERSE does not go with PM_AUCTION_WARM");
  // a warm repair is a kind of warm pass (and the check above keeps PM_AUCTION_REVERSE off it: it ends with its own
  // reverse stage)
  if ((mode & PM_AUCTION_REPAIR) && !(mode & PM_AUCTION_WARM))
    return e->fail(PM_E_INVALID, "pm_match: PM_AUCTION_REPAIR needs PM_AUCTION_WARM");
  if (!(mode & PM_INCREMENTAL)) return PM_OK;
  if ((mode & 0xFFu) == PM_MODE_AUCTION) return e->fail(PM_E_INVALID, "pm_match: PM_INCREMENTAL is for the reference modes, not the auction");
  if ((mode & (PM_PATH_FUSED | PM_NO_ASK_STATS)) != (PM_PATH_FUSED | PM_NO_ASK_STATS))
    return e->fail(PM_E_INVALID, "pm_match: PM_INCREMENTAL needs PM_PATH_FUSED | PM_NO_ASK_STATS");
  if (!local && !e->comm && (e->cfg.shard_first || e->cfg.shard_count))
    return e->fail(PM_E_UNSUPPORTED, "pm_match: PM_INCREMENTAL on a shard engine needs a communicator or pm_match_local");
  return PM_OK;
}

// A pass that fails may have consumed the rows written since the stored evaluation: nothing of it is trusted again.
static int invalidate_on_failure(pm_engine* e, int rc) {
  if (rc != PM_OK) e->invalidate_eval();
  return rc;
}

int pm_match_local(pm_engine* e, uint32_t mode) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if ((mode & 0xFFu) == PM_MODE_AUCTION) return e->fail(PM_E_UNSUPPORTED, "pm_match_local: auction mode is single-GPU (use pm_match)");
  const int rc = check_incremental(e, mode, true);
  if (rc != PM_OK) return rc;
  return invalidate_on_failure(e, match_local_locked(e, mode));
} catch (...) { return pm_guard_rc(); }
int pm_match_finish(pm_engine* e, uint32_t mode) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (mode & PM_AUCTION_WARM) return e->fail(PM_E_INVALID, "pm_match_finish: PM_AUCTION_WARM is for the auction only");
  if (mode & PM_AUCTION_REVERSE) return e->fail(PM_E_INVALID, "pm_match_finish: PM_AUCTION_REVERSE is for the auction only");
  if (mode & PM_AUCTION_REPAIR) return e->fail(PM_E_INVALID, "pm_match_finish: PM_AUCTION_REPAIR is for the auction only");
  return invalidate_on_failure(e, match_finish_locked(e, mode));
} catch (...) { return pm_guard_rc(); }
int pm_match(pm_engine* e, uint32_t mode) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  int rc = check_incremental(e, mode, false);
  if (rc != PM_OK) return rc;
  if ((mode & 0xFFu) == PM_MODE_AUCTION) return match_auction_locked(e, mode);
  rc = match_local_locked(e, mode);
  if (rc != PM_OK) return invalidate_on_failure(e, rc);
  if (e->comm && e->comm->n_ranks > 1) {
    rc = exchange_locked(e);
    if (rc != PM_OK) return invalidate_on_failure(e, rc);
  }
  return invalidate_on_failure(e, match_finish_locked(e, mode));
} catch (...) { return pm_guard_rc(); }

int pm_set_shard(pm_engine* e, uint32_t first, uint32_t count) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  e->cfg.shard_first = first;
  e->cfg.shard_count = count;
  e->invalidate_eval();
  e->auc_discard();
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// ------------------------------------------------------------------ communicators
int pm_comm_unique_id(uint8_t* id_out) try {
  if (!id_out) return PM_E_INVALID;
  const NcclApi& nccl = nccl_api();
  if (!nccl.ok) { g_create_error = nccl.err; return PM_E_UNSUPPORTED; }
  static_assert(sizeof(ncclUniqueId) == PM_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  const ncclResult_t nr = nccl.GetUniqueId(&id);
  if (nr != ncclSuccess) { g_create_error = std::string("ncclGetUniqueId: ") + nccl.GetErrorString(nr); return PM_E_CUDA; }
  std::memcpy(id_out, &id, sizeof id);
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_comm_create(const uint8_t* unique_id, uint32_t n_ranks, uint32_t rank, int32_t device, pm_comm** out) try {
  if (!unique_id || !out || n_ranks == 0 || rank >= n_ranks) return PM_E_INVALID;
  *out = nullptr;
  const NcclApi& nccl = nccl_api();
  if (!nccl.ok) { g_create_error = nccl.err; return PM_E_UNSUPPORTED; }
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); g_create_error = "pm_comm_create: bad device"; return PM_E_INVALID; }
  ncclUniqueId id;
  std::memcpy(&id, unique_id, sizeof id);
  pm_comm* c = new pm_comm;
  c->n_ranks = n_ranks; c->rank = rank; c->device = device;
  const ncclResult_t nr = nccl.CommInitRank(&c->nccl, (int)n_ranks, id, (int)rank);
  if (nr != ncclSuccess) {
    g_create_error = std::string("ncclCommInitRank: ") + nccl.GetErrorString(nr);
    delete c;
    return PM_E_CUDA;
  }
  *out = c;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

void pm_comm_destroy(pm_comm* c) {
  if (!c) return;
  if (c->nccl && nccl_api().ok) {
    cudaSetDevice(c->device);
    nccl_api().CommDestroy(c->nccl);
  }
  delete c;
}

int pm_attach_comm(pm_engine* e, pm_comm* c) try {
  if (!e) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (c && c->device != e->device) return e->fail(PM_E_INVALID, "pm_attach_comm: communicator and engine are on different devices");
  e->comm = c;
  e->invalidate_eval();
  e->auc_discard();
  e->matched = e->local_done = false;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }


int pm_fetch_result(pm_engine* e, pm_result* out) try {
  if (!e || !out) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->matched) return e->fail(PM_E_STATE, "pm_fetch_result: no completed match");
  PM_CUDA(cudaSetDevice(e->device));
  const uint32_t W = e->n_workers, T = e->n_asks, G = e->n_groups, M = e->n_assigned;
  PM_CUDA(e->r_worker_group.ensure(W)); PM_CUDA(e->r_worker_ask.ensure(W));
  PM_CUDA(e->r_group_ask.ensure(G)); PM_CUDA(e->r_group_off.ensure((size_t)G + 1));
  PM_CUDA(e->r_members.ensure(M)); PM_CUDA(e->r_ask_best.ensure(T)); PM_CUDA(e->r_ask_count.ensure(T));
  if (W) {
    PM_CUDA(cudaMemcpyAsync(e->r_worker_group.p, e->worker_group.p, (size_t)W * 4, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaMemcpyAsync(e->r_worker_ask.p, e->worker_ask.p, (size_t)W * 4, cudaMemcpyDeviceToHost, e->stream));
  }
  if (G) PM_CUDA(cudaMemcpyAsync(e->r_group_ask.p, e->group_ask.p, (size_t)G * 4, cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaMemcpyAsync(e->r_group_off.p, e->group_off.p, ((size_t)G + 1) * 4, cudaMemcpyDeviceToHost, e->stream));
  if (M) PM_CUDA(cudaMemcpyAsync(e->r_members.p, e->members.p, (size_t)M * 4, cudaMemcpyDeviceToHost, e->stream));
  if (T) {
    PM_CUDA(cudaMemcpyAsync(e->r_ask_best.p, e->ask_best.p, (size_t)T * 8, cudaMemcpyDeviceToHost, e->stream));
    PM_CUDA(cudaMemcpyAsync(e->r_ask_count.p, e->ask_count.p, (size_t)T * 4, cudaMemcpyDeviceToHost, e->stream));
  }
  PM_CUDA(cudaStreamSynchronize(e->stream));
  out->n_workers = W; out->n_asks = T; out->n_groups = G; out->n_members = M;
  out->worker_group = e->r_worker_group.p; out->worker_ask = e->r_worker_ask.p;
  out->group_ask = e->r_group_ask.p; out->group_off = e->r_group_off.p; out->group_members = e->r_members.p;
  out->ask_best = (const int64_t*)e->r_ask_best.p; out->ask_count = e->r_ask_count.p;
  out->stats = e->stats;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_build_cost_tile(pm_engine* e, uint32_t t0, uint32_t nt, int64_t* host_out) try {
  if (!e || !host_out) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_workers || !e->have_asks) return e->fail(PM_E_STATE, "pm_build_cost_tile: tables not set");
  if (e->max_pattern_row > e->n_patterns || (e->max_pattern_row && !e->have_bits))
    return e->fail(PM_E_STATE, "pm_build_cost_tile: model table missing");
  if ((uint64_t)t0 + nt > e->n_asks || nt == 0) return e->fail(PM_E_INVALID, "pm_build_cost_tile: ask range");
  {
    const int rc = use_ask_form(e, false);
    if (rc != PM_OK) return rc;
  }
  PM_CUDA(cudaSetDevice(e->device));
  const uint32_t W = e->n_workers;
  uint32_t w0 = 0, nw = 0;
  e->shard(&w0, &nw);
  if (nw == 0 || (uint64_t)w0 + nw > W) return e->fail(PM_E_INVALID, "pm_build_cost_tile: empty worker range");
  if (!e->have_bits) {
    PM_CUDA(e->bits.ensure(1));
    PM_CUDA(cudaMemsetAsync(e->bits.p, 0xFF, 4, e->stream));
    e->words = 1;
  }
  const size_t ld = (((size_t)nw + pm::kEvalCols - 1) / pm::kEvalCols) * pm::kEvalCols;
  if (nt > 65535u * pm::kEvalRows) return e->fail(PM_E_INVALID, "pm_build_cost_tile: too many rows");
  if (e->cost.ensure((size_t)nt * ld, e->device, e->tune_compress != 0, e->stream) != cudaSuccess) {
    cudaGetLastError();
    return e->fail(PM_E_NOMEM, "pm_build_cost_tile: cannot allocate the tile");
  }
  dim3 grid(blocks_for(ld, pm::kEvalCols), blocks_for(nt, pm::kEvalRows));
  pm::EvalParams p;
  int bits_mode = 0;
  bool fast = false;
  {
    int rc = pick_predicate(e, &p, &bits_mode, &fast);
    if (rc != PM_OK) return rc;
    rc = bind_rows(e, p.nacc != nullptr);
    if (rc != PM_OK) return rc;
  }
  launch_build(e, p, bits_mode, fast, grid, t0, nt, w0, nw, e->cost.p, ld);   // exports the int64 tile
  PM_LAUNCH_CHECK("pm_build_cost");
  PM_CUDA(cudaMemcpy2DAsync(host_out, (size_t)nw * 8, e->cost.p, ld * 8, (size_t)nw * 8, nt,
                            cudaMemcpyDeviceToHost, e->stream));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_get_stats(const pm_engine* e, pm_stats* out) try {
  if (!e || !out) return PM_E_INVALID;
  *out = e->stats;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_device_buffer(pm_engine* e, uint32_t which, void** dev_ptr, size_t* bytes) try {
  if (!e || !dev_ptr || !bytes) return PM_E_INVALID;
  std::lock_guard<std::mutex> lk(e->mu);
  switch (which) {
    case PM_BUF_WORKER_FIRST_ASK: *dev_ptr = e->first_ask.p; *bytes = (size_t)e->n_workers * 4; break;
    case PM_BUF_ASK_BEST: *dev_ptr = e->ask_best.p; *bytes = (size_t)e->n_asks * 8; break;
    case PM_BUF_ASK_COUNT: *dev_ptr = e->ask_count.p; *bytes = (size_t)e->n_asks * 4; break;
    case PM_BUF_COST_TILE: *dev_ptr = e->cost.p; *bytes = e->cost_tile_used; break;
    default: return e->fail(PM_E_INVALID, "pm_device_buffer: unknown buffer");
  }
  if (!*dev_ptr) return e->fail(PM_E_STATE, "pm_device_buffer: buffer not allocated yet (run pm_match_local)");
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_stream_sync(pm_engine* e) try {
  if (!e) return PM_E_INVALID;
  PM_CUDA(cudaSetDevice(e->device));
  PM_CUDA(cudaStreamSynchronize(e->stream));
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

// ------------------------------------------------------------------ one process, several GPUs
// The orchestrator is one process with one management loop (reference crates/orchestrator/src/main.rs:283-289), so
// the multi-GPU form it can call is this one: N engines, one per device, each with the full (small) tables and an
// equal share of the canonical worker order; communicators from ncclCommInitAll; a pass = every device evaluates its
// share, one all-gather, every device runs the same resolution sweep (engine 0's result is the result).
struct pm_multi {
  std::vector<pm_engine*> engines;
  std::vector<pm_comm*> comms;
  std::vector<int> devices;   // kept to re-create the communicators after a failed pass aborted them
  std::string err;
};

void pm_multi_destroy(pm_multi* m) {
  if (!m) return;
  for (pm_engine* e : m->engines) pm_destroy(e);
  for (pm_comm* c : m->comms) pm_comm_destroy(c);
  delete m;
}

int pm_multi_create(const pm_cfg* cfg, const int32_t* devices, uint32_t n, pm_multi** out) try {
  if (!cfg || !devices || !out || n == 0) return PM_E_INVALID;
  *out = nullptr;
  pm_multi* m = new pm_multi;
  m->devices.assign(devices, devices + n);
  for (uint32_t i = 0; i < n; ++i) {
    pm_cfg c = *cfg;
    c.device = devices[i];
    c.shard_first = c.shard_count = 0;
    c.stream = nullptr;   // one private stream per device
    pm_engine* e = nullptr;
    const int rc = pm_create(&c, &e);
    if (rc != PM_OK) { pm_multi_destroy(m); return rc; }
    m->engines.push_back(e);
  }
  if (n > 1) {
    const NcclApi& nccl = nccl_api();
    if (!nccl.ok) { g_create_error = nccl.err; pm_multi_destroy(m); return PM_E_UNSUPPORTED; }
    std::vector<ncclComm_t> raw(n, nullptr);
    const ncclResult_t nr = nccl.CommInitAll(raw.data(), (int)n, m->devices.data());
    if (nr != ncclSuccess) {
      g_create_error = std::string("ncclCommInitAll: ") + nccl.GetErrorString(nr);
      pm_multi_destroy(m);
      return PM_E_CUDA;
    }
    for (uint32_t i = 0; i < n; ++i) {
      pm_comm* c = new pm_comm;
      c->nccl = raw[i]; c->n_ranks = n; c->rank = i; c->device = devices[i];
      m->comms.push_back(c);
      m->engines[i]->comm = c;
    }
  }
  *out = m;
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

uint32_t pm_multi_size(const pm_multi* m) { return m ? (uint32_t)m->engines.size() : 0u; }
pm_engine* pm_multi_engine(pm_multi* m, uint32_t i) { return (m && i < m->engines.size()) ? m->engines[i] : nullptr; }
const char* pm_multi_last_error(const pm_multi* m) { return m ? m->err.c_str() : g_create_error.c_str(); }

#define PM_MULTI_EACH(call)                                      \
  do {                                                           \
    if (!m) return PM_E_INVALID;                                 \
    for (pm_engine* e : m->engines) {                            \
      const int rc_ = (call);                                    \
      if (rc_ != PM_OK) { m->err = pm_last_error(e); return rc_; } \
    }                                                            \
    return PM_OK;                                                \
  } while (0)

int pm_multi_set_asks(pm_multi* m, const pm_ask* asks, uint32_t n_asks, const pm_gpu_opt* opts, uint32_t n_opts) try {
  PM_MULTI_EACH(pm_set_asks(e, asks, n_asks, opts, n_opts));
} catch (...) { return pm_guard_rc(); }
int pm_multi_set_ask_enabled(pm_multi* m, const uint32_t* idx, const uint8_t* enabled, uint32_t n) try {
  if (m && !m->engines.empty()) {   // an index out of range changes nothing on any device
    pm_engine* e0 = m->engines[0];
    for (uint32_t i = 0; idx && i < n; ++i)
      if (idx[i] >= e0->n_asks) { m->err = "pm_set_ask_enabled: ask index out of range"; return PM_E_INVALID; }
  }
  PM_MULTI_EACH(pm_set_ask_enabled(e, idx, enabled, n));
} catch (...) { return pm_guard_rc(); }
// the ask-table deltas on every device; a call the checks refuse is refused before any device changes
int pm_multi_update_asks(pm_multi* m, const uint32_t* idx, const pm_ask* asks, uint32_t n, const pm_gpu_opt* opts,
                         uint32_t n_opts) try {
  if (m && !m->engines.empty()) {
    pm_engine* e0 = m->engines[0];
    std::lock_guard<std::mutex> lk(e0->mu);
    if (e0->have_asks && !((n && (!idx || !asks)) || (n_opts && !opts))) {
      std::vector<uint32_t> uidx;
      std::vector<pm_ask> urows;
      const int rc = check_ask_rows(e0, "pm_update_asks", idx, asks, n, n_opts, &uidx, &urows, &m->err);
      if (rc != PM_OK) return rc;
    }
  }
  PM_MULTI_EACH(pm_update_asks(e, idx, asks, n, opts, n_opts));
} catch (...) { return pm_guard_rc(); }
int pm_multi_resize_asks(pm_multi* m, uint32_t n_asks, const pm_ask* added, const pm_gpu_opt* opts, uint32_t n_opts) try {
  if (m && !m->engines.empty()) {
    pm_engine* e0 = m->engines[0];
    std::lock_guard<std::mutex> lk(e0->mu);
    const uint32_t n_add = n_asks > e0->n_asks ? n_asks - e0->n_asks : 0u;
    if (e0->have_asks && n_asks < (1u << 30) && !((n_add && !added) || (n_opts && !opts))) {
      std::vector<uint32_t> uidx;
      std::vector<pm_ask> urows;
      const int rc = check_ask_rows(e0, "pm_resize_asks", nullptr, added, n_add, n_opts, &uidx, &urows, &m->err);
      if (rc != PM_OK) return rc;
    }
  }
  PM_MULTI_EACH(pm_resize_asks(e, n_asks, added, opts, n_opts));
} catch (...) { return pm_guard_rc(); }
int pm_multi_remove_asks(pm_multi* m, const uint32_t* idx, uint32_t n) try {
  if (m && !m->engines.empty()) {
    pm_engine* e0 = m->engines[0];
    std::lock_guard<std::mutex> lk(e0->mu);
    std::vector<uint32_t> removed;
    if (e0->have_asks) {
      const int rc = check_remove(e0, idx, n, &removed, &m->err);
      if (rc != PM_OK) return rc;
    }
  }
  PM_MULTI_EACH(pm_remove_asks(e, idx, n));
} catch (...) { return pm_guard_rc(); }
int pm_multi_insert_asks(pm_multi* m, const uint32_t* before, const pm_ask* asks, uint32_t n, const pm_gpu_opt* opts,
                         uint32_t n_opts) try {
  if (m && !m->engines.empty()) {
    pm_engine* e0 = m->engines[0];
    std::lock_guard<std::mutex> lk(e0->mu);
    if (e0->have_asks) {
      const int rc = check_insert(e0, "pm_insert_asks", before, asks, n, opts, n_opts, &m->err);
      if (rc != PM_OK) return rc;
    }
  }
  PM_MULTI_EACH(pm_insert_asks(e, before, asks, n, opts, n_opts));
} catch (...) { return pm_guard_rc(); }
int pm_multi_set_model_table(pm_multi* m, const uint32_t* bits, uint32_t n_patterns, uint32_t n_models, uint32_t words) try {
  PM_MULTI_EACH(pm_set_model_table(e, bits, n_patterns, n_models, words));
} catch (...) { return pm_guard_rc(); }
int pm_multi_set_worker_count(pm_multi* m, uint32_t n_workers) try {
  PM_MULTI_EACH(pm_set_worker_count(e, n_workers));
} catch (...) { return pm_guard_rc(); }
int pm_multi_upsert_workers(pm_multi* m, const pm_worker_a* a, const pm_worker_b* b, uint32_t first, uint32_t n) try {
  PM_MULTI_EACH(pm_upsert_workers(e, a, b, first, n));
} catch (...) { return pm_guard_rc(); }
int pm_multi_set_worker_locations(pm_multi* m, const double* lat, const double* lon, uint32_t first, uint32_t n) try {
  PM_MULTI_EACH(pm_set_worker_locations(e, lat, lon, first, n));
} catch (...) { return pm_guard_rc(); }
int pm_multi_set_worker_addr_rank(pm_multi* m, const uint32_t* rank, uint32_t first, uint32_t n) try {
  PM_MULTI_EACH(pm_set_worker_addr_rank(e, rank, first, n));
} catch (...) { return pm_guard_rc(); }
int pm_multi_set_flags(pm_multi* m, const uint32_t* idx, const uint32_t* flags, uint32_t n) try {
  PM_MULTI_EACH(pm_set_flags(e, idx, flags, n));
} catch (...) { return pm_guard_rc(); }
int pm_multi_resize_workers(pm_multi* m, uint32_t n_workers) try {
  PM_MULTI_EACH(pm_resize_workers(e, n_workers));
} catch (...) { return pm_guard_rc(); }
int pm_multi_update_workers(pm_multi* m, const uint32_t* idx, const pm_worker_a* a, const pm_worker_b* b, const double* lat,
                            const double* lon, uint32_t n) try {
  PM_MULTI_EACH(pm_update_workers(e, idx, a, b, lat, lon, n));
} catch (...) { return pm_guard_rc(); }
// the replicated tables agree, so device 0's checks decide for all of them: a refused call changes no device
int pm_multi_remove_workers(pm_multi* m, const uint32_t* idx, uint32_t n) try {
  if (m && !m->engines.empty()) {
    pm_engine* e0 = m->engines[0];
    std::lock_guard<std::mutex> lk(e0->mu);
    std::vector<uint32_t> removed;
    if (e0->have_workers) {
      const int rc = check_remove_workers(e0, idx, n, &removed, &m->err);
      if (rc != PM_OK) return rc;
    }
  }
  PM_MULTI_EACH(pm_remove_workers(e, idx, n));
} catch (...) { return pm_guard_rc(); }
int pm_multi_insert_workers(pm_multi* m, const uint32_t* before, const pm_worker_a* a, const pm_worker_b* b, const double* lat,
                            const double* lon, uint32_t n) try {
  if (m && !m->engines.empty()) {
    pm_engine* e0 = m->engines[0];
    std::lock_guard<std::mutex> lk(e0->mu);
    if (e0->have_workers) {
      const int rc = check_insert_workers(e0, before, a, b, lat, lon, n, &m->err);
      if (rc != PM_OK) return rc;
    }
  }
  PM_MULTI_EACH(pm_insert_workers(e, before, a, b, lat, lon, n));
} catch (...) { return pm_guard_rc(); }
int pm_multi_sync(pm_multi* m) try {
  PM_MULTI_EACH(pm_stream_sync(e));
} catch (...) { return pm_guard_rc(); }
#undef PM_MULTI_EACH

// every engine's version only grows, so the sum changes whenever any of them does
uint64_t pm_multi_table_version(const pm_multi* m) {
  if (!m) return 0;
  uint64_t v = 0;
  for (const pm_engine* e : m->engines) v += pm_table_version(e);
  return v;
}

// After a failed pass aborted the communicators: new ones over the same devices, attached again.  pm_attach_comm
// discards each engine's stored evaluation, so the pass that follows evaluates every device's share in full.
static int multi_reconnect(pm_multi* m) {
  const NcclApi& nccl = nccl_api();
  const uint32_t n = (uint32_t)m->engines.size();
  std::vector<ncclComm_t> raw(n, nullptr);
  const ncclResult_t nr = nccl.CommInitAll(raw.data(), (int)n, m->devices.data());
  if (nr != ncclSuccess) {
    m->err = std::string("pm_multi_match: ncclCommInitAll: ") + nccl.GetErrorString(nr);
    return PM_E_CUDA;
  }
  for (uint32_t i = 0; i < n; ++i) m->comms[i]->nccl = raw[i];
  for (uint32_t i = 0; i < n; ++i) {
    const int rc = pm_attach_comm(m->engines[i], m->comms[i]);
    if (rc != PM_OK) { m->err = pm_last_error(m->engines[i]); return rc; }
  }
  return PM_OK;
}

int pm_multi_match(pm_multi* m, uint32_t mode) try {
  if (!m) return PM_E_INVALID;
  const size_t n = m->engines.size();
  if (n == 1) {
    const int rc = pm_match(m->engines[0], mode);
    if (rc != PM_OK) m->err = pm_last_error(m->engines[0]);
    return rc;
  }
  // a rank that fails before the collective would leave the others waiting in it: check what can be checked first,
  // and abort every communicator if a rank still fails on the way (the next pass makes new ones)
  for (pm_engine* e : m->engines) {
    if (!e->have_workers || !e->have_asks) { m->err = "pm_multi_match: worker and ask tables must be set first"; return PM_E_STATE; }
    if (e->n_workers != m->engines[0]->n_workers || e->n_asks != m->engines[0]->n_asks) {
      m->err = "pm_multi_match: engines hold different tables";
      return PM_E_STATE;
    }
  }
  if (!m->comms[0]->nccl) {   // the abort below clears every communicator at once
    const int rc = multi_reconnect(m);
    if (rc != PM_OK) return rc;
  }
  std::vector<int> rcs(n, PM_OK);
  std::atomic<bool> aborted{false};
  std::vector<std::thread> threads;
  for (size_t i = 0; i < n; ++i) {
    threads.emplace_back([&, i] {
      rcs[i] = pm_match(m->engines[i], mode);
      if (rcs[i] != PM_OK && !aborted.exchange(true) && nccl_api().ok)
        for (pm_comm* c : m->comms)
          if (c->nccl) { nccl_api().CommAbort(c->nccl); c->nccl = nullptr; }
    });
  }
  for (auto& t : threads) t.join();
  for (size_t i = 0; i < n; ++i)
    if (rcs[i] != PM_OK) { m->err = pm_last_error(m->engines[i]); return rcs[i]; }
  return PM_OK;
} catch (...) { return pm_guard_rc(); }

int pm_multi_fetch_result(pm_multi* m, pm_result* out) try {
  if (!m || m->engines.empty()) return PM_E_INVALID;
  const int rc = pm_fetch_result(m->engines[0], out);
  if (rc != PM_OK) m->err = pm_last_error(m->engines[0]);
  return rc;
} catch (...) { return pm_guard_rc(); }

}  // extern "C"
