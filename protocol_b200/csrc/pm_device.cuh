// pm_device.cuh — device-side table layouts and the feasibility predicate.
//
// The predicate restates, on the SoA tables of include/prime_match.h,
//   NodeGroupsPlugin::is_node_compatible_with_config
//     (crates/orchestrator/src/plugins/node_groups/mod.rs:206-215)
//   ComputeSpecs::meets / GpuSpecs::meets / CpuSpecs::meets
//     (crates/shared/src/models/node.rs:377-541)
// with every Option<> folded into (a) one presence-mask test and (b) unsigned
// interval compares, so that one (ask, worker) evaluation is a handful of
// integer instructions and no string work (the model clause, node.rs:463-484,
// is a bit test against the host-interned table).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/prime_match.h"

namespace pm {

constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr long long kInf = 0x7FFFFFFFFFFFFFFFll;
constexpr uint32_t kNarrowInfeasible = 0x7FFFFFFFu;   // the 32-bit cost tile's "infeasible": kInf's high word

// Synthetic presence bits added on the device side (never part of the ABI):
constexpr uint32_t kCandBit = 1u << 31;        // Healthy && p2p_id.is_some() && !assigned (mod.rs:492-497)
constexpr uint32_t kNeverBit = 1u << 30;       // no worker carries it: "this clause can never pass"
constexpr uint32_t kTotInvalidBit = 1u << 29;  // count or memory_mb is None: total-memory clauses are skipped

// Device form of one ask row (32 B).  `need` = presence bits the worker must
// carry: the candidate bit always; HAS_SPECS when the config has requirements
// (mod.rs:210-214); HAS_CPU / HAS_CPU_CORES / HAS_RAM / HAS_STORAGE for the scalar
// clauses (node.rs:381-418); HAS_GPU when requirements.gpu is non-empty
// (node.rs:420-425).  Thresholds of absent clauses are 0 so the unsigned >=
// compares pass.
struct __align__(16) DevAsk {
  uint32_t need;
  uint32_t n_opts;
  uint32_t opt_off;
  uint32_t cpu_cores;
  uint32_t ram_mb;
  uint32_t storage_gb;
  uint32_t pad0, pad1;
};

// Device form of one GpuRequirements option (32 B).  memory_mb / memory_mb_min
// fold into mem_lo (both are "spec >= req", node.rs:487-498), memory_mb_max into
// the span (:499-503): lo <= x <= hi  <=>  (x - lo) <= (hi - lo) unsigned.  `need`
// carries HAS_GPU_MODEL / HAS_GPU_MEM when the clause is present (a None spec field
// fails a present clause, is_none_or); an empty interval becomes kNeverBit (memory)
// or kTotInvalidBit (total memory: only workers that skip the clause can pass).
struct __align__(16) DevOpt {
  uint32_t need;
  uint32_t count_mask;   // 0xFFFFFFFF when gpu:count is required, else 0
  uint32_t count;
  uint32_t mem_lo, mem_span;
  uint32_t tot_lo, tot_span;
  uint32_t pattern_row;  // row in the device bit table; 0 = no model clause
};

// Fast-path form of an option (same 32 B slot as DevOpt, separate array).  Valid
// when every numeric operand on both sides is < 2^31 and every gpu count < 2^16
// (checked at upload; otherwise the generic predicate is used).  Every clause ends as a SIGN BIT ("set = fails"),
// so clauses combine with OR (AND across the OR-options of an ask) and nothing is compared or selected until the
// very end:
//   * the worker's presence flags and gpu count are packed into one `key` word of 29 bits (layout below), so
//     presence + count is one masked equality z = (key & m) ^ v, with m/v also carrying the owning ask's `need`;
//     the model clause adds ~word & mmask (device acceptance words hold 31 models, so z < 2^31), and
//     0 - z has its sign set exactly when z != 0 — a subtraction, which issues on the FMA pipe (IMAD);
//   * range clauses are the signs of (x - lo) | (hi - x): IMAD subtractions again.
// What is left for the ALU pipe per (option, worker) is five LOP3; the int64 cost is then formed with one shift
// and two IMADs (pm_kernels.cuh) — the integer work is split evenly over the two pipes instead of 2:1 on the ALU.
struct __align__(16) DevOptF {
  uint32_t m, v;
  uint32_t mem_lo, mem_hi;
  uint32_t tot_lo, tot_hi;
  uint32_t pattern_row;
  uint32_t pad;
};
// One ask as the fast build kernel reads it (48 B = three 128-bit shared-memory loads at an address that depends on
// the row number only, so the next row's operands are fetched while the current row is evaluated): the first OR-option
// inline, the scalar thresholds, and where the remaining options are.  `wp` is the option's pattern row until
// pm_bind_rows replaces it, when every acceptance row is a single word, by the word itself.
struct __align__(16) FastRow {
  uint32_t m, v, mem_lo, mem_hi;
  uint32_t tot_lo, tot_hi, wp, n_opts;
  uint32_t cpu_cores, ram_mb, storage_gb, opt_off;
};

// key = flags bits 3..12 (PM_W_HAS_*) in bits 0..9, candidate 10, never 11, total-memory-skipped 12, gpu count 13..28
constexpr uint32_t kKeyCountShift = 13;
constexpr uint32_t kKeyCandBit = 1u << 10, kKeyNeverBit = 1u << 11, kKeyTotInvalidBit = 1u << 12;
constexpr uint32_t kSign = 0x80000000u;
constexpr uint32_t kModelsPerWord = 31;   // device acceptance words keep bit 31 clear (see DevOptF)

// presence bits (ABI flags + the synthetic bits 29..31) -> their positions in `key`
__host__ __device__ __forceinline__ uint32_t key_bits(uint32_t f) {
  return ((f >> 3) & 0x3FFu) | ((f & (1u << 31)) ? kKeyCandBit : 0u) | ((f & (1u << 30)) ? kKeyNeverBit : 0u) |
         ((f & (1u << 29)) ? kKeyTotInvalidBit : 0u);
}

// One worker held in registers.
struct WorkerReg {
  uint32_t flags;      // ABI presence bits + kCandBit / kTotInvalidBit
  uint32_t key;        // fast path: key_bits(flags) | count << 13
  uint32_t count_eff;  // None behaves exactly like Some(0) in the count clause (node.rs:447-461)
  uint32_t mem_eff;
  uint32_t tot;        // count * memory_mb, wrapping (release-build u32 multiply, node.rs:509,518)
  uint32_t tot_keep;   // all-ones when both count and memory_mb are Some, else 0 (clause skipped)
  uint32_t cores, ram, storage;
  uint32_t mword, mmask;
  uint32_t price;
};

__device__ __forceinline__ WorkerReg make_worker(uint4 a, uint4 b) {
  WorkerReg w;
  const bool hc = (a.w & PM_W_HAS_GPU_COUNT) != 0, hm = (a.w & PM_W_HAS_GPU_MEM) != 0;
  const bool cand = (a.w & (PM_W_HEALTHY | PM_W_P2P | PM_W_ASSIGNED)) == (PM_W_HEALTHY | PM_W_P2P);
  w.flags = (a.w & 0x1FFFFFFFu) | (cand ? kCandBit : 0u) | ((hc && hm) ? 0u : kTotInvalidBit);
  w.count_eff = hc ? a.x : 0u;
  w.key = key_bits(w.flags) | (w.count_eff << kKeyCountShift);
  w.mem_eff = hm ? a.y : 0u;
  w.tot = a.x * a.y;
  w.tot_keep = (hc && hm) ? 0xFFFFFFFFu : 0u;
  w.cores = b.x;
  w.ram = b.y;
  w.storage = b.z;
  w.price = b.w;
  const uint32_t mid = (a.w & PM_W_HAS_GPU_MODEL) ? a.z : 0u;
  w.mword = mid / kModelsPerWord;
  w.mmask = 1u << (mid % kModelsPerWord);
  return w;
}

__device__ __forceinline__ WorkerReg null_worker() {
  WorkerReg w;
  w.flags = kTotInvalidBit; w.key = kKeyTotInvalidBit; w.count_eff = 0; w.mem_eff = 0; w.tot = 0; w.tot_keep = 0;
  w.cores = 0; w.ram = 0; w.storage = 0; w.mword = 0; w.mmask = 1u; w.price = 0;
  return w;
}

// GpuSpecs::meets for one option (node.rs:443-527).  `row` points at the
// option's row of the acceptance bit table (any address space).
__device__ __forceinline__ bool opt_meets(const DevOpt& q, const WorkerReg& w,
                                          const uint32_t* __restrict__ bits, uint32_t words) {
  bool ok = (w.flags & q.need) == q.need;
  ok &= (w.count_eff & q.count_mask) == q.count;
  ok &= (w.mem_eff - q.mem_lo) <= q.mem_span;
  ok &= (((w.tot - q.tot_lo) & w.tot_keep) <= q.tot_span);
  if (q.pattern_row != 0u)  // uniform across the warp in the hot kernels
    ok &= (bits[q.pattern_row * words + w.mword] & w.mmask) != 0u;
  return ok;
}

// is_node_compatible_with_config + ComputeSpecs::meets + the candidate filter.
__device__ __forceinline__ bool ask_meets(const DevAsk& a, const DevOpt* __restrict__ opts,
                                          const WorkerReg& w, const uint32_t* __restrict__ bits,
                                          uint32_t words) {
  bool ok = ((w.flags & a.need) == a.need) & (w.cores >= a.cpu_cores) & (w.ram >= a.ram_mb) &
            (w.storage >= a.storage_gb);
  if (a.n_opts != 0u) {
    bool any = false;
    for (uint32_t o = 0; o < a.n_opts; ++o) any |= opt_meets(opts[a.opt_off + o], w, bits, words);
    ok &= any;
  }
  return ok;
}

// ---- Hopper bulk async copy (TMA, 1-D) -------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}

}  // namespace pm
