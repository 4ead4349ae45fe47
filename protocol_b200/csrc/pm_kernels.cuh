// pm_kernels.cuh — sm_90a kernels of the matching pass.
//
//   pm_build_cost   cost-matrix build: int64 cost[t][w] for a tile of asks x a
//                   stripe of workers, HBM-write-bound (8 B per evaluation; the
//                   FastRow form's narrow tile: the 32-bit cost word, 4 B)
//   pm_argmin       one read of the int64 tile (8 B per evaluation): per-ask packed
//                   (min_cost, argmin) + feasible count, per-worker first ask
//   pm_build_argmin the narrow tile's build with the same outputs folded in, never
//                   read back
//   pm_fused_eval   the same outputs without materialising the matrix
//   pm_hist / pm_check_tails / pm_sweep / pm_emit_* : resolution sweep that turns
//                   "first feasible ask per worker" into the reference's groups
//
// Reference semantics being reproduced: NodeGroupsPlugin::try_form_new_groups,
// crates/orchestrator/src/plugins/node_groups/mod.rs:478-628.
#pragma once
#include <type_traits>
#include <cub/block/block_radix_sort.cuh>
#include "pm_device.cuh"

namespace pm {

struct EvalParams {
  const uint4* __restrict__ wa;       // plane A [n_workers]
  const uint4* __restrict__ wb;       // plane B [n_workers]
  const DevAsk* __restrict__ asks;    // [n_asks] priority order
  const DevOpt* __restrict__ opts;    // CSR, ask order
  const DevOptF* __restrict__ opts_fast;  // same CSR, fast-path form
  const FastRow* __restrict__ frows;      // [n_asks] fast build kernel's view of an ask (first option inline)
  const uint32_t* __restrict__ bits;  // [(n_patterns+1) * words], row 0 all-ones
  const uint32_t* __restrict__ nacc;  // worker-major acceptance (pm_worker_nacc), or null: per worker the mask of the pattern
                                      // rows that REJECT its model.  Then `bits` is the one-word table word[r] = ~(1 << r) and a
                                      // worker's mmask is nacc[w]: the fast clause ~word & mmask = (1 << r) & nacc[w] is the same
                                      // test with the roles of row and worker swapped — no table lookup per (row, worker) pair,
                                      // however many distinct model strings the pool has (at most 30 patterns)
  uint32_t words;
  uint32_t n_workers;                 // global
  uint32_t n_asks;
  uint32_t n_opts;
  uint32_t n_bits_rows;               // n_patterns + 1
  uint32_t sign_shift;                // always 31.  A run-time value on purpose: with a literal shift ptxas proves the
                                      // result is 0/1 and turns the two multiply-adds that form the packed cost back
                                      // into a compare and two selects on the (busier) ALU pipe
};

// ------------------------------------------------------------------ evaluation core
constexpr int kEvalThreads = 256;
constexpr int kEvalWPT = 4;                          // workers per thread: two 16 B stores per row
constexpr int kEvalCols = kEvalThreads * kEvalWPT;   // 1024 workers per CTA stripe
constexpr int kEvalRows = 128;                       // asks per CTA (staged in shared memory)
constexpr int kOptCap = 384;                         // options staged at a time
constexpr int kBitsCap = 2048;                       // acceptance-table words kept in shared memory

struct __align__(128) EvalStage {
  DevAsk ask[kEvalRows];
  DevOpt opt[kOptCap];
  uint32_t bits[kBitsCap];
  uint64_t bar;
};

// The predicate for one staged ask against WPT register-resident workers, as
// all-ones / zero masks.  Ask and option operands are warp-uniform shared-memory
// reads; each clause is one subtract/and plus one ISETP chained on a single
// predicate (inline PTX keeps ptxas from materialising booleans in registers).
__device__ __forceinline__ uint32_t base_mask(const DevAsk& a, const WorkerReg& w) {
  uint32_t r;
  asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\t"
      "and.b32 t, %1, %2;\n\t"
      "setp.eq.u32 p, t, %2;\n\t"
      "setp.ge.and.u32 p, %3, %4, p;\n\t"
      "setp.ge.and.u32 p, %5, %6, p;\n\t"
      "setp.ge.and.u32 p, %7, %8, p;\n\t"
      "selp.b32 %0, -1, 0, p;\n\t}"
      : "=r"(r)
      : "r"(w.flags), "r"(a.need), "r"(w.cores), "r"(a.cpu_cores), "r"(w.ram), "r"(a.ram_mb),
        "r"(w.storage), "r"(a.storage_gb));
  return r;
}

// GpuSpecs::meets for one option (node.rs:443-527).  `word` is the worker's word
// of the option's acceptance row (row 0 is all-ones: no model clause).
__device__ __forceinline__ uint32_t opt_mask(const DevOpt& q, const WorkerReg& w, uint32_t word) {
  uint32_t r;
  asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\t"
      "and.b32 t, %1, %2;\n\t"
      "setp.eq.u32 p, t, %2;\n\t"            // presence bits
      "and.b32 t, %3, %4;\n\t"
      "setp.eq.and.u32 p, t, %5, p;\n\t"     // count == (or unconstrained)
      "sub.u32 t, %6, %7;\n\t"
      "setp.le.and.u32 p, t, %8, p;\n\t"     // memory_mb in [lo, hi]
      "sub.u32 t, %9, %11;\n\t"
      "and.b32 t, t, %10;\n\t"               // workers without count*memory skip the clause
      "setp.le.and.u32 p, t, %12, p;\n\t"    // count * memory_mb in [lo, hi]
      "and.b32 t, %13, %14;\n\t"
      "setp.ne.and.u32 p, t, 0, p;\n\t"      // model accepted
      "selp.b32 %0, -1, 0, p;\n\t}"
      : "=r"(r)
      : "r"(w.flags), "r"(q.need), "r"(w.count_eff), "r"(q.count_mask), "r"(q.count),
        "r"(w.mem_eff), "r"(q.mem_lo), "r"(q.mem_span), "r"(w.tot), "r"(w.tot_keep), "r"(q.tot_lo),
        "r"(q.tot_span), "r"(word), "r"(w.mmask));
  return r;
}

// BITS: 0 = acceptance table in global memory, 1 = in shared memory, 2 = in shared
// memory with one word per row (<= 32 worker models): the word is warp-uniform.
template <int WPT, int BITS>
__device__ __forceinline__ void eval_row(const EvalStage& s, const DevAsk& a, uint32_t obegin,
                                         const WorkerReg (&w)[WPT],
                                         const uint32_t* __restrict__ gbits, uint32_t words,
                                         uint32_t (&f)[WPT]) {
#pragma unroll
  for (int k = 0; k < WPT; ++k) f[k] = base_mask(a, w[k]);
  if (a.n_opts != 0u) {
    uint32_t any[WPT];
#pragma unroll
    for (int k = 0; k < WPT; ++k) any[k] = 0u;
    const uint32_t o0 = a.opt_off - obegin;
    for (uint32_t o = 0; o < a.n_opts; ++o) {
      const DevOpt q = s.opt[o0 + o];
      if (BITS == 2) {
        const uint32_t word = s.bits[q.pattern_row];
#pragma unroll
        for (int k = 0; k < WPT; ++k) any[k] |= opt_mask(q, w[k], word);
      } else {
        const uint32_t rowoff = q.pattern_row * words;
#pragma unroll
        for (int k = 0; k < WPT; ++k) {
          const uint32_t word = (BITS == 1) ? s.bits[rowoff + w[k].mword] : __ldg(gbits + rowoff + w[k].mword);
          any[k] |= opt_mask(q, w[k], word);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < WPT; ++k) f[k] &= any[k];
  }
}

// Fast path (all operands < 2^31, counts < 2^16; layout and derivation at DevOptF in pm_device.cuh): the SIGN BIT of
// fail[k] is set <=> worker k does not meet the ask.  Per worker and option: 5 LOP3 on the ALU pipe, 7 IMAD-pipe
// adds/subtractions; clauses are never compared, only OR-ed (AND across the ask's OR-options).  Every converted ask
// has at least one option row (pm_ask_convert adds a neutral one), so there is no option-less special case.
template <int WPT, int BITS>
__device__ __forceinline__ void eval_opt_fast(const EvalStage& s, const DevOptF& q, const WorkerReg (&w)[WPT],
                                              const uint32_t* __restrict__ gbits, uint32_t words, uint32_t (&u)[WPT]) {
  const uint32_t rowoff = q.pattern_row * words;
  const uint32_t uword = (BITS == 2) ? s.bits[q.pattern_row] : 0u;
#pragma unroll
  for (int k = 0; k < WPT; ++k) {
    const uint32_t word = (BITS == 2) ? uword
                          : (BITS == 1) ? s.bits[rowoff + w[k].mword] : __ldg(gbits + rowoff + w[k].mword);
    const uint32_t z = ((w[k].key & q.m) ^ q.v) | (~word & w[k].mmask);          // < 2^31, non-zero = fails
    const uint32_t r = (w[k].mem_eff - q.mem_lo) | (q.mem_hi - w[k].mem_eff) |
                       (((w[k].tot - q.tot_lo) | (q.tot_hi - w[k].tot)) & w[k].tot_keep);
    u[k] = (0u - z) | r;    // z < 2^31: the negation has its sign set exactly when z != 0
  }
}

template <int WPT, int BITS>
__device__ __forceinline__ void eval_row_fast(const EvalStage& s, const DevAsk& a, uint32_t obegin,
                                              const WorkerReg (&w)[WPT],
                                              const uint32_t* __restrict__ gbits, uint32_t words,
                                              uint32_t (&fail)[WPT]) {
  const DevOptF* optf = reinterpret_cast<const DevOptF*>(s.opt) + (a.opt_off - obegin);
  uint32_t um[WPT];
  eval_opt_fast<WPT, BITS>(s, optf[0], w, gbits, words, um);
  for (uint32_t o = 1; o < a.n_opts; ++o) {   // OR-options (node.rs:420-438): the ask fails only if every option does
    uint32_t u[WPT];
    eval_opt_fast<WPT, BITS>(s, optf[o], w, gbits, words, u);
#pragma unroll
    for (int k = 0; k < WPT; ++k) um[k] &= u[k];
  }
#pragma unroll
  for (int k = 0; k < WPT; ++k)
    fail[k] = um[k] | (w[k].cores - a.cpu_cores) | (w[k].ram - a.ram_mb) | (w[k].storage - a.storage_gb);
}

// Slow path for an ask whose option list alone exceeds the staging capacity.
template <int WPT>
__device__ __noinline__ void eval_row_global(const EvalParams& p, const DevAsk& a,
                                             const WorkerReg (&w)[WPT], uint32_t (&f)[WPT]) {
#pragma unroll
  for (int k = 0; k < WPT; ++k) f[k] = ask_meets(a, p.opts, w[k], p.bits, p.words) ? 0xFFFFFFFFu : 0u;
}

template <int WPT>
__device__ __forceinline__ void load_workers(const EvalParams& p, uint32_t w0, uint32_t nw,
                                             uint32_t c, WorkerReg (&w)[WPT]) {
#pragma unroll
  for (int k = 0; k < WPT; ++k) {
    const uint32_t col = c + k;
    if (col < nw) {
      w[k] = make_worker(__ldg(p.wa + w0 + col), __ldg(p.wb + w0 + col));
      if (p.nacc) w[k].mmask = __ldg(p.nacc + w0 + col);
    } else w[k] = null_worker();
  }
}

// Drives `body(row_in_tile, ask, obegin, staged)` over rows [r0, r1) of the tile:
// ask headers, then as many option rows as fit, arrive in shared memory through
// 1-D TMA bulk copies signalled on one mbarrier.  With `list` the tile's rows are the asks list[t0 + r] (increasing):
// their headers are gathered by the CTA's threads, and each staged option range is the one that spans the listed
// asks (the rows between them come along unused, or the step holds fewer asks).
template <class Body>
__device__ __forceinline__ void for_each_staged_row(EvalStage& s, const EvalParams& p, bool fast,
                                                    uint32_t t0, uint32_t r0, uint32_t r1, Body&& body,
                                                    const uint32_t* __restrict__ list = nullptr) {
  const DevOpt* opt_src = fast ? reinterpret_cast<const DevOpt*>(p.opts_fast) : p.opts;
  if (threadIdx.x == 0) mbar_init(&s.bar, 1);
  const uint32_t total_words = (p.n_bits_rows)*p.words;
  if (total_words <= (uint32_t)kBitsCap)
    for (uint32_t i = threadIdx.x; i < total_words; i += blockDim.x) s.bits[i] = __ldg(p.bits + i);
  const uint32_t nrows = r1 - r0;
  if (list)
    for (uint32_t i = threadIdx.x; i < nrows; i += blockDim.x) s.ask[i] = p.asks[__ldg(list + t0 + r0 + i)];
  __syncthreads();
  uint32_t phase = 0;
  if (!list) {
    if (threadIdx.x == 0) {
      mbar_expect_tx(&s.bar, nrows * (uint32_t)sizeof(DevAsk));
      bulk_g2s(s.ask, p.asks + t0 + r0, nrows * (uint32_t)sizeof(DevAsk), &s.bar);
    }
    mbar_wait(&s.bar, phase);
    phase ^= 1u;
  }
  uint32_t row = 0;
  while (row < nrows) {
    const uint32_t obegin = s.ask[row].opt_off;
    // rows [row, row+n) whose options fit (option offsets are non-decreasing in ask order)
    const uint32_t r = row + threadIdx.x;
    const bool fits = r < nrows && (s.ask[r].opt_off + s.ask[r].n_opts - obegin) <= (uint32_t)kOptCap;
    const uint32_t n = (uint32_t)__syncthreads_count(fits);
    if (n == 0) {  // one ask with more options than the stage holds
      body(row, s.ask[row], 0u, false);
      ++row;
      continue;
    }
    const uint32_t oend = s.ask[row + n - 1].opt_off + s.ask[row + n - 1].n_opts;
    if (oend > obegin) {
      if (threadIdx.x == 0) {
        mbar_expect_tx(&s.bar, (oend - obegin) * (uint32_t)sizeof(DevOpt));
        bulk_g2s(s.opt, opt_src + obegin, (oend - obegin) * (uint32_t)sizeof(DevOpt), &s.bar);
      }
      mbar_wait(&s.bar, phase);
      phase ^= 1u;
    }
    for (uint32_t i = 0; i < n; ++i) body(row + i, s.ask[row + i], obegin, true);
    row += n;
    if (row < nrows) __syncthreads();  // everyone is done with s.opt before it is overwritten
  }
}

// ------------------------------------------------------------------ build
// grid = (ld / 1024, ceil(nt / 128)); each thread owns 4 workers in registers and walks
// the staged asks, emitting two 128-bit streaming stores per row: a warp writes 1 KB
// contiguous (two fully coalesced 512-byte stores), the CTA 8 KB contiguous per row.
// ld is a multiple of the CTA's 1024 columns (columns past the shard hold the "infeasible" pattern of a null
// worker), so the stores need no bounds test.
template <int BITS>
__global__ void __launch_bounds__(kEvalThreads, 2)
pm_build_cost(EvalParams p, uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw,
              long long* __restrict__ cost, size_t ld) {
  __shared__ EvalStage s;
  const uint32_t r0 = blockIdx.y * kEvalRows;
  const uint32_t r1 = min(nt, r0 + (uint32_t)kEvalRows);
  // A warp owns 128 consecutive columns; a lane owns the pairs (2l, 2l+1) and (64+2l, 64+2l+1), so each of
  // its two 128-bit stores per row is part of a fully coalesced 512-byte warp store (4 whole lines).
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t cbase = blockIdx.x * kEvalCols + (threadIdx.x >> 5) * 128u + lane * 2u;
  WorkerReg w[kEvalWPT];
  uint32_t gw[kEvalWPT];
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    const uint32_t col = cbase + (k >> 1) * 64u + (k & 1);
    gw[k] = w0 + col;
    if (col < nw) {
      w[k] = make_worker(__ldg(p.wa + w0 + col), __ldg(p.wb + w0 + col));
      if (p.nacc) w[k].mmask = __ldg(p.nacc + w0 + col);
    } else w[k] = null_worker();
  }
  uint4* out = reinterpret_cast<uint4*>(cost + (size_t)r0 * ld + cbase);
  const size_t row_stride = ld / 2;   // in 16-byte units; rows are visited in increasing order
  for_each_staged_row(s, p, false, t0, r0, r1, [&](uint32_t, const DevAsk& a, uint32_t obegin, bool staged) {
    uint4 v0, v1;
    // feasible: (price << 32) | worker ; infeasible: 0x7FFFFFFF_FFFFFFFF
    uint32_t f[kEvalWPT];
    if (staged) eval_row<kEvalWPT, BITS>(s, a, obegin, w, p.bits, p.words, f);
    else eval_row_global<kEvalWPT>(p, a, w, f);
    v0.x = gw[0] | ~f[0]; v0.y = (w[0].price & f[0]) | (0x7FFFFFFFu & ~f[0]);
    v0.z = gw[1] | ~f[1]; v0.w = (w[1].price & f[1]) | (0x7FFFFFFFu & ~f[1]);
    v1.x = gw[2] | ~f[2]; v1.y = (w[2].price & f[2]) | (0x7FFFFFFFu & ~f[2]);
    v1.z = gw[3] | ~f[3]; v1.w = (w[3].price & f[3]) | (0x7FFFFFFFu & ~f[3]);
    __stcs(out, v0);
    __stcs(out + 32, v1);     // + 64 columns
    out += row_stride;
  });
}

// ------------------------------------------------------------------ build, fast form
// Same decomposition and output as pm_build_cost, for tables that fit the fast predicate.  Built so that warps do not
// wait on chained shared-memory loads — ask -> its option -> the option's acceptance word — or on the previous row's
// store reading its registers:
//   * one FastRow per ask: everything a single-option ask needs in three 128-bit loads whose address depends only on
//     the row number; the rows of the CTA arrive by ONE 1-D TMA bulk copy;
//   * the next row's FastRow is loaded while the current row is evaluated (explicit double buffer in registers);
//   * further OR-options (one ask in ten) are read straight from global memory, warp-uniform and L1-resident.
template <int WPT, int BITS>
__device__ __forceinline__ void eval_fast_first(const FastRow& q, const uint32_t* sbits, const WorkerReg (&w)[WPT],
                                                const uint32_t* __restrict__ gbits, uint32_t words, uint32_t (&u)[WPT]) {
#pragma unroll
  for (int k = 0; k < WPT; ++k) {
    const uint32_t word = (BITS == 2) ? q.wp
                          : (BITS == 1) ? sbits[q.wp * words + w[k].mword] : __ldg(gbits + q.wp * words + w[k].mword);
    const uint32_t z = ((w[k].key & q.m) ^ q.v) | (~word & w[k].mmask);
    const uint32_t r = (w[k].mem_eff - q.mem_lo) | (q.mem_hi - w[k].mem_eff) |
                       (((w[k].tot - q.tot_lo) | (q.tot_hi - w[k].tot)) & w[k].tot_keep);
    u[k] = (0u - z) | r;
  }
}

template <int WPT, int BITS>
__device__ __forceinline__ void eval_fast_more(const DevOptF* __restrict__ gopts, uint32_t n_more, const uint32_t* sbits,
                                               const WorkerReg (&w)[WPT], const uint32_t* __restrict__ gbits,
                                               uint32_t words, uint32_t (&um)[WPT]) {
  for (uint32_t o = 0; o < n_more; ++o) {
    const uint4 q0 = __ldg(reinterpret_cast<const uint4*>(gopts + o));
    const uint4 q1 = __ldg(reinterpret_cast<const uint4*>(gopts + o) + 1);   // {tot_lo, tot_hi, pattern_row, pad}
    const uint32_t uword = (BITS == 2) ? __ldg(gbits + q1.z) : 0u;
#pragma unroll
    for (int k = 0; k < WPT; ++k) {
      const uint32_t word = (BITS == 2) ? uword
                            : (BITS == 1) ? sbits[q1.z * words + w[k].mword] : __ldg(gbits + q1.z * words + w[k].mword);
      const uint32_t z = ((w[k].key & q0.x) ^ q0.y) | (~word & w[k].mmask);
      const uint32_t r = (w[k].mem_eff - q0.z) | (q0.w - w[k].mem_eff) |
                         (((w[k].tot - q1.x) | (q1.y - w[k].tot)) & w[k].tot_keep);
      um[k] &= (0u - z) | r;
    }
  }
}

constexpr int kFastRows = 512;   // asks per CTA: the prologue (worker rows from L2, the TMA of the FastRows) is paid once per CTA
struct __align__(128) FastStage {
  FastRow row[kFastRows + 2];   // + 2: the look-ahead loads of the last pair of rows may read past it (never used)
  uint32_t bits[kBitsCap];
  uint64_t bar;
};

// FOLD (pm_build_argmin): the 32-bit tile, folded in the kernel that writes it.  The tile holds only the 32-bit cost
// word — the worker's price when feasible, kNarrowInfeasible when not — and `tile` is uint32_t[rows][ld].  The worker
// index the int64 element carries in its low word is the column (+ w0): 4 B per evaluation instead of 8.  A lane then
// owns the 4 consecutive columns 4l .. 4l+3 of its warp's 128, so each row is one 16-byte store per thread, 512 B per
// warp and 4 KB per CTA, contiguous.  Only for tables whose every price is below kNarrowInfeasible
// (pm_check_worker_ranges): at that price a feasible worker could not be told from the sentinel, and at >= 2^31 the
// int64 tile's signed order differs.  The CTA also folds each row's minimum and feasible count from the registers it
// stores — see pm_build_argmin.  Without FOLD (pm_build_cost_fast) the tile is the int64 one and `fo` is unused.
struct FoldOut {
  const uint32_t* rank;            // [ld] each column's rank within its 1024-column stripe (pm_stripe_rank)
  const long long* best_of_rank;   // [ld] stripe s, rank ρ at s * 1024 + ρ: that column's (price << 32) | (w0 + worker)
  uint32_t* first_ask;
  long long* ask_best;
  uint32_t* ask_count;
  const uint32_t* perm;            // pm_build_argmin_feat: [ld] column -> worker offset (pm_feature_keys); else unused
};

// Two rows per iteration share the loop test and the output-pointer bump.  Each row (q[r], emitted to `out` + r rows)
// is loaded one row ahead, into registers the previous row has finished with, so no row is copied from one buffer to
// another; q holds two entries past the last row for the look-ahead loads of the last pair (never used).
template <class Row, class Emit>
__device__ __forceinline__ void for_each_row_pair(const Row* q, uint32_t nrows, uint4* out, size_t row_stride,
                                                  Emit&& emit) {
  Row a = q[0];
  for (uint32_t r = 0; r < nrows; r += 2, q += 2) {
    const Row b = q[1];                       // in flight while row r is evaluated
    emit(a, out, r);
    a = q[2];                                 // in flight while row r + 1 is evaluated
    if (r + 1 < nrows) emit(b, out + row_stride, r + 1);
    out += 2 * row_stride;
  }
}

// The row fold of the two build + argmin kernels (pm_build_argmin, pm_build_argmin_feat).  Per warp and row of the
// CTA, the warp's least key (the least stripe rank of its feasible columns, or kNoRank and more when it has none) and
// its infeasible columns are kept in s_key / s_nb[warp][row] — plain stores, no atomics; 12 KB at 512 rows.
constexpr int kFoldWarps = kEvalThreads / 32;
constexpr uint32_t kNoRank = 0x8000u;   // added to an infeasible column's rank (< 1024): the key still fits 16 bits

// The warp's key and infeasible count of row r, stored in its slot of the row (key_slot / nb_slot: the warp's row 0,
// shared-window addresses).  Every lane stores the same value to the same address: one store each, without a branch
// around lane 0.
__device__ __forceinline__ void fold_slot(uint32_t key, uint32_t nb, uint32_t key_slot, uint32_t nb_slot, uint32_t r) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(key_slot + 2u * r), "r"(key) : "memory");
  asm volatile("st.shared.u8 [%0], %1;" ::"r"(nb_slot + r), "r"(nb) : "memory");
}

// Row r's lane keys and infeasible counts over the warp's 128 columns: one reduction each, stored in the warp's slot
// of the row.  Returns the warp's infeasible count.
__device__ __forceinline__ uint32_t fold_row(uint32_t key, uint32_t nb, uint32_t key_slot, uint32_t nb_slot, uint32_t r) {
  key = __reduce_min_sync(0xffffffffu, key);
  nb = __reduce_add_sync(0xffffffffu, nb);
  fold_slot(key, nb, key_slot, nb_slot, r);
  return nb;
}

// End of the CTA's rows: each row with a feasible column merges best_of_rank[its least rank] into ask_best and its
// feasible count into ask_count, at its ask: at(p, i) is row i's entry of the per-ask array p.  row_done(i, m, pr) sees every row i < nrows with m's bit j set
// when warp j's 128 columns of the row are all infeasible, and pr's when they are all feasible.  A row for which
// live(i) is false has no feasible column and its warps wrote no slots: it merges nothing, and row_done sees every bit
// of m set and none of pr.
template <int ROWS, class RowLive, class RowAt, class RowDone>
__device__ __forceinline__ void fold_merge_rows(const uint16_t (&s_key)[kFoldWarps][ROWS],
                                                const uint8_t (&s_nb)[kFoldWarps][ROWS], uint32_t nrows,
                                                const FoldOut& fo, RowLive&& live, RowAt&& at, RowDone&& row_done) {
  __syncthreads();                            // every warp has written its slot of every live row
  const long long* best = fo.best_of_rank + blockIdx.x * kEvalCols;
  for (uint32_t i = threadIdx.x; i < nrows; i += kEvalThreads) {
    if (!live(i)) {
      row_done(i, (1u << kFoldWarps) - 1u, 0u);
      continue;
    }
    uint32_t key = kNone, nb = 0, m = 0, pr = 0;
#pragma unroll
    for (int j = 0; j < kFoldWarps; ++j) {
      key = min(key, (uint32_t)s_key[j][i]);
      nb += s_nb[j][i];
      m |= (uint32_t)(s_nb[j][i] == 128u) << j;
      pr |= (uint32_t)(s_nb[j][i] == 0u) << j;
    }
    row_done(i, m, pr);
    if (nb < (uint32_t)kEvalCols) {           // a feasible column: key is its least rank
      atomicMin(at(fo.ask_best, i), __ldg(best + key));
      atomicAdd(at(fo.ask_count, i), kEvalCols - nb);
    }
  }
}

// Per column cbase + k of the thread, its first feasible ask cm[k] (>= 2^31 while there is none) into first_ask of the
// column's worker: w0 + the column, or with PERM w0 + perm[column] (pm_build_argmin_feat's column order; perm is loaded
// only now: held through the row loop it would cost 4 registers there).
template <bool PERM>
__device__ __forceinline__ void fold_flush_first_ask(const uint32_t (&cm)[kEvalWPT], uint32_t cbase, uint32_t w0,
                                                     uint32_t nw, const FoldOut& fo) {
  uint32_t* first = fo.first_ask + w0;
  uint32_t wk[kEvalWPT];   // column cbase + k's worker, as an offset from `first`
  if constexpr (PERM) {
    const uint4 pw = __ldg(reinterpret_cast<const uint4*>(fo.perm + cbase));
    wk[0] = pw.x; wk[1] = pw.y; wk[2] = pw.z; wk[3] = pw.w;
  } else {   // the thread's 4 consecutive columns: constant offsets from first + cbase
    first += cbase;
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) wk[k] = k;
  }
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k)
    if (cm[k] < 0x80000000u && cbase + k < nw) atomicMin(first + wk[k], cm[k]);
}

template <int BITS, bool FOLD>
__device__ __forceinline__ void build_fast(const EvalParams& p, uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw,
                                           void* __restrict__ tile, size_t ld, const FoldOut& fo) {
  __shared__ FastStage s;
  __shared__ uint16_t s_key[FOLD ? kFoldWarps : 1][FOLD ? kFastRows : 1];
  __shared__ uint8_t s_nb[FOLD ? kFoldWarps : 1][FOLD ? kFastRows : 1];
  const uint32_t r0 = blockIdx.y * kFastRows;
  const uint32_t nrows = min(nt - r0, (uint32_t)kFastRows);
  if (threadIdx.x == 0) {
    mbar_init(&s.bar, 1);
    mbar_expect_tx(&s.bar, nrows * (uint32_t)sizeof(FastRow));
    bulk_g2s(s.row, p.frows + t0 + r0, nrows * (uint32_t)sizeof(FastRow), &s.bar);
  }
  if (BITS == 1) {
    const uint32_t total_words = p.n_bits_rows * p.words;
    for (uint32_t i = threadIdx.x; i < total_words; i += blockDim.x) s.bits[i] = __ldg(p.bits + i);
  }
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t cbase = blockIdx.x * kEvalCols + (threadIdx.x >> 5) * 128u + lane * (FOLD ? 4u : 2u);
  WorkerReg w[kEvalWPT];
  uint32_t gw[kEvalWPT], dx[kEvalWPT], dy[kEvalWPT];
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    const uint32_t col = FOLD ? cbase + k : cbase + (k >> 1) * 64u + (k & 1);
    gw[k] = w0 + col;
    if (col < nw) {
      w[k] = make_worker(__ldg(p.wa + w0 + col), __ldg(p.wb + w0 + col));
      if (p.nacc) w[k].mmask = __ldg(p.nacc + w0 + col);
    } else w[k] = null_worker();
    dx[k] = 0xFFFFFFFFu - gw[k];          // infeasible: 0x7FFFFFFF_FFFFFFFF = feasible word + (0/1) * difference
    dy[k] = 0x7FFFFFFFu - w[k].price;     // (the 32-bit tile keeps only this high word)
    asm("" : "+r"(dy[k]));                // kept in a register: ptxas would otherwise recompute it from the price every row
  }
  uint4* out = FOLD ? reinterpret_cast<uint4*>(static_cast<uint32_t*>(tile) + (size_t)r0 * ld + cbase)
                    : reinterpret_cast<uint4*>(static_cast<long long*>(tile) + (size_t)r0 * ld + cbase);
  size_t row_stride = FOLD ? ld / 4 : ld / 2;   // in 16-byte units
  asm("" : "+l"(row_stride));           // held in registers: ptxas would otherwise re-derive it from `ld` every row
  const uint32_t sh = p.sign_shift;
  // FOLD: per column, the first feasible ask so far — the least of ask | fail's sign bit (asks are below 2^31): >= 2^31
  // while there is none
  uint32_t cm[kEvalWPT];
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) cm[k] = kNone;
  const uint32_t t_cta = t0 + r0;       // FOLD: the ask of the CTA's first row
  uint32_t rk[kEvalWPT];                // FOLD: per column, its rank within the stripe
  uint32_t key_slot = 0, nb_slot = 0;   // FOLD: the warp's row 0 in s_key / s_nb (shared-window addresses)
  if constexpr (FOLD) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(fo.rank + cbase));
    rk[0] = v.x; rk[1] = v.y; rk[2] = v.z; rk[3] = v.w;
    key_slot = (uint32_t)__cvta_generic_to_shared(&s_key[threadIdx.x >> 5][0]);
    nb_slot = (uint32_t)__cvta_generic_to_shared(&s_nb[threadIdx.x >> 5][0]);
    asm("" : "+r"(key_slot), "+r"(nb_slot));   // held in registers: ptxas would otherwise re-derive them every row
  }
  // One row (`r` of the CTA).  The ask's scalar thresholds are OR-ed into the first option's clauses before the further
  // OR-options are AND-ed in — fail = AND_o(u_o | s) = (AND_o u_o) | s — so a single-option row is one 7-term OR per worker.
  auto emit = [&](const FastRow& q, uint4* dst, uint32_t r) {
    uint32_t f[kEvalWPT], sc[kEvalWPT];
    eval_fast_first<kEvalWPT, BITS>(q, s.bits, w, p.bits, p.words, f);
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) {
      sc[k] = (w[k].cores - q.cpu_cores) | (w[k].ram - q.ram_mb) | (w[k].storage - q.storage_gb);
      f[k] |= sc[k];
    }
    if (q.n_opts > 1u) {   // OR-options (node.rs:420-438), one ask in ten: the ask fails only if every option does
      uint32_t um[kEvalWPT];
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) um[k] = 0xFFFFFFFFu;
      eval_fast_more<kEvalWPT, BITS>(p.opts_fast + q.opt_off + 1, q.n_opts - 1u, s.bits, w, p.bits, p.words, um);
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) f[k] &= um[k] | sc[k];
    }
    uint32_t o[2 * kEvalWPT];
    uint32_t key = kNone, nb = 0;       // FOLD: the lane's least key and its infeasible columns
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) {
      const uint32_t b = f[k] >> sh;                                    // 1 when infeasible (sh == 31)
      if (FOLD) {
        o[k] = b * dy[k] + w[k].price;                                  // feasible: price ; infeasible: kNarrowInfeasible
        cm[k] = min(cm[k], (t_cta + r) | (f[k] & 0x80000000u));        // the ask, + 2^31 when infeasible
        key = min(key, b * kNoRank + rk[k]);                            // the rank, + kNoRank when infeasible
        nb += b;
      } else {
        o[2 * k] = b * dx[k] + gw[k];                                   // feasible: (price << 32) | worker
        o[2 * k + 1] = b * dy[k] + w[k].price;                          // infeasible: 0x7FFFFFFF_FFFFFFFF
      }
    }
    __stcs(dst, make_uint4(o[0], o[1], o[2], o[3]));
    if (FOLD) fold_row(key, nb, key_slot, nb_slot, r);
    else __stcs(dst + 32, make_uint4(o[4], o[5], o[6], o[7]));     // + 64 columns
  };
  __syncthreads();            // mbarrier initialised, acceptance words staged
  mbar_wait(&s.bar, 0);
  for_each_row_pair(s.row, nrows, out, row_stride, emit);
  if constexpr (FOLD) {
    fold_merge_rows(s_key, s_nb, nrows, fo, [](uint32_t) { return true; }, [&](auto* a, uint32_t i) { return a + t_cta + i; },
                    [](uint32_t, uint32_t, uint32_t) {});
    fold_flush_first_ask<false>(cm, cbase, w0, nw, fo);
  }
}

template <int BITS>
__global__ void __launch_bounds__(kEvalThreads, 2)
pm_build_cost_fast(EvalParams p, uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw, long long* __restrict__ tile,
                   size_t ld) {
  build_fast<BITS, false>(p, t0, nt, w0, nw, tile, ld, FoldOut{});
}

// ------------------------------------------------------------------ build + argmin, one kernel
// The 32-bit tile's build and the int64 pm_argmin's outputs in one pass: the tile is written with streaming stores,
// as the build writes it, and never read back.  Within a 1024-column stripe the packed minimum
// (word << 32) | (w0 + column) over the feasible columns orders them by (price, column) whatever the ask, so a
// column's rank in that order (pm_stripe_rank, once per pass) stands for its packed cost.  Per row and lane the
// fold is one multiply-add per column on the fail bit the store already formed — key = b * kNoRank + rank — the
// least of the 4 keys and the sum of the bits; per warp one min and one add reduction, stored in the warp's slot of
// the row (no atomics, no barrier in the row loop).  At the end of the CTA each row with a feasible column merges
// best_of_rank[its least rank] into ask_best (atomicMin) and its count into ask_count; per column the first feasible
// ask, kept from the same sign bit, is flushed once.  The outputs are those of pm_build_cost_fast and pm_argmin on
// the int64 tile, bit for bit.
template <int BITS>
__global__ void __launch_bounds__(kEvalThreads, 2)
pm_build_argmin(EvalParams p, uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw, uint32_t* __restrict__ tile, size_t ld,
                FoldOut fo) {
  build_fast<BITS, true>(p, t0, nt, w0, nw, tile, ld, fo);
}

// One CTA per 1024-column stripe of a tile with leading dimension ld, whose column c holds worker w0 + perm[c]
// (w0 + c when perm is null): sorts the stripe's columns by (price, worker) — the order of the packed cost
// (price << 32) | (w0 + worker) — and writes rank[c], each column's place in that order (padding columns at or past
// nw last), and best_of_rank[stripe * 1024 + ρ], the packed cost of the column at place ρ (kInf for padding, which is
// never feasible).  Prices are below 2^31 wherever the 32-bit tile runs, so a key is (price << 32) | worker in 63
// bits, and padding's all-ones key sorts past every one; the column is the sorted value.
__global__ void __launch_bounds__(kEvalThreads)
pm_stripe_rank(const uint4* __restrict__ wb, const uint32_t* __restrict__ perm, uint32_t w0, uint32_t nw,
               uint32_t* __restrict__ rank, long long* __restrict__ best_of_rank) {
  using Sort = cub::BlockRadixSort<unsigned long long, kEvalThreads, kEvalWPT, uint32_t>;
  __shared__ typename Sort::TempStorage tmp;
  const uint32_t c0 = blockIdx.x * kEvalCols;
  unsigned long long key[kEvalWPT];
  uint32_t col[kEvalWPT];
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    const uint32_t c = threadIdx.x * kEvalWPT + k;
    col[k] = c;
    key[k] = ~0ull;
    if (c0 + c < nw) {
      const uint32_t w = perm ? __ldg(perm + c0 + c) : c0 + c;
      key[k] = ((unsigned long long)__ldg(&wb[w0 + w].w) << 32) | w;
    }
  }
  Sort(tmp).Sort(key, col, 0, 64);   // blocked: thread i holds places 4i .. 4i + 3
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    const uint32_t rho = threadIdx.x * kEvalWPT + k;
    rank[c0 + col[k]] = rho;
    best_of_rank[c0 + rho] = key[k] == ~0ull ? kInf : (long long)(((key[k] >> 32) << 32) | (w0 + (uint32_t)key[k]));
  }
}

// Worker-major acceptance: bit r of nacc[w] is set when pattern row r rejects worker w's model (row 0 never does).
__device__ __forceinline__ uint32_t worker_nacc(const uint4& a, const uint32_t* __restrict__ bits, uint32_t words,
                                                uint32_t n_rows) {
  const uint32_t mid = (a.w & PM_W_HAS_GPU_MODEL) ? a.z : 0u;
  const uint32_t mword = mid / kModelsPerWord, mmask = 1u << (mid % kModelsPerWord);
  uint32_t rej = 0;
  for (uint32_t r = 1; r < n_rows; ++r)
    if (!(__ldg(bits + (size_t)r * words + mword) & mmask)) rej |= 1u << r;
  return rej;
}
__global__ void pm_worker_nacc(const uint4* __restrict__ wa, const uint32_t* __restrict__ bits, uint32_t words, uint32_t n_rows,
                               uint32_t n, uint32_t* __restrict__ nacc) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  nacc[i] = worker_nacc(wa[i], bits, words, n_rows);
}
// ... for the listed rows only (an incremental pass: the other rows' words are still those of the table in force)
__global__ void pm_worker_nacc_rows(const uint4* __restrict__ wa, const uint32_t* __restrict__ bits, uint32_t words,
                                    uint32_t n_rows, const uint32_t* __restrict__ rows, uint32_t n,
                                    uint32_t* __restrict__ nacc) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t w = rows[i];
  nacc[w] = worker_nacc(wa[w], bits, words, n_rows);
}

// `wp` of every FastRow: the first option's acceptance WORD when rows are one word wide, else its pattern row.
__global__ void pm_bind_rows(FastRow* __restrict__ rows, const DevOptF* __restrict__ opts_fast,
                             const uint32_t* __restrict__ bits, uint32_t words, uint32_t n_asks) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  const uint32_t prow = opts_fast[rows[t].opt_off].pattern_row;
  rows[t].wp = words == 1u ? bits[prow] : prow;
}

// ------------------------------------------------------------------ build + argmin, feature form
// Every clause of the fast predicate compares one worker operand with one threshold of the ask table, and a table has
// few distinct thresholds.  A FEATURE is one such (clause, threshold) pair; a worker's answer to each of them is
// computed once per pass, into the 64-bit word F[w], and each OR-option o of an ask gets the mask R_o of the features
// it requires, with the ask's own scalar clauses OR-ed in.  Then "worker w fails option o" is u_o = R_o & ~F[w] != 0
// (folded to 32 bits as lo | hi) and "w fails the ask" is min_o u_o != 0 — a minimum, not an AND: two failing options
// may miss different features: no threshold in the row loop (DESIGN §3).
// The features of a kind (on the fast domain each equals the sign test eval_fast_first makes):
//   kFeatKey      presence bit j of `key` (values j < 13)      kFeatCount   count_eff == c
//   kFeatModel    pattern row r accepts the worker's model     kFeatMemLo / kFeatMemHi   mem_eff >= lo / <= hi
//   kFeatTotLo / kFeatTotHi   !tot_keep || tot >= lo / <= hi   kFeatCores / kFeatRam / kFeatStorage   >= threshold
// Thresholds that every worker meets (lo 0, hi 0x7FFFFFFF) are no feature.  The candidate and never bits are always
// features: every row requires the first, and toggling an ask sets the second without converting the table again.
enum FeatKind : uint32_t {
  kFeatKey = 0, kFeatCount, kFeatModel, kFeatMemLo, kFeatMemHi, kFeatTotLo, kFeatTotHi, kFeatCores, kFeatRam, kFeatStorage,
  kFeatKinds
};
constexpr uint32_t kFeatMax = 64;     // features of the 64-bit word
constexpr uint32_t kFeatSlots = 64;   // distinct values collected per kind (more cannot fit the word anyway)
constexpr uint32_t kKeyPresence = 13; // key bits 0..12 are presence bits, the gpu count follows

// The dictionary, a kernel parameter: the features of kind k are val[off[k] .. off[k + 1]), increasing, and a
// feature's bit in F / R is its index.
struct FeatDict {
  uint32_t off[kFeatKinds + 1];
  uint32_t val[kFeatMax];
};

// Collection, after pm_ask_convert: buf[0] = the key bits some row requires, buf[1] = overflow (more than kFeatSlots
// values of a kind, or a value equal to the empty slot), buf[2 + (k - 1) * kFeatSlots ..] = the distinct values of
// kind k >= 1 in a table with linear probing, kNone = empty.
__device__ __forceinline__ void feat_insert(uint32_t* __restrict__ buf, uint32_t k, uint32_t v) {
  uint32_t* slots = buf + 2 + (k - 1) * kFeatSlots;
  if (v == kNone) { atomicOr(buf + 1, 1u); return; }
  uint32_t h = (v * 0x9E3779B1u) >> 26;   // 6 bits
  for (uint32_t i = 0; i < kFeatSlots; ++i, h = (h + 1) & (kFeatSlots - 1)) {
    uint32_t cur = *reinterpret_cast<volatile uint32_t*>(slots + h);
    if (cur == kNone) cur = atomicCAS(slots + h, kNone, v);
    if (cur == kNone || cur == v) return;
  }
  atomicOr(buf + 1, 1u);
}

// Calls fn(kind, value) for every feature option `f` requires (the scalar clauses are the ask's: kFeatCores ..).
template <class Fn>
__device__ __forceinline__ void opt_features(const DevOptF& f, Fn&& fn) {
  const uint32_t pres = f.m & ((1u << kKeyPresence) - 1u);
  for (uint32_t j = 0; j < kKeyPresence; ++j)
    if ((pres >> j) & 1u) fn(kFeatKey, j);
  if (f.m >> kKeyPresence) fn(kFeatCount, (f.v >> kKeyCountShift) & 0xFFFFu);
  if (f.pattern_row) fn(kFeatModel, f.pattern_row);
  if (f.mem_lo) fn(kFeatMemLo, f.mem_lo);
  if (f.mem_hi < 0x7FFFFFFFu) fn(kFeatMemHi, f.mem_hi);
  if (f.tot_lo) fn(kFeatTotLo, f.tot_lo);
  if (f.tot_hi < 0x7FFFFFFFu) fn(kFeatTotHi, f.tot_hi);
}
template <class Fn>
__device__ __forceinline__ void ask_features(const FastRow& q, Fn&& fn) {
  if (q.cpu_cores) fn(kFeatCores, q.cpu_cores);
  if (q.ram_mb) fn(kFeatRam, q.ram_mb);
  if (q.storage_gb) fn(kFeatStorage, q.storage_gb);
}

__global__ void pm_feature_collect(const FastRow* __restrict__ frows, const DevOptF* __restrict__ opts_fast, uint32_t n_asks,
                                   uint32_t* __restrict__ buf) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  const FastRow q = frows[t];
  uint32_t pres = 0;
  auto add = [&](uint32_t k, uint32_t v) {
    if (k == kFeatKey) pres |= 1u << v;
    else feat_insert(buf, k, v);
  };
  ask_features(q, add);
  for (uint32_t o = 0; o < q.n_opts; ++o) opt_features(opts_fast[q.opt_off + o], add);
  if (pres & ~*reinterpret_cast<volatile uint32_t*>(buf)) atomicOr(buf, pres);
}

__device__ __forceinline__ unsigned long long feat_bit(const FeatDict& d, uint32_t k, uint32_t v) {
  for (uint32_t i = d.off[k]; i < d.off[k + 1]; ++i)
    if (d.val[i] == v) return 1ull << i;
  return 0ull;   // unreachable: the dictionary holds every value of the converted table (and the never bit)
}

// Per pass, in stream order: per ask {R_0 lo, R_0 hi, n_opts, opt_off} and per option row R_o (scalar bits included).
// Reading the converted rows of this pass, a toggle or a rebind needs nothing else.
__global__ void pm_feature_asks(const FastRow* __restrict__ frows, const DevOptF* __restrict__ opts_fast, uint32_t n_asks,
                                FeatDict d, uint4* __restrict__ arow, uint2* __restrict__ ropt) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  const FastRow q = frows[t];
  unsigned long long s = 0;
  ask_features(q, [&](uint32_t k, uint32_t v) { s |= feat_bit(d, k, v); });
  for (uint32_t o = 0; o < q.n_opts; ++o) {
    unsigned long long r = s;
    opt_features(opts_fast[q.opt_off + o], [&](uint32_t k, uint32_t v) { r |= feat_bit(d, k, v); });
    if (o == 0) arow[t] = make_uint4((uint32_t)r, (uint32_t)(r >> 32), q.n_opts, q.opt_off);
    else ropt[q.opt_off + o] = make_uint2((uint32_t)r, (uint32_t)(r >> 32));
  }
}

// The column order of pm_build_argmin_feat's tile.  Its infeasible words (kNarrowInfeasible) are what compressible
// memory stores compactly, but only in aligned blocks whose words are all equal, and in worker order a row's
// feasible columns are scattered.  So each pass sorts the workers of [w0, w0 + nw) by __brevll(F), stably: workers
// with the same F are adjacent, and F's first features (the dictionary's candidate and presence bits, then gpu count
// and model) vary slowest, so a typical ask's feasible workers become a few dozen runs of columns and nearly every
// other block of its row is uniform.  Column c < nw then holds worker w0 + perm[c]; the padding columns [nw, ld) stay
// at the end, null workers, perm[c] = c.
//
// Step 1, per pass in stream order: per index c of [0, ld) the key __brevll(F) of worker w0 + c (a null worker past
// nw: it lacks the candidate bit every row requires) and the value c, for cub::DeviceRadixSort over [0, nw).  The
// padding entries are written to the sort's output too, which the sort fills only below nw.  `bits` is the acceptance
// table in its own form, `words` per row, whichever form the other kernels read.
__global__ void pm_feature_keys(const uint4* __restrict__ wa, const uint4* __restrict__ wb, const uint32_t* __restrict__ bits,
                                uint32_t words, uint32_t w0, uint32_t nw, size_t ld, FeatDict d,
                                unsigned long long* __restrict__ key, uint32_t* __restrict__ val,
                                unsigned long long* __restrict__ key_sorted, uint32_t* __restrict__ perm) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ld) return;
  const WorkerReg w = c < nw ? make_worker(__ldg(wa + w0 + c), __ldg(wb + w0 + c)) : null_worker();
  unsigned long long F = 0;
  for (uint32_t k = 0; k < kFeatKinds; ++k)
    for (uint32_t i = d.off[k]; i < d.off[k + 1]; ++i) {
      const uint32_t v = d.val[i];
      bool b;
      switch (k) {
        case kFeatKey: b = (w.key >> v) & 1u; break;
        case kFeatCount: b = w.count_eff == v; break;
        case kFeatModel: b = (__ldg(bits + (size_t)v * words + w.mword) & w.mmask) != 0u; break;
        case kFeatMemLo: b = w.mem_eff >= v; break;
        case kFeatMemHi: b = w.mem_eff <= v; break;
        case kFeatTotLo: b = !w.tot_keep || w.tot >= v; break;
        case kFeatTotHi: b = !w.tot_keep || w.tot <= v; break;
        case kFeatCores: b = w.cores >= v; break;
        case kFeatRam: b = w.ram >= v; break;
        default: b = w.storage >= v; break;
      }
      F |= (unsigned long long)b << i;
    }
  key[c] = __brevll(F);
  val[c] = c;
  if (c >= nw) {
    key_sorted[c] = __brevll(F);
    perm[c] = c;
  }
}

// Step 3, after the sort and pm_stripe_rank over the sorted columns: per column c of [0, ld) {F lo, F hi, price,
// stripe rank} of its worker w0 + perm[c], the 16 B pm_build_argmin_feat's prologue reads.
__global__ void pm_feature_gather(const uint4* __restrict__ wb, const unsigned long long* __restrict__ key_sorted,
                                  const uint32_t* __restrict__ perm, const uint32_t* __restrict__ rank, uint32_t w0,
                                  uint32_t nw, size_t ld, uint4* __restrict__ feat) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ld) return;
  const unsigned long long F = __brevll(key_sorted[c]);
  const uint32_t price = c < nw ? __ldg(&wb[w0 + perm[c]].w) : 0u;   // the null worker's price
  feat[c] = make_uint4((uint32_t)F, (uint32_t)(F >> 32), price, rank[c]);
}

// The slot schedule of pm_build_argmin_feat's launches.  A pass over T asks in tiles of `rows` row slots writes each
// slot once per launch, and the blocks it stores are the transitions: a block that held the sentinel or the prices for
// the slot's last ask and does not for this one.  In natural order a slot's successive asks t and t + rows are
// unrelated, so most stores are transitions; the outputs do not depend on which asks share a launch (atomic min and
// add per ask, a per-column minimum of asks), so the launches take the asks in an order that makes them rare.
//
// The contract of the buffer (PM_BUF_COST_TILE) is what the natural order leaves: slot i holds ask a of [T - rows, T)
// with a % rows == i.  Those final writers form the last launch, in slot order.  The other M = T - rows asks are
// sorted by (__brevll(R_0), ask) — R_0 the first option's requirement mask, its first features varying slowest, as the
// column order's key — into S, and laid out slot-major over Ks = ceil(M / rows) launches: slot r of launch k holds
// S[r * Ks + k], so a slot's successive asks are neighbours in S, and launch k covers the slots r < ceil((M - k) / Ks),
// a prefix.  The launches stay ceil(T / rows).  The rows go in write order into srow (R_0 lo, R_0 hi, n_opts,
// opt_off, as feat_a) and sask (the ask): launch k's at base_k = k * a + min(k, b) with M = a * Ks + b, the last at M.
// With at most two tiles each slot is written at most twice a pass: the schedule is the natural order (Ks = 0).
//
// Key step, per pass in stream order: asks [0, M) keyed for cub::DeviceRadixSort.
__global__ void pm_sched_keys(const uint4* __restrict__ arow, uint32_t m, unsigned long long* __restrict__ key,
                              uint32_t* __restrict__ val) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const uint4 q = arow[t];
  key[t] = __brevll((unsigned long long)q.y << 32 | q.x);
  val[t] = t;
}

// Gather step: write position p of [0, T) from the sorted asks (Ks > 0) or the natural order (Ks = 0).
__global__ void pm_sched_gather(const uint4* __restrict__ arow, const uint32_t* __restrict__ sorted, uint32_t n_asks,
                                uint32_t rows, uint32_t ks, uint4* __restrict__ srow, uint32_t* __restrict__ sask) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_asks) return;
  uint32_t t = p;
  if (ks) {
    const uint32_t m = n_asks - rows;
    if (p >= m) {   // the last launch: slot i's final writer, row i of the last tile or of the one before it
      const uint32_t i = p - m, t_last = (n_asks - 1) / rows * rows;
      t = i < n_asks - t_last ? t_last + i : t_last - rows + i;
    } else {        // launch k's slot r: launches k < b take a + 1 slots, the others a
      const uint32_t a = m / ks, b = m % ks, big = b * (a + 1);
      const uint32_t k = p < big ? p / (a + 1) : b + (p - big) / a;
      const uint32_t r = p < big ? p % (a + 1) : (p - big) % a;
      t = sorted[r * ks + k];
    }
  }
  srow[p] = arow[t];
  sask[p] = t;
}

// pm_build_argmin with the feature predicate: the same stores, row fold, first-ask minimum and end-of-CTA merge
// (build_fast<.., true>), the outputs bit for bit, on a tile whose column c holds worker w0 + perm[c] (the
// column order above; the ranks and best_of_rank carry the workers, and first_ask is flushed to them).  A warp first
// decides its 128 columns of a row as a whole (dead or full, from the OR and AND of their F); only a mixed block is
// evaluated per worker: two LOP3 for u = R & ~F over the two words and one min for the fail bit b = min(u, 1).
// A worker is one 16-byte load in the prologue; a row is one 16-byte shared-memory load; further OR-options (R_o) are
// read from global memory, warp-uniform.
//
// The CTA's rows are positions t0 + r0 + i of the slot schedule (pm_sched_gather): their requirement rows come from
// srow, their asks from sask, and row i goes to tile slot r0 + i.
//
// `held` (TileBuf::held) has one byte per row slot and 1024-column stripe of the tile, at slot * (ld / 1024) + stripe:
// bit j set when warp j's 512-byte block of it holds kNarrowInfeasible in every word.  `priced` (TileBuf::priced),
// indexed the same way, has bit j set when the block holds this pass's price of each of its columns in every word —
// what a row feasible in all 128 columns stores; it is zeroed at every pass start, as column order and prices may
// change between passes.  A block's two bits are never both set.  Most blocks are all infeasible row after row (the
// column order), and in the scheduled order a slot's next ask usually needs what the last one did, so a warp stores its
// block only when some word changes: unless the row is infeasible there and the held bit set, or feasible in every
// column and the priced bit set.  The tile stays what the stores would have made it.  The CTA reads its rows' bytes in
// the prologue and writes back those that change after the merge; each byte belongs to one CTA of a launch, and
// launches are stream-ordered.
//
// Most rows have nothing to do in the whole stripe, and the column order makes that knowable for the CTA at once: So,
// the OR of the 8 warps' Fo, is nearly as selective as each Fo.  Once the rows have landed, one thread per row triages
// it: if R_o & ~So != 0 for every option, every block of the row is dead (each Fo ⊆ So).  Such a row is SKIP when its
// map byte is 0xFF (every block already holds the sentinel: no store, no slot, no fold, no byte to write) and
// SENTINEL otherwise (each warp whose bit is clear stores the sentinel block; the byte becomes 0xFF and the priced
// byte 0).  Every other row
// is LIVE and runs the per-block code.  The LIVE and SENTINEL rows are compacted, in increasing order, into two lists
// the warps walk; the merge takes no slot of a row that is not LIVE.
//
// A CTA takes 256 rows, not the FastRow kernels' 512.  Chosen while the scattered store stream bound the kernel (cfg3,
// H100 SXM, 700 W, per step in this kernel: 45.6 ms at 512 rows, 29.1 at 256, 32.0 at 128, 12.7 with its stores
// removed), and kept with the slot schedule, which stores few blocks: cfg3 steps of 17.3 ms at 256 rows and 3 CTAs/SM,
// 17.6 at 512 rows and 3, 18.1 at 256 and 2, 19.9 at 512 and 2 (one session, 10 steps each); then 16.7 at 256 rows
// and 4 CTAs/SM against 17.1-17.3 at 3 (20 steps each), so four CTAs per SM, 64 registers, no spills.
constexpr int kFeatRows = 256;
__global__ void __launch_bounds__(kEvalThreads, 4)
pm_build_argmin_feat(const uint4* __restrict__ srow, const uint32_t* __restrict__ sask, const uint2* __restrict__ ropt,
                     const uint4* __restrict__ feat, uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw,
                     uint32_t* __restrict__ tile, size_t ld, uint8_t* __restrict__ held, uint8_t* __restrict__ priced,
                     FoldOut fo) {
  __shared__ __align__(128) uint4 s_row[kFeatRows];
  __shared__ uint64_t s_bar;
  __shared__ uint16_t s_key[kFoldWarps][kFeatRows];
  __shared__ uint8_t s_nb[kFoldWarps][kFeatRows];    // fold_row's infeasible counts
  __shared__ uint8_t s_held[kFeatRows], s_priced[kFeatRows];   // each row's map bytes as the launch found them
  __shared__ uint32_t s_ask[kFeatRows];              // each row's ask
  __shared__ uint2 s_fo[kFoldWarps];                 // each warp's Fo
  __shared__ uint32_t s_live_bits[kFeatRows / 32], s_sent_bits[kFeatRows / 32];   // bit i & 31 of word i / 32: row i
  __shared__ uint16_t s_live[kFeatRows + 2], s_sent[kFeatRows];   // + 2: the look-ahead loads past the last live row
  const uint32_t r0 = blockIdx.y * kFeatRows;
  const uint32_t nrows = min(nt - r0, (uint32_t)kFeatRows);
  if (threadIdx.x == 0) {
    mbar_init(&s_bar, 1);
    mbar_expect_tx(&s_bar, nrows * 16u);
    bulk_g2s(s_row, srow + t0 + r0, nrows * 16u, &s_bar);
  }
  const size_t held_stride = ld / kEvalCols;
  uint8_t* held_cta = held + (size_t)r0 * held_stride + blockIdx.x;
  uint8_t* priced_cta = priced + (size_t)r0 * held_stride + blockIdx.x;
  for (uint32_t i = threadIdx.x; i < nrows; i += kEvalThreads) {
    s_held[i] = held_cta[i * held_stride];
    s_priced[i] = priced_cta[i * held_stride];
    s_ask[i] = __ldg(sask + t0 + r0 + i);
  }
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t cbase = blockIdx.x * kEvalCols + (threadIdx.x >> 5) * 128u + lane * 4u;
  uint32_t fl[kEvalWPT], fh[kEvalWPT], price[kEvalWPT], dy[kEvalWPT], rk[kEvalWPT], cm[kEvalWPT];
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    const uint4 v = __ldg(feat + cbase + k);
    fl[k] = v.x; fh[k] = v.y; price[k] = v.z; rk[k] = v.w;
    dy[k] = 0x7FFFFFFFu - v.z;
    asm("" : "+r"(dy[k]));   // kept in a register: ptxas would otherwise recompute it from the price every row
    cm[k] = kNone;
  }
  // The warp's block of a row, classified as a whole: Fo / Fa = the OR / AND of its 128 words F, kmin its least rank.
  // Column c fails option o when R_o & ~F_c != 0, and Fa ⊆ F_c ⊆ Fo: so if R_o & ~Fo != 0 for every option, every
  // column fails the row (dead), and if R_o & ~Fa == 0 for some option, every column meets it (full).  Padding columns
  // (F = 0) make Fa = 0, and every row requires the candidate bit, so a padded block is never full.
  const uint32_t fo_lo = __reduce_or_sync(0xffffffffu, fl[0] | fl[1] | fl[2] | fl[3]);
  const uint32_t fo_hi = __reduce_or_sync(0xffffffffu, fh[0] | fh[1] | fh[2] | fh[3]);
  const uint32_t fa_lo = __reduce_and_sync(0xffffffffu, fl[0] & fl[1] & fl[2] & fl[3]);
  const uint32_t fa_hi = __reduce_and_sync(0xffffffffu, fh[0] & fh[1] & fh[2] & fh[3]);
  const uint32_t kmin = __reduce_min_sync(0xffffffffu, min(min(rk[0], rk[1]), min(rk[2], rk[3])));
  if (lane == 0) s_fo[warp] = make_uint2(fo_lo, fo_hi);
  uint4* out = reinterpret_cast<uint4*>(tile + (size_t)r0 * ld + cbase);
  size_t row_stride = ld / 4;
  asm("" : "+l"(row_stride));
  uint32_t key_slot = (uint32_t)__cvta_generic_to_shared(&s_key[warp][0]);
  uint32_t nb_slot = (uint32_t)__cvta_generic_to_shared(&s_nb[warp][0]);
  asm("" : "+r"(key_slot), "+r"(nb_slot));
  // 1 behind an opaque move: with the literal, ptxas proves b = min(u, 1) is 0 or 1 and turns the multiply-adds below
  // into compares and selects on the busier ALU pipe (EvalParams::sign_shift does the same for the FastRow kernel)
  uint32_t one = 1u;
  asm("" : "+r"(one));
  constexpr uint32_t S = kNarrowInfeasible;
  // A LIVE row r.  The warp's block needs no store when the row leaves every word as the block holds it: the sentinel
  // (its bit of `held`) and the row infeasible there, or the prices (its bit of `priced`) and the row feasible there.
  // skip_at is the infeasible count at which that is so: 128, 0, or 0xFF (never); the two bits are never both set.
  auto emit = [&](const uint4& q, uint4* dst, uint32_t r) {
    const uint32_t hb = (s_held[r] >> warp) & 1u, pb = (s_priced[r] >> warp) & 1u;
    const uint32_t skip_at = hb ? 128u : pb ? 0u : 0xFFu;
    const uint32_t ask = s_ask[r];
    // the least over the options, as for a column: dead != 0 when every option misses a feature of Fo, full == 0 when
    // some option needs only features of Fa
    uint32_t dead = (q.x & ~fo_lo) | (q.y & ~fo_hi), full = (q.x & ~fa_lo) | (q.y & ~fa_hi);
    for (uint32_t o = 1; o < q.z; ++o) {
      const uint2 R = __ldg(ropt + q.w + o);
      dead = min(dead, (R.x & ~fo_lo) | (R.y & ~fo_hi));
      full = min(full, (R.x & ~fa_lo) | (R.y & ~fa_hi));
    }
    if (__all_sync(0xffffffffu, dead != 0u)) {   // every word the sentinel, no feasible column: as fold_row would leave it
      fold_slot(kNoRank, 128u, key_slot, nb_slot, r);
      if (!hb) __stcs(dst, make_uint4(S, S, S, S));
      return;
    }
    if (__all_sync(0xffffffffu, full == 0u)) {   // every word the column's price, every column feasible
      fold_slot(kmin, 0u, key_slot, nb_slot, r);
      if (!pb) __stcs(dst, make_uint4(price[0], price[1], price[2], price[3]));
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) cm[k] = min(cm[k], ask);
      return;
    }
    uint32_t u[kEvalWPT];
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) u[k] = (q.x & ~fl[k]) | (q.y & ~fh[k]);
    for (uint32_t o = 1; o < q.z; ++o) {   // OR-options (node.rs:420-438): the ask fails only if every option does
      const uint2 R = __ldg(ropt + q.w + o);
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) u[k] = min(u[k], (R.x & ~fl[k]) | (R.y & ~fh[k]));   // non-zero: every option fails
    }
    uint32_t o[kEvalWPT];
    uint32_t key = kNone, nb = 0;
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) {
      const uint32_t b = min(u[k], one);                      // 1 when infeasible
      o[k] = b * dy[k] + price[k];                            // feasible: price ; infeasible: kNarrowInfeasible
      cm[k] = min(cm[k], b * 0x80000000u + ask);              // the ask, + 2^31 when infeasible
      key = min(key, b * kNoRank + rk[k]);                    // the rank, + kNoRank when infeasible
      nb += b;
    }
    if (fold_row(key, nb, key_slot, nb_slot, r) != skip_at) __stcs(dst, make_uint4(o[0], o[1], o[2], o[3]));
  };
  __syncthreads();            // mbarrier initialised, s_held, s_priced, s_ask and s_fo written
  uint32_t so_lo = 0, so_hi = 0;   // the stripe's So
#pragma unroll
  for (int j = 0; j < kFoldWarps; ++j) {
    const uint2 v = s_fo[j];
    so_lo |= v.x;
    so_hi |= v.y;
  }
  mbar_wait(&s_bar, 0);
  // The triage of rows h * 256 + threadIdx.x: the ballots of a warp's 32 rows are word h * 8 + warp of the bit sets
  constexpr int kTriage = (kFeatRows + kEvalThreads - 1) / kEvalThreads;
  uint32_t lb[kTriage], sb[kTriage];
#pragma unroll
  for (int h = 0; h < kTriage; ++h) {
    const uint32_t i = h * kEvalThreads + threadIdx.x;
    bool live = false, sent = false;
    if (i < nrows) {   // nrows <= kFeatRows
      const uint4 q = s_row[i];
      uint32_t dead = (q.x & ~so_lo) | (q.y & ~so_hi);   // the least over the options, as emit's dead test
      for (uint32_t o = 1; o < q.z; ++o) {
        const uint2 R = __ldg(ropt + q.w + o);
        dead = min(dead, (R.x & ~so_lo) | (R.y & ~so_hi));
      }
      live = dead == 0u;
      sent = !live && s_held[i] != 0xFFu;
    }
    lb[h] = __ballot_sync(0xffffffffu, live);
    sb[h] = __ballot_sync(0xffffffffu, sent);
    if (lane == 0 && i < kFeatRows) {
      s_live_bits[i >> 5] = lb[h];
      s_sent_bits[i >> 5] = sb[h];
    }
  }
  __syncthreads();
  // Each LIVE / SENTINEL row's place in its list: the rows of the words before its own, then the lanes below it
  uint32_t n_live = 0, n_sent = 0, pl[kTriage] = {}, ps[kTriage] = {};
#pragma unroll
  for (int k = 0; k < kFeatRows / 32; ++k) {
    const uint32_t a = __popc(s_live_bits[k]), b = __popc(s_sent_bits[k]);
#pragma unroll
    for (int h = 0; h < kTriage; ++h)
      if (k < h * kFoldWarps + (int)warp) {
        pl[h] += a;
        ps[h] += b;
      }
    n_live += a;
    n_sent += b;
  }
  const uint32_t below = (1u << lane) - 1u;
#pragma unroll
  for (int h = 0; h < kTriage; ++h) {
    const uint32_t i = h * kEvalThreads + threadIdx.x;
    if ((lb[h] >> lane) & 1u) s_live[pl[h] + __popc(lb[h] & below)] = (uint16_t)i;
    if ((sb[h] >> lane) & 1u) s_sent[ps[h] + __popc(sb[h] & below)] = (uint16_t)i;
  }
  if (threadIdx.x == 0) s_live[n_live] = s_live[n_live + 1] = 0;   // the look-ahead past the last rows: row 0, unused
  __syncthreads();
  // LIVE rows: each index loaded two rows ahead, each row one row ahead, in registers the row before has finished with
  uint32_t r = s_live[0], rn = s_live[1];
  uint4 q = s_row[r];
  for (uint32_t j = 0; j < n_live; ++j) {
    const uint4 qn = s_row[rn];
    const uint32_t rnn = s_live[j + 2];
    emit(q, out + r * row_stride, r);
    r = rn;
    rn = rnn;
    q = qn;
  }
  // SENTINEL rows: the sentinel block wherever the map's bit is clear
  for (uint32_t j = 0; j < n_sent; ++j) {
    const uint32_t i = s_sent[j];
    if (!((s_held[i] >> warp) & 1u)) __stcs(out + i * row_stride, make_uint4(S, S, S, S));
  }
  fold_merge_rows(
      s_key, s_nb, nrows, fo, [&](uint32_t i) { return (s_live_bits[i >> 5] >> (i & 31u)) & 1u; },
      [&](auto* a, uint32_t i) { return a + s_ask[i]; },
      [&](uint32_t i, uint32_t m, uint32_t pr) {   // only the bytes that change: a SKIP row's are 0xFF and 0 already
        if (m != s_held[i]) held_cta[i * held_stride] = (uint8_t)m;
        if (pr != s_priced[i]) priced_cta[i * held_stride] = (uint8_t)pr;
      });
  fold_flush_first_ask<true>(cm, cbase, w0, nw, fo);
}

// ------------------------------------------------------------------ argmin
constexpr int kArgThreads = 256;
constexpr int kArgWarps = kArgThreads / 32;
constexpr int kArgRows = 64;                     // rows per CTA

// grid = (ceil(ld / (8*S*64)), ceil(nt / 64)).  All 8 warps of a CTA work on the SAME
// RPW rows at a time, each on its own S*64-column slice (so a CTA touches RPW DRAM
// pages / TLB entries at a time even when rows are megabytes apart); a lane issues
// S*RPW independent 128-bit streaming loads before the first use (8 KB per warp in
// flight at S=8, RPW=2), folds them lane-locally, then one shuffle reduction per
// row.  Per-column "first feasible ask" never leaves the lane's registers; per-row
// (min, count) partials are merged in shared memory and flushed once per CTA.
template <int S, int RPW>
__global__ void __launch_bounds__(kArgThreads)
pm_argmin(const long long* __restrict__ tile, size_t ld, uint32_t nt, uint32_t t0, uint32_t w0,
          uint32_t nw, uint32_t* __restrict__ first_ask, long long* __restrict__ ask_best,
          uint32_t* __restrict__ ask_count) {
  constexpr int kWarpCols = S * 64;
  __shared__ long long s_best[kArgRows];   // signed, as the packed cost: a price >= 2^31 makes it negative
  __shared__ uint32_t s_cnt[kArgRows];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t c0 = (blockIdx.x * kArgWarps + warp) * kWarpCols;   // this warp's first column
  const uint32_t r0 = blockIdx.y * kArgRows;
  const uint32_t rows = min((uint32_t)kArgRows, nt - r0);
  for (uint32_t i = threadIdx.x; i < (uint32_t)kArgRows; i += kArgThreads) {
    s_best[i] = kInf;
    s_cnt[i] = 0;
  }
  __syncthreads();

  constexpr int CPL = 2;                               // columns per 128-bit load
  uint32_t cm[S][CPL];
#pragma unroll
  for (int s = 0; s < S; ++s)
#pragma unroll
    for (int j = 0; j < CPL; ++j) cm[s][j] = kNone;

  if (c0 < ld) {
    for (uint32_t rr = 0; rr < rows; rr += RPW) {
      longlong2 v[RPW][S];
#pragma unroll
      for (int q = 0; q < RPW; ++q) {
        const uint32_t r = r0 + rr + q;
        const longlong2* rowp = reinterpret_cast<const longlong2*>(tile) + (size_t)r * (ld / CPL);
#pragma unroll
        for (int s = 0; s < S; ++s) {
          const uint32_t col = c0 + s * 32 * CPL + lane * CPL;
          if (rr + q < rows && col < ld) v[q][s] = __ldcs(rowp + col / CPL);
          else v[q][s] = make_longlong2(kInf, kInf);
        }
      }
#pragma unroll
      for (int q = 0; q < RPW; ++q) {
        const uint32_t t = t0 + r0 + rr + q;
        long long best = kInf;
        uint32_t cnt = 0;
#pragma unroll
        for (int s = 0; s < S; ++s) {
          best = min(best, min(v[q][s].x, v[q][s].y));
          const bool fx = v[q][s].x != kInf, fy = v[q][s].y != kInf;
          cnt += (uint32_t)fx + (uint32_t)fy;
          cm[s][0] = fx ? min(cm[s][0], t) : cm[s][0];
          cm[s][1] = fy ? min(cm[s][1], t) : cm[s][1];
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          best = min(best, __shfl_xor_sync(0xffffffffu, best, off));
          cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
        }
        if (lane == 0 && cnt) {
          atomicMin(&s_best[rr + q], best);
          atomicAdd(&s_cnt[rr + q], cnt);
        }
      }
    }
#pragma unroll
    for (int s = 0; s < S; ++s) {
#pragma unroll
      for (int j = 0; j < CPL; ++j) {
        const uint32_t col = c0 + s * 32 * CPL + lane * CPL + j;
        if (cm[s][j] != kNone && col < nw) atomicMin(first_ask + w0 + col, cm[s][j]);
      }
    }
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < rows; i += kArgThreads) {
    if (s_cnt[i]) {
      atomicMin(ask_best + t0 + r0 + i, s_best[i]);
      atomicAdd(ask_count + t0 + r0 + i, s_cnt[i]);
    }
  }
}

// ------------------------------------------------------------------ fused
// Same stripe/row decomposition as pm_build_cost, but the int64 cost never
// leaves the SM: per-worker results stay in registers, and each row's minimum is
// the one pm_argmin finds, the signed int64 least (price << 32) | worker over the
// feasible workers.  A warp takes it in two steps: the least price read as int32
// (signed redux; that order is the packed cost's for prices >= 2^31 too), then
// the lowest worker at that price from one ballot per k.  Integer-issue-bound,
// not HBM-bound.
// STATS = false skips the per-ask (min, count) outputs — the reference modes only need the
// per-worker first feasible ask — which removes the reductions from the inner loop.
template <int BITS, bool FAST, bool STATS>
__global__ void __launch_bounds__(kEvalThreads, 2)
pm_fused_eval(EvalParams p, uint32_t t0, uint32_t nt, uint32_t w0, uint32_t nw,
              uint32_t* __restrict__ first_ask, long long* __restrict__ ask_best,
              uint32_t* __restrict__ ask_count) {
  __shared__ EvalStage s;
  __shared__ uint32_t s_cnt[kEvalRows];
  // signed, as the packed cost: a price >= 2^31 makes it negative.  Unused without STATS, where it keeps the 32-bit
  // form the lean kernel has always been compiled with.
  using Best = std::conditional_t<STATS, long long, uint32_t>;
  __shared__ Best s_best[kEvalRows];
  const uint32_t r0 = blockIdx.y * kEvalRows;
  const uint32_t r1 = min(nt, r0 + (uint32_t)kEvalRows);
  for (uint32_t i = threadIdx.x; i < (uint32_t)kEvalRows; i += kEvalThreads) {
    s_cnt[i] = 0;
    s_best[i] = STATS ? (Best)kInf : (Best)kNone;
  }
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t c = blockIdx.x * kEvalCols + threadIdx.x * kEvalWPT;
  WorkerReg w[kEvalWPT];
  load_workers<kEvalWPT>(p, w0, nw, c, w);
  uint32_t first[kEvalWPT];
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) first[k] = kNone;
  const uint32_t warp_gw0 = w0 + (c - lane * kEvalWPT);
  for_each_staged_row(s, p, FAST, t0, r0, r1, [&](uint32_t r, const DevAsk& a, uint32_t obegin, bool staged) {
    uint32_t f[kEvalWPT];
    if (FAST && staged) {
      uint32_t fail[kEvalWPT];
      eval_row_fast<kEvalWPT, BITS>(s, a, obegin, w, p.bits, p.words, fail);
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) f[k] = ~(uint32_t)((int32_t)fail[k] >> 31);   // all-ones <=> feasible
    } else if (staged) {
      eval_row<kEvalWPT, BITS>(s, a, obegin, w, p.bits, p.words, f);
    } else {
      eval_row_global<kEvalWPT>(p, a, w, f);
    }
    const uint32_t t = t0 + r0 + r;
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) first[k] = min(first[k], t | ~f[k]);
    if (STATS) {
      uint32_t n = 0;
      int lp = INT32_MAX;   // the lane's least feasible price, or INT32_MAX: the ballots below only see feasible workers
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) {
        n += f[k] & 1u;
        if (f[k]) lp = min(lp, (int)w[k].price);
      }
      const uint32_t cnt = __reduce_add_sync(0xffffffffu, n);
      const int price = __reduce_min_sync(0xffffffffu, lp);
      uint32_t best = kNone;   // the warp's lowest worker offset at that price
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) {
        const uint32_t b = __ballot_sync(0xffffffffu, f[k] != 0u && (int)w[k].price == price);
        if (b) best = min(best, ((uint32_t)__ffs(b) - 1u) * kEvalWPT + k);
      }
      if (cnt && lane == 0) {
        atomicAdd(&s_cnt[r], cnt);
        atomicMin(&s_best[r], (long long)(((unsigned long long)(uint32_t)price << 32) | (warp_gw0 + best)));
      }
    }
  });
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k)
    if (first[k] != kNone) atomicMin(first_ask + w0 + c + k, first[k]);
  if (!STATS) return;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < r1 - r0; i += kEvalThreads) {
    if (s_cnt[i]) {
      atomicAdd(ask_count + t0 + r0 + i, s_cnt[i]);
      atomicMin(ask_best + t0 + r0 + i, s_best[i]);
    }
  }
}

// ------------------------------------------------------------------ incremental: first feasible ask of listed rows
// pm_fused_eval's per-worker output (the lowest ask t with feasible(t, w)) for the workers named in `rows` only: an
// incremental pass re-evaluates the rows written since the stored evaluation and keeps the others.  Same predicate
// code as pm_fused_eval (for_each_staged_row, eval_row_fast / eval_row / eval_row_global, every BITS form, the
// worker-major `nacc` word), so the values are the fused pass's by construction.
//
// grid = (ceil(n / 1024), chunks): a CTA gathers 1024 listed workers into registers (4 per thread, as the fused
// kernel holds its stripe) and walks its chunk of `chunk` asks in steps of kEvalRows staged rows.  Asks are in
// priority order, so a hit is final for the chunk; before each step the CTA stops once every one of its workers has a
// hit of its own, or a hit below the step's first row in `first_ask` (published by the CTAs of earlier chunks with
// atomicMin), or is not a candidate at all (no ask can accept it).  The result is min(first_ask[w] on entry, the
// first hit): a written row enters with kNone.  `evals` gains the pairs evaluated: rows walked x listed workers of the
// CTA.
//
// The same kernel makes the two other walks of an incremental pass after configurations were enabled or disabled
// (AskWalk):
//   * the E-pass: every worker of the engine's range (rows == null: workers row0 + [0, n)) against the newly enabled
//     asks only (asks = their increasing list).  A worker enters with its stored first ask f, so the first step's test
//     already drops it when f lies below every listed ask, and a CTA whose workers all do exits before its first row;
//   * the orphans: workers whose stored first ask was disabled, each with a start bound (the ask after it).  Asks
//     below the start that were enabled then still reject the worker; those enabled since are the E-pass's.  The CTA
//     starts at the least bound of its workers.
struct AskWalk {
  const uint32_t* rows;     // listed workers, or null: workers [row0, row0 + n)
  const uint32_t* starts;   // per listed worker, the first ask it can still need; null: 0
  const uint32_t* asks;     // the asks walked, increasing; null: the whole table
  uint32_t n;               // listed workers
  uint32_t n_seq;           // asks walked: entries of `asks`, or the table's n_asks
  uint32_t chunk;           // asks per grid row (blockIdx.y)
  uint32_t row0;            // rows == null: the first worker
};

__device__ __forceinline__ void gather_workers(const EvalParams& p, const uint32_t* __restrict__ rows, uint32_t row0,
                                               uint32_t n, uint32_t c, WorkerReg (&w)[kEvalWPT],
                                               uint32_t (&gw)[kEvalWPT]) {
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    const uint32_t col = c + k;
    if (col < n) {
      gw[k] = rows ? __ldg(rows + col) : row0 + col;
      w[k] = make_worker(__ldg(p.wa + gw[k]), __ldg(p.wb + gw[k]));
      if (p.nacc) w[k].mmask = __ldg(p.nacc + gw[k]);
    } else {
      gw[k] = kNone;
      w[k] = null_worker();
    }
  }
}

template <int BITS, bool FAST>
__global__ void __launch_bounds__(kEvalThreads, 2)
pm_first_ask_rows(EvalParams p, AskWalk a, uint32_t* __restrict__ first_ask, unsigned long long* __restrict__ evals) {
  __shared__ EvalStage s;
  __shared__ uint32_t s_lo;
  const uint32_t cta0 = blockIdx.x * kEvalCols;
  const uint32_t c = cta0 + threadIdx.x * kEvalWPT;
  WorkerReg w[kEvalWPT];
  uint32_t gw[kEvalWPT];
  gather_workers(p, a.rows, a.row0, a.n, c, w, gw);
  const uint32_t n_cta = min(a.n - cta0, (uint32_t)kEvalCols);   // listed workers of this CTA
  uint32_t first[kEvalWPT];
  bool open[kEvalWPT];   // a listed candidate without a hit published yet
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    first[k] = kNone;
    open[k] = gw[k] != kNone && (w[k].flags & kCandBit) != 0u;
  }
  uint32_t c0 = blockIdx.y * a.chunk;
  const uint32_t c1 = min(a.n_seq, c0 + a.chunk);
  if (a.starts) {   // the CTA's least start bound
    if (threadIdx.x == 0) s_lo = kNone;
    __syncthreads();
    uint32_t lo = kNone;
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k)
      if (c + k < a.n) lo = min(lo, __ldg(a.starts + c + k));
    lo = __reduce_min_sync(0xffffffffu, lo);
    if ((threadIdx.x & 31u) == 0u) atomicMin(&s_lo, lo);
    __syncthreads();
    c0 = max(c0, s_lo);
  }
  unsigned long long pairs = 0;
  for (uint32_t r0 = c0; r0 < c1; r0 += kEvalRows) {
    const uint32_t t_first = a.asks ? __ldg(a.asks + r0) : r0;   // the step's first ask
    // publish this CTA's hits (each is final: later rows are higher), then stop when no worker can still improve
    bool done = true;
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) {
      if (!open[k]) continue;
      if (first[k] != kNone) {
        atomicMin(first_ask + gw[k], first[k]);
        open[k] = false;
      } else {
        done &= *reinterpret_cast<volatile const uint32_t*>(first_ask + gw[k]) < t_first;
      }
    }
    // also the barrier that lets for_each_staged_row re-initialise its mbarrier and overwrite the stage
    if (__syncthreads_and(done)) break;
    const uint32_t r1 = min(c1, r0 + (uint32_t)kEvalRows);
    for_each_staged_row(s, p, FAST, r0, 0u, r1 - r0, [&](uint32_t r, const DevAsk& q, uint32_t obegin, bool staged) {
      uint32_t f[kEvalWPT];
      if (FAST && staged) {
        uint32_t fail[kEvalWPT];
        eval_row_fast<kEvalWPT, BITS>(s, q, obegin, w, p.bits, p.words, fail);
#pragma unroll
        for (int k = 0; k < kEvalWPT; ++k) f[k] = ~(uint32_t)((int32_t)fail[k] >> 31);   // all-ones <=> feasible
      } else if (staged) {
        eval_row<kEvalWPT, BITS>(s, q, obegin, w, p.bits, p.words, f);
      } else {
        eval_row_global<kEvalWPT>(p, q, w, f);
      }
      const uint32_t t = a.asks ? __ldg(a.asks + r0 + r) : r0 + r;
#pragma unroll
      for (int k = 0; k < kEvalWPT; ++k) first[k] = min(first[k], t | ~f[k]);
    }, a.asks);
    pairs += (unsigned long long)(r1 - r0) * n_cta;
  }
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k)
    if (open[k] && first[k] != kNone) atomicMin(first_ask + gw[k], first[k]);
  if (threadIdx.x == 0 && pairs) atomicAdd(evals, pairs);
}

// ------------------------------------------------------------------ ask-table conversion
// pm_ask / pm_gpu_opt (ABI form, field-for-field NodeGroupConfiguration + GpuRequirements) ->
// DevAsk / DevOpt / DevOptF, on the device: the upload is a plain memcpy of the caller's tables
// and one pass of these two kernels instead of a host loop.
enum AskStatusBit : uint32_t {
  kAskBadSizes = 1u << 0,   // max_group_size < min_group_size (is_valid, mod.rs:55-60)
  kAskBadRange = 1u << 1,   // opt_off + n_opts out of bounds
  kAskNotSmall = 1u << 2    // an operand does not fit the fast predicate
};

__global__ void pm_ask_counts(const pm_ask* __restrict__ asks, uint32_t n_asks, uint32_t n_opts,
                              uint32_t* __restrict__ counts, uint32_t* __restrict__ status) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n_asks) return;
  if (t == n_asks) { counts[t] = 0; return; }
  const pm_ask a = asks[t];
  uint32_t st = 0;
  if (a.max_group_size < a.min_group_size) st |= kAskBadSizes;
  if ((unsigned long long)a.opt_off + a.n_opts > n_opts) st |= kAskBadRange;
  if (st) atomicOr(status, st);
  // every converted ask owns at least one option row: an ask without GPU options gets a neutral one (pm_ask_convert)
  counts[t] = max(((a.flags & PM_A_HAS_REQ) && !(st & kAskBadRange)) ? a.n_opts : 0u, 1u);
}

struct AskTables {   // the converted forms of the ask table the kernels read
  DevAsk* dasks;
  DevOpt* dopts;
  DevOptF* doptsf;
  FastRow* frows;
  uint32_t* amin;
  uint32_t* amax;
};

// Ask t in every converted form.  A disabled ask (`off`) carries kNeverBit in its presence mask — DevAsk.need and the
// m / v of each of its DevOptF rows and its FastRow — so every predicate variant rejects every worker, and its amin is
// at least 1, so it forms no empty group either: it behaves as if it were absent from the table.  Converting it again
// with off == false restores the rows exactly.  `status` / `max_row` may be null (a toggle: the table was checked).
// `sizes`: the reference modes' group-size clause (max_group_size == 0 takes nobody) is part of the rows; the auction,
// which has no group sizes, converts its max_group_size == 0 asks without it.
__device__ __forceinline__ void convert_ask(uint32_t t, bool off, bool sizes, bool bad_range, const pm_ask* __restrict__ asks,
                                            const pm_gpu_opt* __restrict__ opts, const uint32_t* __restrict__ new_off,
                                            const AskTables& o, uint32_t* __restrict__ status,
                                            uint32_t* __restrict__ max_row) {
  DevAsk* __restrict__ dasks = o.dasks;
  DevOpt* __restrict__ dopts = o.dopts;
  DevOptF* __restrict__ doptsf = o.doptsf;
  const pm_ask a = asks[t];
  DevAsk d;
  d.n_opts = 0; d.cpu_cores = 0; d.ram_mb = 0; d.storage_gb = 0; d.pad0 = 0; d.pad1 = 0;
  const bool has_req = (a.flags & PM_A_HAS_REQ) != 0;
  uint32_t need = kCandBit;
  const uint32_t n_rows = new_off[t + 1] - new_off[t];                  // >= 1
  const uint32_t n_eff = (has_req && !bad_range) ? min(a.n_opts, n_rows) : 0u;
  if (has_req) {
    need |= PM_W_HAS_SPECS;
    if (a.flags & PM_A_REQ_CPU) need |= PM_W_HAS_CPU;
    if ((a.flags & PM_A_REQ_CPU) && (a.flags & PM_A_REQ_CPU_CORES)) { need |= PM_W_HAS_CPU_CORES; d.cpu_cores = a.cpu_cores; }
    if (a.flags & PM_A_REQ_RAM) { need |= PM_W_HAS_RAM; d.ram_mb = a.ram_mb; }
    if (a.flags & PM_A_REQ_STORAGE) { need |= PM_W_HAS_STORAGE; d.storage_gb = a.storage_gb; }
    if (a.n_opts) need |= PM_W_HAS_GPU;
  }
  d.n_opts = n_rows;
  if ((sizes && a.max_group_size == 0) || off) need |= kNeverBit;   // first-fit with max_group_size == 0 takes nobody (mod.rs:555-556)
  d.need = need;
  d.opt_off = new_off[t];
  uint32_t st = 0, mrow = 0;
  if ((d.cpu_cores | d.ram_mb | d.storage_gb) >= kSign) st |= kAskNotSmall;
  for (uint32_t o = 0; o < n_eff; ++o) {
    const pm_gpu_opt q = opts[a.opt_off + o];
    DevOpt x;
    x.need = 0;
    x.count_mask = (q.present & PM_O_COUNT) ? 0xFFFFFFFFu : 0u;
    x.count = (q.present & PM_O_COUNT) ? q.count : 0u;
    uint32_t mem_lo = 0, mem_hi = 0xFFFFFFFFu, tot_lo = 0, tot_hi = 0xFFFFFFFFu;
    if (q.present & PM_O_MEM) mem_lo = max(mem_lo, q.memory_mb);
    if (q.present & PM_O_MEM_MIN) mem_lo = max(mem_lo, q.memory_mb_min);
    if (q.present & PM_O_MEM_MAX) mem_hi = q.memory_mb_max;
    if (q.present & (PM_O_MEM | PM_O_MEM_MIN | PM_O_MEM_MAX)) x.need |= PM_W_HAS_GPU_MEM;
    if (q.present & PM_O_TOT_MIN) tot_lo = q.total_memory_min;
    if (q.present & PM_O_TOT_MAX) tot_hi = q.total_memory_max;
    if (mem_lo > mem_hi) { x.need |= kNeverBit; mem_lo = 0; mem_hi = 0xFFFFFFFFu; }
    if (tot_lo > tot_hi) { x.need |= kTotInvalidBit; tot_lo = 0; tot_hi = 0xFFFFFFFFu; }
    x.mem_lo = mem_lo; x.mem_span = mem_hi - mem_lo;
    x.tot_lo = tot_lo; x.tot_span = tot_hi - tot_lo;
    x.pattern_row = 0;
    if (q.present & PM_O_MODEL) {
      x.need |= PM_W_HAS_GPU_MODEL;
      x.pattern_row = q.pattern_id + 1;
      // pattern_id 0xFFFFFFFF wraps to row 0 ("no model clause"): count it as the largest row, so that the table is
      // refused (PM_E_STATE) as for any pattern past the model table
      mrow = max(mrow, q.pattern_id == 0xFFFFFFFFu ? 0xFFFFFFFFu : x.pattern_row);
    }
    dopts[d.opt_off + o] = x;
    DevOptF f;
    const uint32_t need_all = need | x.need;
    f.m = key_bits(need_all); f.v = f.m;
    if (q.present & PM_O_COUNT) {
      if (q.count >= 65536u) st |= kAskNotSmall;
      f.m |= 0xFFFFu << kKeyCountShift;
      f.v |= (q.count & 0xFFFFu) << kKeyCountShift;
    }
    if (mem_lo >= kSign || tot_lo >= kSign) st |= kAskNotSmall;
    f.mem_lo = mem_lo; f.mem_hi = min(mem_hi, 0x7FFFFFFFu);
    f.tot_lo = tot_lo; f.tot_hi = min(tot_hi, 0x7FFFFFFFu);
    f.pattern_row = x.pattern_row; f.pad = 0;
    doptsf[d.opt_off + o] = f;
  }
  if (n_eff == 0u) {
    // no GPU clause (requirements.gpu empty, or no requirements at all): one neutral option row — it accepts every
    // worker, so the ask's presence bits and scalar thresholds decide alone — keeps the evaluation loops free of an
    // option-less special case
    DevOpt x;
    x.need = 0; x.count_mask = 0; x.count = 0; x.mem_lo = 0; x.mem_span = 0xFFFFFFFFu; x.tot_lo = 0; x.tot_span = 0xFFFFFFFFu;
    x.pattern_row = 0;
    dopts[d.opt_off] = x;
    DevOptF f;
    f.m = key_bits(need); f.v = f.m;
    f.mem_lo = 0; f.mem_hi = 0x7FFFFFFFu; f.tot_lo = 0; f.tot_hi = 0x7FFFFFFFu; f.pattern_row = 0; f.pad = 0;
    doptsf[d.opt_off] = f;
  }
  dasks[t] = d;
  {
    const DevOptF f = doptsf[d.opt_off];   // written above by this thread
    FastRow fr;
    fr.m = f.m; fr.v = f.v; fr.mem_lo = f.mem_lo; fr.mem_hi = f.mem_hi;
    fr.tot_lo = f.tot_lo; fr.tot_hi = f.tot_hi; fr.wp = f.pattern_row; fr.n_opts = n_rows;
    fr.cpu_cores = d.cpu_cores; fr.ram_mb = d.ram_mb; fr.storage_gb = d.storage_gb; fr.opt_off = d.opt_off;
    o.frows[t] = fr;
  }
  o.amin[t] = off ? max(a.min_group_size, 1u) : a.min_group_size;
  o.amax[t] = a.max_group_size;
  if (st && status) atomicOr(status, st);
  if (mrow && max_row) atomicMax(max_row, mrow);
}

__global__ void pm_ask_convert(const pm_ask* __restrict__ asks, const pm_gpu_opt* __restrict__ opts,
                               uint32_t n_asks, const uint32_t* __restrict__ new_off, AskTables o,
                               uint32_t* __restrict__ status, uint32_t* __restrict__ max_row) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  // option rows that come from the caller (none are read when pm_ask_counts found a range out of bounds: the call fails)
  const bool bad_range = (*reinterpret_cast<volatile uint32_t*>(status) & kAskBadRange) != 0u;
  convert_ask(t, false, true, bad_range, asks, opts, new_off, o, status, max_row);
}

// pm_set_ask_enabled: the listed asks converted again, enabled or disabled; entry i = ask << 1 | enabled, one entry
// per ask.  Also the switch of the max_group_size == 0 asks between the reference modes' form and the auction's (sizes).
__global__ void pm_ask_toggle(const pm_ask* __restrict__ asks, const pm_gpu_opt* __restrict__ opts,
                              const uint32_t* __restrict__ new_off, const uint32_t* __restrict__ list, uint32_t n,
                              AskTables o, bool sizes) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = list[i];
  convert_ask(v >> 1, (v & 1u) == 0u, sizes, false, asks, opts, new_off, o, nullptr, nullptr);
}

// pm_update_asks / pm_resize_asks: the caller's rows scattered into the resident raw table (idx distinct, each < n_asks)
__global__ void pm_scatter_asks(pm_ask* __restrict__ asks, const uint32_t* __restrict__ idx, const pm_ask* __restrict__ rows,
                                uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) asks[idx[i]] = rows[i];
}

// pm_remove_asks / pm_insert_asks / pm_resize_asks under a stored evaluation: each stored first ask f of the range
// [w0, w0 + nw) moves to f - (removed asks below f) + (rows inserted before a position <= f); `removed` and `before`
// are increasing old indices.  A removed f lands on the new index of its next kept row, whose orphans the engine lists
// for the next incremental pass; past the new end (n_asks) there is none, and the worker has no feasible ask.
__global__ void pm_splice_first_asks(uint32_t* __restrict__ eval_first, uint32_t w0, uint32_t nw, const uint32_t* __restrict__ removed,
                                     uint32_t nr, const uint32_t* __restrict__ before, uint32_t ni, uint32_t n_asks) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nw; i += gridDim.x * blockDim.x) {
    const uint32_t f = eval_first[w0 + i];
    if (f == kNone) continue;
    uint32_t lo = 0, hi = nr;   // removed asks < f
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(removed + mid) < f) lo = mid + 1; else hi = mid;
    }
    const uint32_t r = lo;
    lo = 0, hi = ni;            // inserted rows with before <= f
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(before + mid) <= f) lo = mid + 1; else hi = mid;
    }
    const uint32_t g = f - r + lo;
    eval_first[w0 + i] = g < n_asks ? g : kNone;
  }
}

// An incremental pass after configurations were disabled or replaced: the workers of the range [w0, w0 + nw) whose
// stored first ask is one of them (`dis`, entries ask << 1 | replaced, increasing, nd entries).  Each is appended to
// out[] with its walk's start bound — the ask after its stored one, or the stored one itself when that row was
// replaced (the new row may still accept it) — and its stored entry is reset.  One thread per worker, one atomic per
// warp.
__global__ void pm_collect_orphans(uint32_t* __restrict__ eval_first, uint32_t w0, uint32_t nw, const uint32_t* __restrict__ dis,
                                   uint32_t nd, uint32_t* __restrict__ out, uint32_t* __restrict__ starts,
                                   uint32_t* __restrict__ count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t w = w0 + i;
  const uint32_t f = i < nw ? eval_first[w] : kNone;
  bool hit = false;
  uint32_t d = 0;
  if (f != kNone) {
    uint32_t lo = 0, hi = nd;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if ((__ldg(dis + mid) >> 1) < f) lo = mid + 1; else hi = mid;
    }
    if (lo < nd) d = __ldg(dis + lo);
    hit = lo < nd && (d >> 1) == f;
  }
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t b = __ballot_sync(0xffffffffu, hit);
  if (!b) return;
  uint32_t base = 0;
  if (lane == 0) base = atomicAdd(count, (uint32_t)__popc(b));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (hit) {
    const uint32_t pos = base + (uint32_t)__popc(b & ((1u << lane) - 1u));
    out[pos] = w;
    starts[pos] = f + 1u - (d & 1u);
    eval_first[w] = kNone;
  }
}

// ------------------------------------------------------------------ small utilities
__global__ void pm_fill_u32(uint32_t* p, uint32_t v, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void pm_fill_i64(long long* p, long long v, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void pm_iota_u32(uint32_t* p, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = (uint32_t)i;
}
__global__ void pm_scatter_flags(uint4* wa, const uint32_t* idx, const uint32_t* flags, uint32_t n, uint32_t n_workers) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && idx[i] < n_workers) wa[idx[i]].w = flags[i];
}

// pm_update_workers: rows that changed since the last pass, scattered into the resident table
__global__ void pm_scatter_rows(uint4* wa, uint4* wb, double* lat, double* lon, const uint32_t* __restrict__ idx,
                                const uint4* __restrict__ a, const uint4* __restrict__ b, const double* __restrict__ la,
                                const double* __restrict__ lo, uint32_t n, uint32_t n_workers) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t w = idx[i];
  if (w >= n_workers) return;
  wa[w] = a[i];
  wb[w] = b[i];
  if (lat) { lat[w] = la[i]; lon[w] = lo[i]; }
}

// ---- worker-table splice (pm_remove_workers / pm_insert_workers) ------------------------------------------------
// `removed`: old rows, increasing and distinct (nr); `before`: per inserted row the old row it goes before,
// non-decreasing (ni).  Kept old row i goes to i - |{r < i}| + |{before <= i}|; inserted row k to
// before[k] - |{r < before[k]}| + k.
struct WorkerSplice {
  const uint32_t* removed;
  const uint32_t* before;
  uint32_t nr, ni, n_old;
  // every column is moved from its old buffer into the second one of its pair; a null column is not in use
  const uint4 *wa, *wb, *ins_a, *ins_b;
  uint4 *wa_out, *wb_out;
  const double *lat, *lon, *ins_lat, *ins_lon;   // ins_lat null: inserted rows at (0, 0)
  double *lat_out, *lon_out;
  const uint32_t *rank, *rep;
  uint32_t *rank_out, *rep_out;
  // the worker-major acceptance words: old rows below nacc_n hold them; inserted rows are listed as written
  const uint32_t* nacc;
  uint32_t* nacc_out;
  uint32_t nacc_n;
  // the stored evaluation: kept where the old row was in [a0, a1) and the new one is in [b0, b1), else PM_NONE
  const uint32_t* first;
  uint32_t* first_out;
  uint32_t a0, a1, b0, b1;
  // the stored auction state: old rows below auc_kept keep price and owner, every other row is 0 / unowned
  const long long* price;
  long long* price_out;
  const uint32_t* owner;
  uint32_t* owner_out;
  uint32_t auc_kept;
};
__device__ __forceinline__ uint32_t splice_lower(const uint32_t* __restrict__ v, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;   // entries < x
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(v + mid) < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ uint32_t splice_upper(const uint32_t* __restrict__ v, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;   // entries <= x
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(v + mid) <= x) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// One thread per old row and per inserted row: every output row is written exactly once (the destinations of the
// kept and inserted rows are disjoint and cover [0, n_old - nr + ni)), in increasing order along the grid, so the
// stores stay coalesced.
__global__ void pm_splice_workers(WorkerSplice s) {
  const uint32_t n = s.n_old + s.ni;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < s.n_old) {
      const uint32_t r = splice_lower(s.removed, s.nr, i);
      if (r < s.nr && __ldg(s.removed + r) == i) continue;
      const uint32_t j = i - r + splice_upper(s.before, s.ni, i);
      s.wa_out[j] = s.wa[i];
      s.wb_out[j] = s.wb[i];
      if (s.lat_out) { s.lat_out[j] = s.lat[i]; s.lon_out[j] = s.lon[i]; }
      if (s.rank_out) s.rank_out[j] = s.rank[i];
      if (s.rep_out) s.rep_out[j] = s.rep[i];
      if (s.nacc_out) s.nacc_out[j] = i < s.nacc_n ? s.nacc[i] : 0u;
      if (s.first_out)
        s.first_out[j] = (i - s.a0 < s.a1 - s.a0 && j - s.b0 < s.b1 - s.b0) ? s.first[i] : kNone;
      if (s.price_out) {
        const bool kept = i < s.auc_kept;
        s.price_out[j] = kept ? s.price[i] : 0ll;
        s.owner_out[j] = kept ? s.owner[i] : kNone;
      }
    } else {
      const uint32_t k = i - s.n_old, b = __ldg(s.before + k);
      const uint32_t j = b - splice_lower(s.removed, s.nr, b) + k;
      s.wa_out[j] = s.ins_a[k];
      s.wb_out[j] = s.ins_b[k];
      if (s.lat_out) {
        s.lat_out[j] = s.ins_lat ? s.ins_lat[k] : 0.0;
        s.lon_out[j] = s.ins_lat ? s.ins_lon[k] : 0.0;
      }
      if (s.rank_out) s.rank_out[j] = 0u;
      if (s.rep_out) s.rep_out[j] = 0u;
      if (s.nacc_out) s.nacc_out[j] = 0u;
      if (s.first_out) s.first_out[j] = kNone;
      if (s.price_out) {
        s.price_out[j] = 0ll;
        s.owner_out[j] = kNone;
      }
    }
  }
}
// The stored auction assignment under a worker splice, in place (one entry per slot): a kept row's hold moves to its
// new index; a hold on a removed row, or on a row at or past auc_kept (cut off by an earlier shrink), becomes
// kCutHold, which the next warm pass releases in its step 1 as it releases the holder of a row a shrink cut off.
constexpr uint32_t kCutHold = 0xFFFFFFFEu;
__global__ void pm_splice_worker_holds(uint32_t* __restrict__ assigned, uint32_t n_slots, const uint32_t* __restrict__ removed,
                                       uint32_t nr, const uint32_t* __restrict__ before, uint32_t ni, uint32_t auc_kept) {
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_slots; s += gridDim.x * blockDim.x) {
    const uint32_t w = assigned[s];
    if (w == kNone) continue;
    if (w >= auc_kept) {
      assigned[s] = kCutHold;
      continue;
    }
    const uint32_t r = splice_lower(removed, nr, w);
    assigned[s] = (r < nr && __ldg(removed + r) == w) ? kCutHold : w - r + splice_upper(before, ni, w);
  }
}

// Do all workers satisfy the fast-path operand limits (values < 2^31, gpu count < 2^16,
// count * memory_mb < 2^31 without wrapping)?  Clears ok[0] otherwise.  Is every price below
// kNarrowInfeasible, so that the 32-bit cost tile can hold it?  Clears ok[1] otherwise.
__device__ __forceinline__ void check_worker_range(const uint4& a, const uint4& b, uint32_t* __restrict__ ok) {
  bool small = (b.x | b.y | b.z) < kSign;
  if (a.w & PM_W_HAS_GPU_COUNT) small &= a.x < 65536u;
  if (a.w & PM_W_HAS_GPU_MEM) small &= a.y < kSign;
  if ((a.w & PM_W_HAS_GPU_COUNT) && (a.w & PM_W_HAS_GPU_MEM))
    small &= (unsigned long long)a.x * (unsigned long long)a.y < (unsigned long long)kSign;
  if (!small) ok[0] = 0u;
  if (b.w >= kNarrowInfeasible) ok[1] = 0u;
}
__global__ void pm_check_worker_ranges(const uint4* __restrict__ wa, const uint4* __restrict__ wb,
                                       uint32_t n, uint32_t* __restrict__ ok) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  check_worker_range(wa[i], wb[i], ok);
}
// ... over the listed rows only: an incremental pass starts from the flags of the last full check, so a flag cleared
// once stays cleared until a full check (both predicates give the same answers; only the speed differs)
__global__ void pm_check_worker_rows(const uint4* __restrict__ wa, const uint4* __restrict__ wb,
                                     const uint32_t* __restrict__ rows, uint32_t n, uint32_t* __restrict__ ok) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t w = rows[i];
  check_worker_range(wa[w], wb[w], ok);
}

__global__ void pm_scatter_value(uint32_t* __restrict__ dst, const uint32_t* __restrict__ rows, uint32_t n, uint32_t v) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[rows[i]] = v;
}

// ------------------------------------------------------------------ resolution
// Sort key of a worker: its (first feasible) ask; in proximity mode with solo
// groups the key also orders located workers first (seed rule, mod.rs:526-530).
__global__ void pm_make_keys(const uint32_t* __restrict__ cur, const uint4* __restrict__ wa,
                             uint32_t n_workers, uint32_t shift, uint32_t* __restrict__ keys,
                             uint32_t* __restrict__ hist) {
  uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_workers) return;
  uint32_t c = cur[w], k = kNone;
  if (c != kNone) {
    k = c << shift;
    if (shift) k |= (wa[w].w & PM_W_HAS_LOC) ? 0u : 1u;
    atomicAdd(hist + k, 1u);
  }
  keys[w] = k;
}

// any configuration whose member count leaves an under-filled tail
// (0 < K mod max < min: the tail group is not formed, mod.rs:517,564)?
__global__ void pm_check_tails(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ amin,
                               const uint32_t* __restrict__ amax, uint32_t n_asks,
                               uint32_t* __restrict__ any_bad) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_asks) return;
  const uint32_t mx = amax[c];
  if (mx == 0) return;
  const uint32_t r = hist[c] % mx;
  if (r != 0 && r < amin[c]) *any_bad = 1u;
}

struct SweepParams {
  EvalParams ev;
  uint32_t* cur;             // [W] current ask of each worker
  uint32_t* base_len;        // [T] members still in the sorted base segment
  const uint32_t* seg_start; // [T]
  const uint32_t* order;     // [W] workers sorted by (ask, index)
  uint32_t* xhead;           // [T] list of workers bumped into the ask
  uint32_t* xnext;           // [W]
  uint32_t* xcount;          // [T]
  const uint32_t* amin;
  const uint32_t* amax;
  uint32_t* popped;          // [W] scratch
  uint32_t* n_bumped;
  const uint32_t* any_bad;   // written by pm_check_tails: 0 = no configuration has an under-filled tail, nothing to do
};

// Sequential-in-priority sweep (single CTA): configurations are final in
// increasing priority index; the first one with an under-filled tail hands its
// last `K mod max` members (largest canonical index — groups are cut from the
// front, mod.rs:554-561) to their next feasible configuration.
__global__ void __launch_bounds__(1024) pm_sweep(SweepParams p) {
  __shared__ uint32_t s_first_bad, s_npop;
  if (*p.any_bad == 0u) return;   // the common case costs one launch, not a host round trip
  const uint32_t T = p.ev.n_asks;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  uint32_t c_lo = 0;
  while (c_lo < T) {
    if (tid == 0) s_first_bad = kNone;
    __syncthreads();
    const uint32_t c = c_lo + tid;
    if (c < T) {
      const uint32_t mx = p.amax[c];
      if (mx) {
        const uint32_t r = (p.base_len[c] + p.xcount[c]) % mx;
        if (r && r < p.amin[c]) atomicMin(&s_first_bad, c);
      }
    }
    __syncthreads();
    const uint32_t cb = s_first_bad;
    if (cb == kNone) {
      c_lo += 1024;
      continue;
    }
    if (tid == 0) {
      uint32_t bl = p.base_len[cb], xc = p.xcount[cb];
      const uint32_t r = (bl + xc) % p.amax[cb];
      for (uint32_t i = 0; i < r; ++i) {
        uint32_t bx = kNone, bprev = kNone, prev = kNone;  // largest index among bumped-in
        for (uint32_t x = p.xhead[cb]; x != kNone; prev = x, x = p.xnext[x])
          if (bx == kNone || x > bx) { bx = x; bprev = prev; }
        const uint32_t bw = bl ? p.order[p.seg_start[cb] + bl - 1] : kNone;
        uint32_t take;
        if (bx != kNone && (bw == kNone || bx > bw)) {
          take = bx;
          if (bprev == kNone) p.xhead[cb] = p.xnext[bx];
          else p.xnext[bprev] = p.xnext[bx];
          --xc;
        } else {
          take = bw;
          --bl;
        }
        p.popped[i] = take;
      }
      p.base_len[cb] = bl;
      p.xcount[cb] = xc;
      s_npop = r;
    }
    __syncthreads();
    const uint32_t npop = s_npop;
    for (uint32_t i = warp; i < npop; i += 32) {
      const uint32_t w = p.popped[i];
      const WorkerReg wr = make_worker(p.ev.wa[w], p.ev.wb[w]);
      uint32_t found = kNone;
      for (uint32_t cbase = cb + 1; cbase < T; cbase += 32) {
        const uint32_t c2 = cbase + lane;
        bool ok = false;
        if (c2 < T) ok = ask_meets(p.ev.asks[c2], p.ev.opts, wr, p.ev.bits, p.ev.words);
        const uint32_t b = __ballot_sync(0xffffffffu, ok);
        if (b) {
          found = cbase + (uint32_t)__ffs(b) - 1u;
          break;
        }
      }
      if (lane == 0) {
        p.cur[w] = found;
        if (found != kNone) {
          const uint32_t old = atomicExch(&p.xhead[found], w);
          p.xnext[w] = old;
          atomicAdd(&p.xcount[found], 1u);
        }
        atomicAdd(p.n_bumped, 1u);
      }
    }
    __syncthreads();
    c_lo = cb + 1;
  }
}

// groups per bin (bin = ask << shift | located-first bit): full chunks of `max`
// plus the tail when it reaches `min` (mod.rs:545-566), plus the empty group a
// min_group_size == 0 configuration produces on its last iteration (:564,:606).
__global__ void pm_count_groups(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ amin,
                                const uint32_t* __restrict__ amax, uint32_t n_bins, uint32_t shift,
                                uint32_t* __restrict__ ngroups) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_bins) return;
  const uint32_t c = b >> shift, mx = amax[c], mn = amin[c], K = hist[b];
  uint32_t g = 0;
  if (mx) {
    g = K / mx;
    const uint32_t r = K % mx;
    if (r && r >= mn) ++g;
  }
  if (mn == 0 && (!shift || (b & 1u))) ++g;
  ngroups[b] = g;
}

// one thread per sorted position: worker -> (group, ask); group heads write the
// group table.  Positions past the formed groups of a bin (an unformed tail can
// only exist if the sweep was skipped by the caller) stay unassigned.
__global__ void pm_emit_workers(const uint32_t* __restrict__ keys_sorted,
                                const uint32_t* __restrict__ order, const uint32_t* __restrict__ n_assigned_dev,
                                const uint32_t* __restrict__ hist,
                                const uint32_t* __restrict__ seg_start,
                                const uint32_t* __restrict__ group_base,
                                const uint32_t* __restrict__ amin, const uint32_t* __restrict__ amax,
                                uint32_t shift, uint32_t* __restrict__ worker_group,
                                uint32_t* __restrict__ worker_ask, uint32_t* __restrict__ group_ask,
                                uint32_t* __restrict__ group_off) {
  uint32_t pidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (pidx >= *n_assigned_dev) return;   // launched over all workers: no host read of the count
  const uint32_t b = keys_sorted[pidx], c = b >> shift, w = order[pidx];
  const uint32_t mx = amax[c], K = hist[b], r = pidx - seg_start[b];
  if (mx == 0) return;
  const uint32_t full = K / mx, rem = K % mx;
  if (r >= full * mx && rem < amin[c]) return;  // unformed tail
  const uint32_t g = group_base[b] + r / mx;
  worker_group[w] = g;
  worker_ask[w] = c;
  if (r % mx == 0) {
    group_ask[g] = c;
    group_off[g] = pidx;
  }
}

// the trailing empty group of min_group_size == 0 configurations
__global__ void pm_emit_empty_groups(const uint32_t* __restrict__ hist,
                                     const uint32_t* __restrict__ seg_start,
                                     const uint32_t* __restrict__ group_base,
                                     const uint32_t* __restrict__ ngroups,
                                     const uint32_t* __restrict__ amin, uint32_t n_bins,
                                     uint32_t shift, uint32_t* __restrict__ group_ask,
                                     uint32_t* __restrict__ group_off) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_bins) return;
  const uint32_t c = b >> shift;
  if (amin[c] != 0 || (shift && !(b & 1u))) return;
  const uint32_t g = group_base[b] + ngroups[b] - 1;
  group_ask[g] = c;
  group_off[g] = seg_start[b] + hist[b];
}

// members of a group in BTreeSet<String> order (mod.rs:63-69): position = number
// of members whose address rank is smaller.
__global__ void pm_order_members(const uint32_t* __restrict__ order, const uint32_t* __restrict__ n_assigned_dev,
                                 const uint32_t* __restrict__ worker_group,
                                 const uint32_t* __restrict__ group_off,
                                 const uint32_t* __restrict__ addr_rank,
                                 uint32_t* __restrict__ members) {
  uint32_t pidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (pidx >= *n_assigned_dev) return;
  const uint32_t w = order[pidx];
  const uint32_t g = worker_group[w];
  if (g == kNone) { members[pidx] = w; return; }
  const uint32_t gs = group_off[g], ge = group_off[g + 1];
  uint32_t pos = 0;
  // without address ranks the row index stands in for the address order
  const uint32_t mine = addr_rank ? addr_rank[w] : w;
  for (uint32_t q = gs; q < ge; ++q) {
    const uint32_t o = order[q];
    pos += ((addr_rank ? addr_rank[o] : o) < mine) ? 1u : 0u;
  }
  members[gs + pos] = w;
}

// The CSR end marker group_off[G] and the pass's scalars {G, members, bumped}, written on the device so the
// resolution chain needs no host round trip before its last kernel.
__global__ void pm_close_groups(const uint32_t* __restrict__ n_groups_dev, const uint32_t* __restrict__ n_assigned_dev,
                                const uint32_t* __restrict__ n_bumped_dev, uint32_t* __restrict__ group_off,
                                uint32_t* __restrict__ scalars) {
  const uint32_t G = *n_groups_dev, M = *n_assigned_dev;
  group_off[G] = M;
  scalars[0] = G;
  scalars[1] = M;
  scalars[2] = *n_bumped_dev;
}

// ------------------------------------------------------------------ multi-GPU exchange (SURVEY 8e)
// One rank's contribution to the single collective of a sharded pass, packed into one buffer:
//   [ ask_best int64[T] | ask_count u32[T] | first_ask of the rank's own worker range u32[per] ]
// (`per` = ceil(W / ranks): every rank sends the same size; the last rank's tail is padding.)
__global__ void pm_xchg_pack(const uint32_t* __restrict__ first_ask_shard, uint32_t nw, uint32_t per,
                             const long long* __restrict__ ask_best, const uint32_t* __restrict__ ask_count, uint32_t T,
                             unsigned char* __restrict__ send) {
  long long* s_best = reinterpret_cast<long long*>(send);
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(send + (size_t)T * 8);
  uint32_t* s_first = s_cnt + T;
  const size_t n = (size_t)max(T, per);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (i < T) { s_best[i] = ask_best[i]; s_cnt[i] = ask_count[i]; }
    if (i < per) s_first[i] = i < nw ? first_ask_shard[i] : kNone;
  }
}

// After the all-gather: every rank folds the `ranks` contributions into the same global arrays — per ask the
// packed (cost, worker) minimum and the feasible-count sum, per worker the first feasible ask from its owner.
__global__ void pm_xchg_unpack(const unsigned char* __restrict__ recv, uint32_t ranks, size_t stride, uint32_t per,
                               uint32_t W, uint32_t T, uint32_t* __restrict__ first_ask,
                               long long* __restrict__ ask_best, uint32_t* __restrict__ ask_count) {
  const size_t n = (size_t)max(T, W);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (i < T) {
      long long best = kInf;
      uint32_t cnt = 0;
      for (uint32_t r = 0; r < ranks; ++r) {
        const unsigned char* base = recv + (size_t)r * stride;
        best = min(best, reinterpret_cast<const long long*>(base)[i]);
        cnt += reinterpret_cast<const uint32_t*>(base + (size_t)T * 8)[i];
      }
      ask_best[i] = best;
      ask_count[i] = cnt;
    }
    if (i < W) {
      const uint32_t r = (uint32_t)(i / per);
      const uint32_t* f = reinterpret_cast<const uint32_t*>(recv + (size_t)r * stride + (size_t)T * 12);
      first_ask[i] = f[i - (size_t)r * per];
    }
  }
}

}  // namespace pm
