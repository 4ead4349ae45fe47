// pm_auction_cert.cuh — NORTH-STAR EXTENSION: a certificate for the last auction pass (pm_auction_certificate).
//
// Weak LP duality for the auction's problem (one worker per ask, an ask may stay unheld at its outside cost):
// for ANY prices p >= 0,
//     LB = sum_t min((cap[t] + 1) * S, min over feasible w of key(w)) - sum_w p[w],   key(w) = ask_price[w] * S + p[w]
// is a lower bound on the optimal total cost, whatever produced p.  The stored assignment's cost is
//     cost = sum over held asks of ask_price[w_t] * S + sum over unheld asks of (cap[t] + 1) * S,
// so gap = cost - LB bounds its distance from the optimum.  When no hold is shared,
//     gap = sum_t slack(t) + sum of the prices of unowned workers,
// slack(t) = key(w_t) (held) or (cap[t] + 1) * S (unheld) minus the row term above: eps-CS with every unowned worker at
// price 0 gives gap <= T * eps (DESIGN 4).
//
// The certificate shares nothing with the auction's machinery (class caches, sorted planes, skip keys, pools): the
// row terms come from one sweep over every (ask, worker) pair built from the fused pass's pieces (load_workers,
// for_each_staged_row, eval_row_fast / eval_row / eval_row_global, every BITS form, the worker-major `nacc` word), so
// the predicate is the fused pass's by construction; ownership is recounted from the assignment.  Every sum is exact:
// each term (< 2^64) is added as its two 32-bit halves into separate 64-bit counters, and the host joins them in 128 bits.
#pragma once
#include <climits>
#include "pm_kernels.cuh"

namespace pm {

// accumulators of one certificate (zeroed before the kernels)
enum CertAcc : int {
  kCertCostLo, kCertCostHi,       // sum of the asks' costs (32-bit halves)
  kCertRowLo, kCertRowHi,         // sum of the row terms min(outside, least feasible key)
  kCertPriceLo, kCertPriceHi,     // sum of every worker's price
  kCertFreeLo, kCertFreeHi,       // sum of the prices of unowned workers with price > 0
  kCertHeld, kCertBadHolds, kCertSlackOver, kCertMaxSlack,   // max slack: int64 ^ 2^63, so that 0 is the least
  kCertShared, kCertFree, kCertMaxAskPrice,
  kCertAccWords
};

struct CertParams {
  const long long* __restrict__ price;       // [W] stored prices
  const uint32_t* __restrict__ rep;          // [W] reputation, or null: a column of zeros
  const uint32_t* __restrict__ cap;          // [T]
  const uint32_t* __restrict__ floor;        // [T] reputation floors, or null: no clause
  const uint32_t* __restrict__ assigned;     // [T] stored assignment (PM_NONE: unheld)
  unsigned long long* __restrict__ row_min;  // [T] least feasible key, ~0 before the sweep
  uint32_t* __restrict__ held_ok;            // [T] the held pair is feasible (written for held asks only); per slot, [D],
                                             // with demands (pm_auction_cert_slots)
  uint32_t* __restrict__ own;                // [W] asks holding the worker, zero before pm_auction_cert_asks
  long long* __restrict__ ask_bound;         // [T] the row terms
  unsigned long long* __restrict__ acc;      // [kCertAccWords]
  unsigned long long scale;
  uint32_t n_workers, n_asks;
};

__device__ __forceinline__ unsigned long long cert_warp_sum(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// adds v (< 2^64) to the 128-bit sum kept as two halves at acc[i], acc[i + 1]; one atomic per warp and half
__device__ __forceinline__ void cert_add128(unsigned long long* acc, int i, unsigned long long v) {
  const unsigned long long lo = cert_warp_sum(v & 0xFFFFFFFFull), hi = cert_warp_sum(v >> 32);
  if ((threadIdx.x & 31u) == 0u) {
    if (lo) atomicAdd(acc + i, lo);
    if (hi) atomicAdd(acc + i + 1, hi);
  }
}

__device__ __forceinline__ void cert_count(unsigned long long* acc, int i, bool b) {
  const uint32_t n = __popc(__ballot_sync(0xffffffffu, b));
  if ((threadIdx.x & 31u) == 0u && n) atomicAdd(acc + i, (unsigned long long)n);
}

// ------------------------------------------------------------------ the sweep
// grid = (ceil(W / 1024), ceil(nt / 128)), as pm_fused_eval: each thread holds 4 workers in registers with their key
// ask_price * S + price (64-bit) and reputation, and walks the CTA's staged asks.  Per row: feasible = the fused
// predicate && ask_price <= cap[t] && reputation >= floor[t] (pm_auction.cuh's feasible(t, w)); the row's least feasible
// key is taken per warp in two steps (the least high word, then the least low word among the lanes at that high word)
// and per CTA with a shared-memory atomicMin.  The lane that holds the ask's assigned worker records whether that pair
// is feasible: a hold that table changes made infeasible shows up at no extra cost.
template <int BITS, bool FAST>
__global__ void __launch_bounds__(kEvalThreads, 2)
pm_auction_cert_sweep(EvalParams p, CertParams c, uint32_t t0, uint32_t nt) {
  __shared__ EvalStage s;
  __shared__ unsigned long long s_min[kEvalRows];
  __shared__ uint32_t s_cap[kEvalRows], s_floor[kEvalRows], s_held[kEvalRows];
  const uint32_t r0 = blockIdx.y * kEvalRows;
  const uint32_t r1 = min(nt, r0 + (uint32_t)kEvalRows);
  for (uint32_t i = threadIdx.x; i < (uint32_t)kEvalRows; i += kEvalThreads) {
    s_min[i] = ~0ull;
    const uint32_t t = t0 + r0 + i;
    const bool in = r0 + i < r1;
    s_cap[i] = in ? __ldg(c.cap + t) : 0u;
    s_floor[i] = in && c.floor ? __ldg(c.floor + t) : 0u;
    s_held[i] = in ? __ldg(c.assigned + t) : kNone;
  }   // (for_each_staged_row's first barrier publishes these before any row is visited)
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t col = blockIdx.x * kEvalCols + threadIdx.x * kEvalWPT;
  WorkerReg w[kEvalWPT];
  load_workers<kEvalWPT>(p, 0u, c.n_workers, col, w);
  unsigned long long key[kEvalWPT];
  uint32_t rep[kEvalWPT];
#pragma unroll
  for (int k = 0; k < kEvalWPT; ++k) {
    const bool in = col + k < c.n_workers;
    key[k] = in ? (unsigned long long)w[k].price * c.scale + (unsigned long long)__ldg(c.price + col + k) : ~0ull;
    rep[k] = in && c.rep ? __ldg(c.rep + col + k) : 0u;
  }
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
    const uint32_t cap = s_cap[r], fl = s_floor[r], dh = s_held[r] - col;   // dh < 4: this thread holds the ask's worker
    unsigned long long m = ~0ull;
#pragma unroll
    for (int k = 0; k < kEvalWPT; ++k) {
      const bool ok = f[k] != 0u && w[k].price <= cap && rep[k] >= fl;
      if (ok) m = min(m, key[k]);
      if (dh == (uint32_t)k) c.held_ok[t0 + r0 + r] = ok ? 1u : 0u;
    }
    const uint32_t hi = __reduce_min_sync(0xffffffffu, (uint32_t)(m >> 32));
    const uint32_t lo = __reduce_min_sync(0xffffffffu, (uint32_t)(m >> 32) == hi ? (uint32_t)m : 0xFFFFFFFFu);
    if (lane == 0 && hi != 0xFFFFFFFFu) atomicMin(&s_min[r], ((unsigned long long)hi << 32) | lo);   // keys < 2^62
  });
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < r1 - r0; i += kEvalThreads)
    if (s_min[i] != ~0ull) atomicMin(c.row_min + t0 + r0 + i, s_min[i]);
}

// ------------------------------------------------------------------ per ask
// The row term min(outside, least feasible key), the ask's cost and slack, whether its hold is feasible, and the
// ownership count of its worker (recounted here from the assignment, not read from the auction's owner array).
__global__ void pm_auction_cert_asks(CertParams c, const uint4* __restrict__ wb) {
  const uint32_t n = c.n_asks;
  for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {   // warp-uniform trip count
    const uint32_t t = base + threadIdx.x;
    const bool in = t < n;
    unsigned long long cost = 0, bound = 0;
    long long slack = LLONG_MIN;
    bool held = false, bad = false;
    if (in) {
      const unsigned long long outside = ((unsigned long long)__ldg(c.cap + t) + 1ull) * c.scale;
      bound = min(outside, c.row_min[t]);
      c.ask_bound[t] = (long long)bound;
      const uint32_t a = __ldg(c.assigned + t);
      held = a < c.n_workers;
      if (held) {
        cost = (unsigned long long)__ldg(&wb[a].w) * c.scale;
        slack = (long long)(cost + (unsigned long long)__ldg(c.price + a)) - (long long)bound;
        bad = c.held_ok[t] == 0u;
        atomicAdd(c.own + a, 1u);
      } else {
        cost = outside;
        slack = (long long)(outside - bound);
      }
    }
    cert_add128(c.acc, kCertCostLo, cost);
    cert_add128(c.acc, kCertRowLo, bound);
    cert_count(c.acc, kCertHeld, held);
    cert_count(c.acc, kCertBadHolds, bad);
    cert_count(c.acc, kCertSlackOver, in && slack > 1);
    long long ms = slack;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ms = max(ms, __shfl_xor_sync(0xffffffffu, ms, o));
    if ((threadIdx.x & 31u) == 0u && ms != LLONG_MIN)
      atomicMax(c.acc + kCertMaxSlack, (unsigned long long)ms ^ 0x8000000000000000ull);
  }
}

// ------------------------------------------------------------------ per slot (ask demands)
// With demands (pm_set_ask_demand) the sweep stays per ask, T x W (every slot of an ask has the ask's row term), run
// with no holds, and this pass takes pm_auction_cert_asks' place over the slots: slot s of ask slot_ask[s] adds the
// ask's row term, so the row sum is sum_t d[t] * row(t), and its own hold's cost, slack and ownership count.  A held
// pair's feasibility is checked here with the predicate of eval_row_global (ask_meets), cap and floor as in the sweep,
// and stored per slot in held_ok (D entries; written for held slots only), which pm_auction_restore_asks reads.
// c.assigned is the slots' assignment; the ask's first slot writes ask_bound.
__global__ void pm_auction_cert_slots(CertParams c, EvalParams p, const uint32_t* __restrict__ slot_ask, uint32_t n_slots) {
  for (uint32_t base = blockIdx.x * blockDim.x; base < n_slots; base += gridDim.x * blockDim.x) {   // warp-uniform trip count
    const uint32_t s = base + threadIdx.x;
    const bool in = s < n_slots;
    unsigned long long cost = 0, bound = 0;
    long long slack = LLONG_MIN;
    bool held = false, bad = false;
    if (in) {
      const uint32_t t = __ldg(slot_ask + s);
      const uint32_t cap = __ldg(c.cap + t);
      const unsigned long long outside = ((unsigned long long)cap + 1ull) * c.scale;
      bound = min(outside, c.row_min[t]);
      if (s == 0 || __ldg(slot_ask + s - 1) != t) c.ask_bound[t] = (long long)bound;
      const uint32_t a = __ldg(c.assigned + s);
      held = a < c.n_workers;
      if (held) {
        const WorkerReg wr = make_worker(__ldg(p.wa + a), __ldg(p.wb + a));
        const uint32_t rep = c.rep ? __ldg(c.rep + a) : 0u, fl = c.floor ? __ldg(c.floor + t) : 0u;
        bad = !(wr.price <= cap && rep >= fl && ask_meets(p.asks[t], p.opts, wr, p.bits, p.words));
        c.held_ok[s] = bad ? 0u : 1u;
        cost = (unsigned long long)wr.price * c.scale;
        slack = (long long)(cost + (unsigned long long)__ldg(c.price + a)) - (long long)bound;
        atomicAdd(c.own + a, 1u);
      } else {
        cost = outside;
        slack = (long long)(outside - bound);
      }
    }
    cert_add128(c.acc, kCertCostLo, cost);
    cert_add128(c.acc, kCertRowLo, bound);
    cert_count(c.acc, kCertHeld, held);
    cert_count(c.acc, kCertBadHolds, bad);
    cert_count(c.acc, kCertSlackOver, in && slack > 1);
    long long ms = slack;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ms = max(ms, __shfl_xor_sync(0xffffffffu, ms, o));
    if ((threadIdx.x & 31u) == 0u && ms != LLONG_MIN)
      atomicMax(c.acc + kCertMaxSlack, (unsigned long long)ms ^ 0x8000000000000000ull);
  }
}

// ------------------------------------------------------------------ per worker
// Every price into sum_w p[w]; the shared holds; the unowned workers with a positive price; the largest ask price of
// the table (the integer domain's P).  After pm_auction_cert_asks (the ownership counts).
__global__ void pm_auction_cert_workers(CertParams c, const uint4* __restrict__ wb) {
  const uint32_t n = c.n_workers;
  for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
    const uint32_t w = base + threadIdx.x;
    const bool in = w < n;
    unsigned long long pr = 0;
    uint32_t own = 0, ap = 0;
    if (in) {
      pr = (unsigned long long)__ldg(c.price + w);   // >= 0: every price the auction sets
      own = c.own[w];
      ap = __ldg(&wb[w].w);
    }
    const bool free_priced = in && own == 0u && pr != 0ull;
    cert_add128(c.acc, kCertPriceLo, pr);
    cert_add128(c.acc, kCertFreeLo, free_priced ? pr : 0ull);
    cert_count(c.acc, kCertShared, own > 1u);
    cert_count(c.acc, kCertFree, free_priced);
    const uint32_t mp = __reduce_max_sync(0xffffffffu, ap);
    if ((threadIdx.x & 31u) == 0u && mp) atomicMax(c.acc + kCertMaxAskPrice, (unsigned long long)mp);
  }
}

// ------------------------------------------------------------------ restore (pm_auction_restore, pm_auction_restore_slots)
// The caller's state is audited by the certificate's own sweep and per-ask (or per-slot) pass (CertParams pointed at
// the staged prices and assignment): row terms, held-pair feasibility and ownership counts.  Then one decision per
// bidder and one pass over the workers, both into staging buffers; the engine copies them over the stored state once
// nothing can refuse any more.  Prices are never changed: a dropped hold's worker is unowned at its given price.
enum RestoreAcc : int { kRstHeld, kRstBad, kRstShared, kRstSlack, kRstAccWords };
constexpr uint32_t kRstHolder = 0x80000000u;   // own[w] after the audit: kRstHolder | b for the kept hold of bidder b

// Per bidder b < n, after pm_auction_cert_asks (the asks: slot_ask null, n = T) or pm_auction_cert_slots (the slots of
// ask demands: slot_ask the slot -> ask map, n = D): a hold is dropped when it is infeasible, else when its worker is
// named by more than one bidder, else when its slack key(w_b) - row(ask of b) exceeds 1; a kept hold marks its worker's
// count (1: nobody else writes it; counts and bidder indices stay below 2^30, so the mark is told apart).
__global__ void pm_auction_restore_asks(CertParams c, const uint4* __restrict__ wb, const uint32_t* __restrict__ slot_ask,
                                        uint32_t n, uint32_t* __restrict__ kept, unsigned long long* __restrict__ acc) {
  for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {   // warp-uniform trip count
    const uint32_t b = base + threadIdx.x;
    bool keep = false, bad = false, shared = false, over = false;
    if (b < n) {
      const uint32_t a = __ldg(c.assigned + b);
      if (a < c.n_workers) {
        bad = c.held_ok[b] == 0u;
        shared = !bad && c.own[a] > 1u;
        if (!bad && !shared) {
          const uint32_t t = slot_ask ? __ldg(slot_ask + b) : b;
          const unsigned long long key = (unsigned long long)__ldg(&wb[a].w) * c.scale + (unsigned long long)__ldg(c.price + a);
          over = (long long)key - c.ask_bound[t] > 1;
          keep = !over;
        }
        if (keep) c.own[a] = kRstHolder | b;
      }
      kept[b] = keep ? a : kNone;
    }
    cert_count(acc, kRstHeld, keep);
    cert_count(acc, kRstBad, bad);
    cert_count(acc, kRstShared, shared);
    cert_count(acc, kRstSlack, over);
  }
}

// Per worker, after pm_auction_restore_asks: the owner array of the kept holds (ask indices, or slot indices with
// demands: what the auction's kernels read)
__global__ void pm_auction_restore_workers(const uint32_t* __restrict__ own, uint32_t n_workers, uint32_t* __restrict__ owner) {
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < n_workers; w += gridDim.x * blockDim.x) {
    const uint32_t o = own[w];
    owner[w] = (o & kRstHolder) ? (o & ~kRstHolder) : kNone;
  }
}

}  // namespace pm
