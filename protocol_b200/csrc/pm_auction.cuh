// pm_auction.cuh — NORTH-STAR EXTENSION: price-capped forward auction (one worker per ask, or per slot of an ask's
// demand: the kernels run on the slot table as on an ask table, "ask demands" at the end).
//
// The reference orchestrator has no prices, caps, reputation or auction (SURVEY.md 0):
// nothing here restates reference code, and parity for this mode is against the
// builder's own sequential restatement (the auction checker of the test suite) —
// "self-oracle, parity unpinned by the reference".  The mode is inert unless
// PM_MODE_AUCTION is requested; the reference modes never read ext_ask_price.
//
// Synchronous (Jacobi) Bertsekas auction:
//   feasible(t,w) = candidate(w) && compatible(t,w) && ask_price[w] <= price_cap[t]
//                   && reputation[w] >= min_reputation[t]   (the north-star `reputation` column; both default to 0.
//                   The floor is part of the ask's class, so cached and pooled workers never need the test again.)
//   value(t,w)    = -(ask_price[w] * S) - price[w]      outside(t) = -((price_cap[t] + 1) * S)
//   bid(t)        = price[w1] + (best - max(second, outside)) + eps    on the best worker w1
//   a worker takes the highest bid (ties: lowest ask index), releasing its previous owner.
//
// What makes a round cheap (every bid stays bit-identical to a full scan of all workers by every
// unassigned ask every round, which is what the sequential checker does):
//
//  * ASK CLASSES.  value(t,w) does not depend on t; only feasibility does.  Asks with identical
//    requirement rows form a class (found on the device: content hash, radix sort, adjacent
//    compare — a hash collision can only split a class, never merge two).  A class keeps ONE cache
//    of its 32 best compatible workers (cap ignored) and the bound (theta, theta_w): every
//    compatible worker outside the cache ranked at or below it at scan time, and prices only
//    rise, so it still does.
//  * THE CAP IS THE OUTSIDE OPTION.  A worker with ask_price > cap[t] has value <= outside(t), so
//    it can neither raise max(second, outside) nor beat a bid-worthy best: an ask's bid follows
//    from the class cache as  w1 = best cached worker with ask_price <= cap,
//    second = max(best cached value other than w1, outside)  whenever w1 beats (theta, theta_w)
//    and theta <= max(that value, outside); it withdraws when nothing cached or bounded by theta
//    can reach outside(t).  Anything else is "ambiguous": the class is rescanned once for all its
//    asks (pm_auction_scan, class mode) and the ask bids again; an ask that is still ambiguous
//    after a fresh class scan (a value tie exactly at outside) gets its own cap-filtered scan.
//  * COST-SORTED WORKERS.  Scans walk a copy of the worker table sorted by (ask_price * S + price,
//    index) as of the last sort (redone every few batches of rounds).  Prices only rise, so a
//    worker's value is at most minus its sort key: once 33 kept candidates beat the key of the
//    stripe's last worker no later worker can enter the top 32 or the bound, and the walk stops —
//    after a stripe or two for most classes, because the workers whose prices were bid up have
//    moved back in the order.
//  * SKIP TO THE CLASS'S COST LEVEL.  A class whose compatible workers are all expensive (eight H100s) would walk
//    through the cheap end of the table every time — tens of stripes with nobody in them.  Compatibility of a
//    (class, worker) pair never changes during an auction and sort keys only rise, so "no compatible worker has a
//    key below K" stays true for good once a walk has seen it: every walk records the key at which it met its first
//    compatible worker and the next one starts at the stripe that key falls into (a 32-ary search over stripe ends).
//  * CLASS POOL.  The candidates the lanes held at the end of a walk (up to 1024) stay as the
//    class's pool; a rescan request first re-ranks the pool at the current prices and walks the
//    table only when the pool's best two no longer beat the bound on everything outside it.
//  * SPLIT WALKS.  When a round has few walks (the long tail of an auction: a handful of scarce
//    classes), each is split over up to 16 CTAs that take interleaved stripes; every part leaves
//    its top 32 and one bound, and the part that arrives last (a ticket) merges them.
//  * DEVICE-DRIVEN ROUNDS.  List lengths live in device memory; every kernel of a round is
//    launched with a fixed grid and strides over its list, so the host launches rounds in batches
//    (32 rounds = one CUDA graph) and only polls the number of unassigned asks.  A round is 6 launches:
//    bid from the caches, pool re-rank, class walks, bid again, per-ask scans, apply (which also
//    writes the next round's active list and advances the round).
//  * FEWER INSTRUCTIONS.  The kernels of a round are issue-bound, not memory-bound (the whole worker
//    table fits in L2, and every round is a chain of dependent launches): the selection of the top 32 is a bitonic
//    network in shared memory that keeps the best 64 only, on ONE packed 64-bit key per candidate when
//    every reachable cost fits 40 bits (auction_select_cta); the claim is the atomicMax itself when bid
//    and bidder fit one word (auction_commit).
//
// pm_auction_scan: stripes of the sorted worker planes, their prices and original indices are
// staged into shared memory with 1-D TMA bulk copies, double-buffered; one item per CTA (its 8 warps split
// each stripe), items drawn from a counter because their lengths differ by two orders of magnitude.
// Collisions are resolved by atomicMax on (bid, bidder) packed in one word — or, when they do not fit, by atomicMax on
// the bid and atomicMin on the bidder (pm_auction_claim) — applied by the single winner of each worker.
//
// PM_AUCTION_REVERSE ends every eps phase with reverse rounds (the section at the end): they only lower prices, so the
// engine rebuilds the class caches and the worker order after a stage that lowered one.  PM_AUCTION_REPAIR's raise
// (pm_auction_repair_raise) reuses the reverse bid's gain walk before the forward rounds and ends with a reverse stage.
#pragma once
#include "pm_kernels.cuh"

namespace pm {

constexpr int kAucThreads = 256;
constexpr int kAucWarps = kAucThreads / 32;
constexpr int kAucStripe = 1024;  // workers staged per step
constexpr int kAucStages = 2;     // stripes in flight per CTA
constexpr long long kAucNeg = (long long)(0x8000000000000000ull) / 4;
constexpr int kAucCache = 32;
constexpr int kAucPool = 1024;       // pool slots per class (4 per thread of the scanning CTA)
constexpr int kAucPoolGood = 256;    // a class walk goes on until this many candidates beat every unseen worker ...
constexpr int kAucPoolExtra = 8;     // ... or for this many stripes past the point where it could have stopped
constexpr int kAucClaimShift = 23;                       // packed claim: bids below 2^40, fewer than 2^23 asks
constexpr uint32_t kAucClaimMask = (1u << kAucClaimShift) - 1u;
constexpr long long kThetaComplete = (long long)0x8000000000000000ull;   // the cache holds every compatible worker
constexpr long long kThetaInvalid = 0x7FFFFFFFFFFFFFFFll;                // no cache yet

// device-side control block of the round loop
struct AuctionCtl {
  uint32_t n_active;     // unassigned, not withdrawn asks of the current round
  uint32_t n_next;       // ... being collected for the next one
  uint32_t n_cls;        // classes whose cache must be refreshed this round
  uint32_t n_walk;       // ... of which the pool could not decide: they walk the worker table
  uint32_t n_retry;      // asks that bid again after the class rescans
  uint32_t n_fallback;   // asks that need their own scan
  uint32_t rounds;       // rounds in which at least one ask was active
  uint32_t flip;         // which half of active[] holds the current round's list (the other half collects the next one)
  uint32_t ticket;       // blocks of pm_auction_apply that are through: the last one advances the round
  uint32_t walk_taken, fb_taken;   // items of the round's walk / fallback list already drawn by a scanning CTA
  uint32_t max_ask_price, max_cap; // over the worker table / the asks (pm_auction_limits)
  uint32_t packed;                 // every reachable cost < 2^40 and fewer than 2^24 workers: selections sort packed keys
  uint32_t packed_claim;           // ... and fewer than 2^23 asks: bid_max[] holds (bid, bidder), pm_auction_claim has nothing to do
  unsigned long long evals;
  unsigned long long n_class_scans, n_ask_scans, n_refills;
  uint32_t n_released;             // warm start: asks released from the stored assignment
  uint32_t n_raised;               // ... workers whose price was reset (the list R of the release closure)
  uint32_t n_bid;                  // reverse stage: bidders of the current round (unowned, positive price)
  uint32_t rev_last;               // ... of the last round run (0: the stage is over)
  uint32_t rev_rounds;             // ... rounds with at least one bidder, over the pass
  uint32_t rev_lowered;            // ... some price went down since the host last cleared this
  unsigned long long rev_bids;     // ... bids over the pass
};

struct AuctionParams {
  EvalParams ev;               // original worker order (gathers); asks / options / model bits
  const uint4* wa_s;           // worker planes sorted by (cost at the last sort, index)
  const uint4* wb_s;
  const uint32_t* perm;        // [W] sorted position -> worker
  const uint32_t* pos_of;      // [W] worker -> sorted position
  long long* price_s;          // [W + 2] price mirror in sorted order
  const unsigned long long* csort_s;  // [W] the sort key: ask_price * S + price at the time of the last sort
  const uint32_t* price_cap;   // [T]
  const uint32_t* rep_s;       // [W + 4] `reputation` column in sorted order, or null (no reputation clause)
  const uint32_t* min_rep;     // [T] per-ask floor on it (part of the ask's class); null with rep_s
  long long* price;            // [W] dual price of each worker
  uint32_t* owner;             // [W] ask currently holding the worker
  uint32_t* assigned;          // [T] worker held by the ask
  uint32_t* withdrawn;         // [T]
  uint32_t* active;            // [2 * T] the round's active asks | the next round's, roles swapped by ctl->flip
  uint32_t n_asks;
  uint32_t* bid_w;             // [T]
  long long* bid_p;            // [T]
  long long* bid_max;          // [W] highest bid of the round (reset by the winner)
  uint32_t* winner;            // [W]
  const uint32_t* class_of;    // [T]
  const uint32_t* class_rep;   // [C] lowest ask of the class
  uint32_t* class_req;         // [C] round stamp of the last rescan request
  uint32_t* cand;              // [C * 32] cached best compatible workers of each class
  long long* theta;            // [C]
  uint32_t* theta_w;           // [C]
  uint32_t* pool;              // [C * kAucPool] candidates of the class's last walk
  long long* pool_bound_v;     // [C] every compatible worker outside the pool ranks at or below this
  uint32_t* pool_bound_w;      // [C]
  uint32_t* class_list;        // [C]
  uint32_t* walk_list;         // [C]
  long long* split_bound_v;    // [grid * 16] per-part bounds of a walk split over several CTAs
  uint32_t* split_bound_w;
  uint32_t* split_ticket;      // [grid]
  uint32_t* split_first;       // [grid] first stripe in which any part of a split walk met a compatible worker
  unsigned long long* skip_key;  // [C] every compatible worker of the class has a sort key >= this (keys only rise)
  uint32_t* retry;             // [T]
  uint32_t* fallback;          // [T]
  AuctionCtl* ctl;
  long long scale, eps;
  uint32_t pool_good, pool_extra;   // pool fill of a class walk (kAucPoolGood / kAucPoolExtra unless PM_TUNE_AUCTION_POOL=good,extra)
  uint32_t dbg;                // PM_TUNE_AUCTION: 1 = no early exit, 2 = every ask scans for itself
};

struct __align__(128) AuctionStage {
  uint4 a[kAucStripe];
  uint4 b[kAucStripe];
  long long price[kAucStripe];
  uint32_t perm[kAucStripe];
  uint32_t rep[kAucStripe];
  uint64_t bar;
};

// The scan's predicate: the generic clause masks of pm_kernels.cuh (predicated PTX, no branches) with the class's
// first option row held in registers for the whole walk (nine asks in ten have one option); same result as ask_meets.
__device__ __forceinline__ bool auc_meets(const DevAsk& a, const DevOpt& q0, const DevOpt* __restrict__ opts, const WorkerReg& w,
                                          const uint32_t* __restrict__ bits, uint32_t words) {
  uint32_t ok = base_mask(a, w);
  if (a.n_opts != 0u) {
    uint32_t any = opt_mask(q0, w, q0.pattern_row ? bits[q0.pattern_row * words + w.mword] : 0xFFFFFFFFu);   // row 0: no model clause
    for (uint32_t o = 1; o < a.n_opts; ++o) {
      const DevOpt q = opts[a.opt_off + o];
      any |= opt_mask(q, w, q.pattern_row ? bits[q.pattern_row * words + w.mword] : 0xFFFFFFFFu);
    }
    ok &= any;
  }
  return ok != 0u;
}

__device__ __forceinline__ const uint32_t* auc_active(const AuctionParams& p) { return p.active + (p.ctl->flip ? p.n_asks : 0u); }
__device__ __forceinline__ uint32_t* auc_next(const AuctionParams& p) { return p.active + (p.ctl->flip ? 0u : p.n_asks); }
__device__ __forceinline__ void auc_advance(AuctionCtl* ctl, int first) {
  if (!first && ctl->n_active) ++ctl->rounds;
  ctl->n_active = ctl->n_next;
  ctl->n_next = 0;
  ctl->n_cls = 0;
  ctl->n_walk = 0;
  ctl->n_retry = 0;
  ctl->n_fallback = 0;
  ctl->flip ^= 1u;
  ctl->ticket = 0;
  ctl->walk_taken = 0;
  ctl->fb_taken = 0;
}

__device__ __forceinline__ bool auc_better(long long v1, uint32_t w1, long long v2, uint32_t w2) {
  return v1 > v2 || (v1 == v2 && w1 < w2);
}

__device__ __forceinline__ void auction_withdraw(const AuctionParams& p, uint32_t t) {
  p.withdrawn[t] = 1u;       // prices only rise: it can never come back
  p.bid_w[t] = kNone;
}
__device__ __forceinline__ void auction_commit(const AuctionParams& p, uint32_t t, uint32_t w1, long long b1, long long second) {
  const long long bid = p.price[w1] + (b1 - second) + p.eps;
  p.bid_w[t] = w1;
  p.bid_p[t] = bid;
  // packed claim: bid and bidder in one word, (bid << 23) | (2^23 - 1 - ask) — the highest bid wins, among equal bids the
  // lowest ask: the atomicMax IS the claim (no separate pass over the bidders)
  atomicMax(p.bid_max + w1, p.ctl->packed_claim ? ((bid << kAucClaimShift) | (long long)(kAucClaimMask - t)) : bid);
}
// exact top-2 over the ask's feasible workers -> bid or withdrawal
__device__ __forceinline__ void auction_place_bid(const AuctionParams& p, uint32_t t, uint32_t cap,
                                                  long long b1, uint32_t w1, long long b2) {
  const long long outside = -(((long long)cap + 1) * p.scale);
  if (w1 == kNone || b1 < outside) auction_withdraw(p, t);
  else auction_commit(p, t, w1, b1, max(b2, outside));
}

// (value desc, worker asc) arg-max across the warp; returns the winning lane (the same on every lane)
__device__ __forceinline__ uint32_t warp_argbest(long long v, uint32_t w, long long* bv, uint32_t* bw) {
  uint32_t lane_id = threadIdx.x & 31u;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const long long ov = __shfl_xor_sync(0xffffffffu, v, off);
    const uint32_t ow = __shfl_xor_sync(0xffffffffu, w, off);
    const uint32_t ol = __shfl_xor_sync(0xffffffffu, lane_id, off);
    if (ov > v || (ov == v && (ow < w || (ow == w && ol < lane_id)))) { v = ov; w = ow; lane_id = ol; }
  }
  *bv = v;
  *bw = w;
  return lane_id;
}
__device__ __forceinline__ long long warp_max_i64(long long v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}

struct AuctionMerge {   // per-CTA control words of a walk
  uint32_t cnt[3];  // good candidates after stripe k (three slots in rotation: one barrier per stripe)
  uint32_t flag;
  uint32_t j0;      // first stripe of the walk (class mode: where the class's compatible workers begin)
  uint32_t first;   // first stripe in which the CTA met a compatible worker
};

struct AuctionPick {
  uint32_t mine;            // lane r: the r-th best worker (kNone past the end)
  long long b1, b2;         // best and second-best value
  uint32_t w1;
  long long bound_v;        // best (value, worker) among the candidates that are not in the top 32
  uint32_t bound_w;
  long long drop_v;         // best (value, worker) no lane kept at all
  uint32_t drop_w;
};

__device__ __forceinline__ void auc_insert(long long (&cv)[4], uint32_t (&cw)[4], long long& dropped, uint32_t& dropped_w,
                                           long long v, uint32_t w) {
  if (auc_better(v, w, cv[3], cw[3])) {
    if (auc_better(cv[3], cw[3], dropped, dropped_w)) { dropped = cv[3]; dropped_w = cw[3]; }
    cv[3] = v; cw[3] = w;
#pragma unroll
    for (int j = 3; j > 0; --j)
      if (auc_better(cv[j], cw[j], cv[j - 1], cw[j - 1])) {
        const long long tv = cv[j - 1]; const uint32_t tw = cw[j - 1];
        cv[j - 1] = cv[j]; cw[j - 1] = cw[j]; cv[j] = tv; cw[j] = tw;
      }
  } else if (auc_better(v, w, dropped, dropped_w)) {
    dropped = v; dropped_w = w;
  }
}

// CTA-wide selection (all 256 threads, one item): the best 64 of the 1024 kept candidates, in (value desc, worker asc)
// order, by a bitonic network in shared memory that sorts blocks of 64 and then merges them keeping the better half
// (below) — instead of 2 x 32 dependent warp arg-max rounds.  A thread's 4 candidates arrive sorted, so
// the network is entered at run length 4 (odd threads store their run reversed: every 8 entries are then a bitonic
// sequence).  The result is valid in warp 0.
struct __align__(16) AuctionSort {
  long long v[kAucPool];
  uint32_t w[kAucPool];
  long long drop_v[kAucWarps];
  uint32_t drop_w[kAucWarps];
};
static_assert(kAucPool == 4 * kAucThreads, "one sorted run of 4 per thread");

// PACKED: (value, worker) as ONE sortable 64-bit key, (-value) << 24 | worker — ascending key = value descending,
// worker ascending; an empty slot is all ones.  Valid when every cost the auction can reach is below 2^40 and there are
// fewer than 2^24 workers (pm_auction_limits decides once per auction; ctl->packed): a compare-exchange is then two
// 64-bit loads, one compare and two stores instead of four loads, a two-word compare and four stores.
constexpr int kAucPackShift = 24;
__device__ __forceinline__ unsigned long long auc_pack(long long v, uint32_t w) {
  return (w == kNone || v <= kAucNeg) ? ~0ull : (((unsigned long long)(-v)) << kAucPackShift) | (unsigned long long)w;
}
__device__ __forceinline__ void auc_unpack(unsigned long long k, long long* v, uint32_t* w) {
  const bool none = k == ~0ull;
  *v = none ? kAucNeg : -(long long)(k >> kAucPackShift);
  *w = none ? kNone : (uint32_t)(k & ((1ull << kAucPackShift) - 1ull));
}

template <bool PACKED>
__device__ __forceinline__ AuctionPick auction_select_cta_t(const long long (&cv)[4], const uint32_t (&cw)[4], long long dropped,
                                                            uint32_t dropped_w, AuctionSort& ss) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  unsigned long long* const kk = reinterpret_cast<unsigned long long*>(ss.v);
  {
    const bool rev = (tid & 1u) != 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t at = tid * 4u + (rev ? 3u - (uint32_t)j : (uint32_t)j);
      if (PACKED) kk[at] = auc_pack(cv[j], cw[j]);
      else { ss.v[at] = cv[j]; ss.w[at] = cw[j]; }
    }
    long long dv;
    uint32_t dw;
    warp_argbest(dropped, dropped_w, &dv, &dw);
    if (lane == 0) { ss.drop_v[warp] = dv; ss.drop_w[warp] = dw; }
  }
  __syncthreads();
  auto cmpx = [&](uint32_t i, uint32_t j, bool desc) {   // compare-exchange of the entries i and i + j
    if (PACKED) {
      const unsigned long long ka = kk[i], kb = kk[i + j];
      if (desc ? kb < ka : ka < kb) { kk[i] = kb; kk[i + j] = ka; }
    } else {
      const long long va = ss.v[i], vb = ss.v[i + j];
      const uint32_t wa = ss.w[i], wb = ss.w[i + j];
      const bool swap = desc ? auc_better(vb, wb, va, wa) : auc_better(va, wa, vb, wb);
      if (swap) { ss.v[i] = vb; ss.w[i] = wb; ss.v[i + j] = va; ss.w[i + j] = wa; }
    }
  };
  // phase 1: the sixteen blocks of 64 entries, each sorted (even blocks descending, odd ones ascending).  A warp owns
  // the blocks `warp` and `8 + warp` (idx -> i maps 32 consecutive idx onto one aligned block of 64): warp barriers only.
#pragma unroll 1
  for (uint32_t k = 8; k <= 64u; k <<= 1) {
#pragma unroll 1
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (uint32_t r = 0; r < 2; ++r) {
        const uint32_t idx = tid + r * (uint32_t)kAucThreads;
        const uint32_t i = 2u * idx - (idx & (j - 1u));   // bit j of i is clear
        cmpx(i, j, (i & k) == 0u);
      }
      __syncwarp();
    }
  }
  // phase 2: only the best 64 are wanted, so a merge keeps the better half and drops the rest: of a descending block A
  // and an ascending block B the entry-wise better one goes to A (a bitonic sequence holding the 64 best of both),
  // six more stages sort it — descending or ascending by turns, so that the survivors pair up again.  8 + 4 + 2 + 1
  // merges by one warp each instead of the four full-width merge passes of a complete sort (half the instructions).
#pragma unroll 1
  for (uint32_t S = 64u, P = 8u; P > 0u; S <<= 1, P >>= 1) {
    __syncthreads();
    if (warp < P) {
      const uint32_t A = warp * 2u * S, B = A + S;
#pragma unroll
      for (uint32_t r = 0; r < 2; ++r) {
        const uint32_t i = lane + 32u * r;
        if (PACKED) {
          const unsigned long long kb = kk[B + i];
          if (kb < kk[A + i]) kk[A + i] = kb;
        } else {
          const long long vb = ss.v[B + i];
          const uint32_t wb = ss.w[B + i];
          if (auc_better(vb, wb, ss.v[A + i], ss.w[A + i])) { ss.v[A + i] = vb; ss.w[A + i] = wb; }
        }
      }
      __syncwarp();
      const bool desc = (warp & 1u) == 0u;
#pragma unroll 1
      for (uint32_t j = 32u; j > 0; j >>= 1) {
        cmpx(A + 2u * lane - (lane & (j - 1u)), j, desc);
        __syncwarp();
      }
    }
  }
  __syncthreads();
  AuctionPick r;
  long long mine_v, next_v;
  uint32_t mine_w, next_w;
  if (PACKED) {
    uint32_t w2;
    auc_unpack(kk[0], &r.b1, &r.w1);
    auc_unpack(kk[1], &r.b2, &w2);
    auc_unpack(kk[lane], &mine_v, &mine_w);
    auc_unpack(kk[32], &next_v, &next_w);
  } else {
    r.b1 = ss.v[0]; r.w1 = ss.w[0]; r.b2 = ss.v[1];
    mine_v = ss.v[lane]; mine_w = ss.w[lane];
    next_v = ss.v[32]; next_w = ss.w[32];
  }
  r.mine = (mine_v > kAucNeg) ? mine_w : kNone;
  warp_argbest(lane < (uint32_t)kAucWarps ? ss.drop_v[lane] : kAucNeg, lane < (uint32_t)kAucWarps ? ss.drop_w[lane] : kNone, &r.drop_v, &r.drop_w);
  const bool use_next = auc_better(next_v, next_w, r.drop_v, r.drop_w);
  r.bound_v = use_next ? next_v : r.drop_v;
  r.bound_w = use_next ? next_w : r.drop_w;
  __syncthreads();   // ss may be rewritten by the next select
  return r;
}
__device__ __forceinline__ AuctionPick auction_select_cta(const long long (&cv)[4], const uint32_t (&cw)[4], long long dropped,
                                                          uint32_t dropped_w, AuctionSort& ss, bool packed) {
  return packed ? auction_select_cta_t<true>(cv, cw, dropped, dropped_w, ss) : auction_select_cta_t<false>(cv, cw, dropped, dropped_w, ss);
}

// One scan item (a class, or a single ask in fallback mode) per CTA.
//
// Class mode keeps, next to the 32-entry cache the asks bid from, a POOL: every candidate the lanes
// held at the end of the class's last full scan (up to 1024 workers) and a bound on everything else.
// A rescan request first re-ranks the pool at the current prices (a few gathers per thread); only when
// the pool's best two no longer beat its bound does the class walk the price-sorted worker table again.
__device__ __forceinline__ void auction_scan_items(const AuctionParams& p, AuctionStage* stage, AuctionMerge& mg,
                                                   uint32_t& phase_bits, uint32_t base, const uint32_t* __restrict__ list,
                                                   uint32_t n_list, bool cls_mode, uint32_t part, uint32_t G) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t slot = base;
  const uint32_t in_item = threadIdx.x;           // this thread's pool slot (4 workers)
  const bool live = slot < n_list;
  const uint32_t item = live ? list[slot] : 0u;
  const uint32_t t = live ? (cls_mode ? p.class_rep[item] : item) : 0u;
  const DevAsk ask = p.ev.asks[t];
  const DevOpt opt0 = p.ev.opts[ask.n_opts ? ask.opt_off : 0u];
  const uint32_t cap = cls_mode ? 0xFFFFFFFFu : p.price_cap[t];
  const bool use_rep = p.rep_s != nullptr;
  const uint32_t floor_rep = use_rep ? p.min_rep[t] : 0u;
  // per lane: its 4 best (value, worker) in order, and the best (value, worker) it did not keep
  long long cv[4] = {kAucNeg, kAucNeg, kAucNeg, kAucNeg};
  uint32_t cw[4] = {kNone, kNone, kNone, kNone};
  long long dropped = kAucNeg;
  uint32_t dropped_w = kNone;
  const uint32_t W = p.ev.n_workers;
  const uint32_t n_all = (W + kAucStripe - 1) / kAucStripe;
  // one class per CTA: start where its compatible workers begin — the first stripe whose last key reaches skip_key
  const bool skipping = cls_mode && !(p.dbg & 64u);
  if (threadIdx.x == 0) { mg.cnt[0] = 0; mg.cnt[1] = 0; mg.cnt[2] = 0; mg.flag = 0; mg.first = kNone; mg.j0 = 0; }
  if (skipping && warp == 0) {
    const unsigned long long key = p.skip_key[item];
    uint32_t lo = 0, hi = n_all;   // every stripe below lo ends under the key; stripe hi (if any) does not
    while (lo < hi) {
      const uint32_t step = (hi - lo + 31u) / 32u;
      const uint32_t j = lo + lane * step;
      bool ge = true;
      if (j < hi) ge = p.csort_s[min((j + 1u) * (uint32_t)kAucStripe, W) - 1u] >= key;
      const uint32_t m = __ballot_sync(0xffffffffu, ge);
      const uint32_t f = m ? (uint32_t)__ffs((int)m) - 1u : 32u;   // ge is monotone in the lane
      if (f == 0u) { hi = lo; break; }
      const uint32_t nlo = lo + (f - 1u) * step + 1u;
      if (f < 32u && lo + f * step < hi) hi = lo + f * step;
      lo = nlo;
    }
    __syncwarp();
    if (lane == 0) mg.j0 = min(lo, hi);
  }
  __syncthreads();
  const uint32_t j0 = mg.j0;

  const bool scan = live;

  // a walk split over G CTAs: part `part` takes the stripes j0 + part, j0 + part + G, j0 + part + 2G, ...
  const uint32_t n_stripes = n_all > j0 + part ? (n_all - j0 - part + G - 1u) / G : 0u;
  auto issue = [&](uint32_t j) {
    AuctionStage& s = stage[j % kAucStages];
    const uint32_t w0 = (j0 + part + j * G) * kAucStripe;
    const uint32_t n = min((uint32_t)kAucStripe, W - w0);
    const uint32_t np = (n + 1u) & ~1u;   // bulk copies move multiples of 16 B; price_s[] and perm[] are padded
    const uint32_t nq = (n + 3u) & ~3u;
    mbar_expect_tx(&s.bar, n * 32u + np * 8u + nq * 4u + (use_rep ? nq * 4u : 0u));
    bulk_g2s(s.a, p.wa_s + w0, n * 16u, &s.bar);
    bulk_g2s(s.b, p.wb_s + w0, n * 16u, &s.bar);
    bulk_g2s(s.price, p.price_s + w0, np * 8u, &s.bar);
    bulk_g2s(s.perm, p.perm + w0, nq * 4u, &s.bar);
    if (use_rep) bulk_g2s(s.rep, p.rep_s + w0, nq * 4u, &s.bar);
  };
  auto wait_stage = [&](uint32_t j) {
    const uint32_t b = j % kAucStages;   // bit b of phase_bits = parity of the buffer's next completed phase
    mbar_wait(&stage[b].bar, (phase_bits >> b) & 1u);
    phase_bits ^= 1u << b;
  };
  uint32_t scanned = 0;
  uint32_t first_hit = kNone;    // first stripe in which this thread met a compatible worker
  uint32_t first_good = kNone;   // first stripe after which 33 candidates beat every unseen worker
  bool unseen = false;           // the walk stopped before the end of its stripes ...
  long long unseen_u = kAucNeg;  // ... where every remaining worker ranks at or below (unseen_u, unseen_w)
  uint32_t unseen_w = 0;
  if (threadIdx.x == 0)
    for (uint32_t k = 0; k < (uint32_t)(kAucStages - 1) && k < n_stripes; ++k) issue(k);
  for (uint32_t k = 0; k < n_stripes; ++k) {
    // stripe k + kAucStages - 1 goes into the buffer stripe k - 1 used: released by the barrier that ended it
    if (threadIdx.x == 0 && k + kAucStages - 1 < n_stripes) issue(k + kAucStages - 1);
    AuctionStage& s = stage[k % kAucStages];
    wait_stage(k);
    const uint32_t w0 = (j0 + part + k * G) * kAucStripe;
    const uint32_t n = min((uint32_t)kAucStripe, W - w0);
    if (scan) {
      scanned += n;
      for (uint32_t i = threadIdx.x; i < n; i += (uint32_t)kAucThreads) {
        const WorkerReg wr = make_worker(s.a[i], s.b[i]);
        if (wr.price <= cap && (!use_rep || s.rep[i] >= floor_rep) && auc_meets(ask, opt0, p.ev.opts, wr, p.ev.bits, p.ev.words)) {
          auc_insert(cv, cw, dropped, dropped_w, -((long long)wr.price * p.scale) - s.price[i], s.perm[i]);
          if (first_hit == kNone) first_hit = j0 + part + k * G;
        }
      }
    }
    // The table is sorted by the cost ask_price * S + price each worker had at the last sort; prices only rise, so
    // every later worker has value <= U = -(the stripe's last sort key).  Once 33 of the item's kept candidates beat the
    // unseen workers, at least one of them stays outside the 32-entry cache, so the bound (best candidate not cached) beats
    // every unseen worker and the walk may stop; a class walks a little further to fill its pool (not a part of a split
    // walk: it leaves its top 32 only, and those are final at this point); a single ask also stops once the unseen
    // workers cannot reach its outside option.
    const long long u = -(long long)p.csort_s[w0 + n - 1];
    const bool past_cap = !cls_mode && u < -(((long long)cap + 1) * p.scale);
    // ... and a later worker whose value still equals U has the same sort key as the stripe's last worker, hence a
    // larger index: the unseen workers rank at or below (U, last index + 1) in (value desc, worker asc) order, which
    // lets a walk stop inside a plateau of equal costs (where the whole bid-up mass of the market sits).
    const uint32_t il = s.perm[n - 1];
    auto beats = [&](long long v, uint32_t w) { return v > u || (v == u && w <= il); };
    uint32_t cnt = __popc(__ballot_sync(0xffffffffu, beats(cv[0], cw[0]))) + __popc(__ballot_sync(0xffffffffu, beats(cv[1], cw[1]))) +
                   __popc(__ballot_sync(0xffffffffu, beats(cv[2], cw[2]))) + __popc(__ballot_sync(0xffffffffu, beats(cv[3], cw[3])));
    if (lane == 0) atomicAdd(&mg.cnt[k % 3u], cnt);
    if (threadIdx.x == 0) mg.cnt[(k + 1u) % 3u] = 0;
    __syncthreads();   // (also: stripe k fully consumed, its buffer may be refilled)
    cnt = mg.cnt[k % 3u];
    if (cnt > (uint32_t)kAucCache && first_good == kNone) first_good = k;
    bool done = !scan || past_cap ||
                (first_good != kNone && (!cls_mode || G > 1u || cnt > p.pool_good || k - first_good >= p.pool_extra));
    if (p.dbg & 1u) done = false;
    if (done) {
      if (k + 1 < n_stripes) { unseen = true; unseen_u = u; unseen_w = il + 1u; }
      // the copies already in flight must land before the buffers are reused
      for (uint32_t j = k + 1; j < k + kAucStages && j < n_stripes; ++j) wait_stage(j);
      break;
    }
  }
  if (skipping) {   // (the selections below have CTA barriers: mg.first is complete when it is read)
    const uint32_t fh = __reduce_min_sync(0xffffffffu, first_hit);
    if (lane == 0 && fh != kNone) atomicMin(&mg.first, fh);
  }
  if (cls_mode && scan && G == 1u) {   // the new pool: what the lanes hold now
    uint4* pool = reinterpret_cast<uint4*>(p.pool) + (size_t)item * (kAucPool / 4);
    pool[in_item] = make_uint4(cw[0], cw[1], cw[2], cw[3]);
  }
  // the stage buffers are idle from here to the item's end (every copy issued was waited for): the sort scratch lives there
  AuctionSort& ss = *reinterpret_cast<AuctionSort*>(&stage[0]);
  static_assert(sizeof(AuctionSort) <= sizeof(AuctionStage), "sort scratch aliases one stage");
  const bool packed = p.ctl->packed != 0u && !(p.dbg & 128u);
  AuctionPick r = auction_select_cta(cv, cw, dropped, dropped_w, ss, packed);
  if (scan && threadIdx.x == 0) atomicAdd(&p.ctl->evals, (unsigned long long)scanned);
  long long pb_v = kAucNeg;   // outside the pool: what no lane kept, and the part of the table the walk did not reach
  uint32_t pb_w = kNone;
  if (G > 1u) {
    // Split walk: this part's top 32 become its slice of the pool, everything else it saw or skipped is summed up in
    // one bound; the part that arrives last re-ranks the G slices into the class cache.
    uint4* pool4 = reinterpret_cast<uint4*>(p.pool) + (size_t)item * (kAucPool / 4);
    if (warp == 0) {
      p.pool[(size_t)item * kAucPool + part * 32u + lane] = r.mine;
      if (lane == 0) {
        long long bv = r.bound_v;
        uint32_t bw = r.bound_w;
        if (unseen && auc_better(unseen_u, unseen_w, bv, bw)) { bv = unseen_u; bw = unseen_w; }
        p.split_bound_v[slot * 16u + part] = bv;
        p.split_bound_w[slot * 16u + part] = bw;
      }
    }
    {
      const uint32_t j = G * 8u + threadIdx.x;   // the slots no slice uses
      if (j < (uint32_t)(kAucPool / 4) && j % G == part) pool4[j] = make_uint4(kNone, kNone, kNone, kNone);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      if (skipping && mg.first != kNone) atomicMin(p.split_first + slot, mg.first);
      __threadfence();
      mg.flag = (atomicAdd(p.split_ticket + slot, 1u) == G - 1u) ? 1u : 0u;
    }
    __syncthreads();
    if (mg.flag == 0u) return;   // uniform; the CTA has no further item in split mode
    __threadfence();
    if (skipping && threadIdx.x == 0) {   // all parts are in: the earliest stripe any of them met a compatible worker in
      mg.first = __ldcg(p.split_first + slot);
      p.split_first[slot] = kNone;
    }
    long long bv = kAucNeg;
    uint32_t bw = kNone;
    if (warp == 0) {
      if (lane < G) { bv = __ldcg(p.split_bound_v + slot * 16u + lane); bw = __ldcg(p.split_bound_w + slot * 16u + lane); }
      warp_argbest(bv, bw, &pb_v, &pb_w);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { cv[j] = kAucNeg; cw[j] = kNone; }
    dropped = kAucNeg; dropped_w = kNone;
    {
      const uint4 e = __ldcg(pool4 + in_item);
      const uint32_t pw[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (pw[j] != kNone) auc_insert(cv, cw, dropped, dropped_w, -((long long)p.ev.wb[pw[j]].w * p.scale) - p.price[pw[j]], pw[j]);
    }
    if (in_item == 0) { dropped = pb_v; dropped_w = pb_w; }
    r = auction_select_cta(cv, cw, dropped, dropped_w, ss, packed);
    if (threadIdx.x == 0) p.split_ticket[slot] = 0u;
  } else if (scan && warp == 0) {
    pb_v = r.drop_v;
    pb_w = r.drop_w;
    if (unseen && auc_better(unseen_u, unseen_w, pb_v, pb_w)) { pb_v = unseen_u; pb_w = unseen_w; }
  }
  if (scan && warp == 0) {
    if (cls_mode) {
      p.cand[(size_t)item * kAucCache + lane] = r.mine;
      if (skipping && lane == 0) {
        // nobody compatible before stripe mg.first (none at all if the walk ran to the end without meeting one)
        const uint32_t fs = mg.first;
        const unsigned long long k_new = (fs == kNone) ? ~0ull : p.csort_s[(size_t)fs * kAucStripe];
        if (k_new > p.skip_key[item]) p.skip_key[item] = k_new;
      }
      if (lane == 0) {
        p.theta[item] = (r.bound_v == kAucNeg) ? kThetaComplete : r.bound_v;
        p.theta_w[item] = r.bound_w;
        p.pool_bound_v[item] = (pb_v == kAucNeg) ? kThetaComplete : pb_v;
        p.pool_bound_w[item] = pb_w;
        atomicAdd(&p.ctl->n_class_scans, 1ull);
      }
    } else if (lane == 0) {
      auction_place_bid(p, t, cap, r.b1, r.w1, r.b2);
      atomicAdd(&p.ctl->n_ask_scans, 1ull);
    }
  }
  __syncthreads();   // mg and the stage buffers are reused by the CTA's next item
}

// Rescan requests first re-rank the class pool at the current prices (a few gathers per thread); the classes
// whose pool cannot decide go on the walk list.
__global__ void __launch_bounds__(kAucThreads) pm_auction_refill(AuctionParams p) {
  __shared__ AuctionSort ss;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t n = p.ctl->n_cls;
  for (uint32_t slot = blockIdx.x; slot < n; slot += gridDim.x) {
    const uint32_t item = p.class_list[slot];
    const long long pool_bound = p.pool_bound_v[item];
    if (pool_bound == kThetaInvalid || (p.dbg & 8u)) {   // no pool yet (uniform across the CTA)
      if (threadIdx.x == 0) p.walk_list[atomicAdd(&p.ctl->n_walk, 1u)] = item;
      continue;
    }
    long long cv[4] = {kAucNeg, kAucNeg, kAucNeg, kAucNeg};
    uint32_t cw[4] = {kNone, kNone, kNone, kNone};
    long long dropped = kAucNeg;
    uint32_t dropped_w = kNone;
    const uint4 e = (reinterpret_cast<const uint4*>(p.pool) + (size_t)item * (kAucPool / 4))[threadIdx.x];
    const uint32_t pw[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (pw[j] != kNone) auc_insert(cv, cw, dropped, dropped_w, -((long long)p.ev.wb[pw[j]].w * p.scale) - p.price[pw[j]], pw[j]);
    if (threadIdx.x == 0) { dropped = pool_bound; dropped_w = p.pool_bound_w[item]; }   // everything outside the pool
    const AuctionPick r = auction_select_cta(cv, cw, dropped, dropped_w, ss, p.ctl->packed != 0u && !(p.dbg & 128u));
    if (warp == 0) {
      const bool ok = !(p.dbg & 16u) && (r.bound_v == kAucNeg || (r.b2 >= r.bound_v && auc_better(r.b1, r.w1, r.bound_v, r.bound_w)));
      if (ok) {
        p.cand[(size_t)item * kAucCache + lane] = r.mine;
        if (lane == 0) {
          p.theta[item] = (r.bound_v == kAucNeg) ? kThetaComplete : r.bound_v;
          p.theta_w[item] = r.bound_w;
          atomicAdd(&p.ctl->n_refills, 1ull);
        }
      } else if (lane == 0) {
        p.walk_list[atomicAdd(&p.ctl->n_walk, 1u)] = item;
      }
    }
  }
}

__global__ void __launch_bounds__(kAucThreads) pm_auction_scan(AuctionParams p, int cls_mode) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  AuctionStage* stage = reinterpret_cast<AuctionStage*>(smem_raw);            // [kAucStages]
  AuctionMerge& mg = *reinterpret_cast<AuctionMerge*>(smem_raw + kAucStages * sizeof(AuctionStage));
  const uint32_t n = cls_mode ? p.ctl->n_walk : p.ctl->n_fallback;
  const uint32_t* list = cls_mode ? p.walk_list : p.fallback;
  // few class walks (the long tail of an auction): each is split over G CTAs, so that its latency, which is what a
  // round then waits for, drops by G
  uint32_t G = 1u;
  if (cls_mode && n && 2u * n <= gridDim.x && !(p.dbg & 32u)) {
    G = 16u;
    while (n * G > gridDim.x) G >>= 1;
  }
  if (blockIdx.x >= n * G) return;
  if (threadIdx.x == 0)
    for (int b = 0; b < kAucStages; ++b) mbar_init(&stage[b].bar, 1);
  __syncthreads();
  uint32_t phase_bits = 0u;
  if (G > 1u) {
    auction_scan_items(p, stage, mg, phase_bits, blockIdx.x / G, list, n, true, blockIdx.x % G, G);
  } else {
    // items differ by two orders of magnitude in length (a broad class is done after a few stripes, a scarce one walks
    // to the end of the table): the CTAs draw them from a counter instead of taking every gridDim-th
    uint32_t* next = cls_mode ? &p.ctl->walk_taken : &p.ctl->fb_taken;
    for (;;) {
      if (threadIdx.x == 0) mg.flag = atomicAdd(next, 1u);
      __syncthreads();
      const uint32_t base = mg.flag;
      __syncthreads();   // (auction_scan_items resets mg.flag)
      if (base >= n) break;
      auction_scan_items(p, stage, mg, phase_bits, base, list, n, cls_mode != 0, 0u, 1u);
    }
  }
}

// One round for an ask from its class cache: 32 gathers instead of a scan.
// pass 0: the round's active asks; an undecided ask requests a rescan of its class and is retried.
// pass 1: the retried asks after the class scans; still undecided -> its own scan.
__global__ void __launch_bounds__(kAucThreads) pm_auction_bid_cached(AuctionParams p, int pass) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t n = pass ? p.ctl->n_retry : p.ctl->n_active;
  const uint32_t* list = pass ? p.retry : auc_active(p);
  const uint32_t stamp = p.ctl->rounds + 1u;
  for (uint32_t slot = blockIdx.x * kAucWarps + warp; slot < n; slot += gridDim.x * kAucWarps) {
    const uint32_t t = list[slot];
    const uint32_t c = p.class_of[t];
    const long long theta = p.theta[c];
    const uint32_t theta_w = p.theta_w[c];
    const uint32_t cap = p.price_cap[t];
    const long long outside = -(((long long)cap + 1) * p.scale);
    const uint32_t w = (theta != kThetaInvalid) ? p.cand[(size_t)c * kAucCache + lane] : kNone;
    long long v = kAucNeg;
    bool feas = false;
    if (w != kNone) {
      const uint32_t ap = p.ev.wb[w].w;
      v = -((long long)ap * p.scale) - p.price[w];
      feas = ap <= cap;
    }
    long long bf;
    uint32_t wf;
    const uint32_t lf = warp_argbest(feas ? v : kAucNeg, feas ? w : kNone, &bf, &wf);
    const bool has = wf != kNone;
    const long long bx = warp_max_i64((has && lane == lf) ? kAucNeg : v);   // best cached value other than w1
    if (lane == 0) {
      // every compatible worker outside the cache ranks at or below (theta, theta_w); kThetaComplete is
      // INT64_MIN (nothing outside), kThetaInvalid INT64_MAX (nothing known): both fall out of the compares
      int verdict;   // 0 withdraw, 1 bid, 2 ambiguous
      if (p.dbg & 2u) verdict = 2;
      else if (has && auc_better(bf, wf, theta, theta_w)) {
        if (bf < outside) verdict = 0;
        else verdict = (theta <= max(bx, outside)) ? 1 : 2;
      } else {
        const long long ub = has ? max(bf, theta) : theta;
        verdict = (ub < outside) ? 0 : 2;
      }
      if (verdict == 0) auction_withdraw(p, t);
      else if (verdict == 1) auction_commit(p, t, wf, bf, max(bx, outside));
      else {
        p.bid_w[t] = kNone;
        if (pass == 0) {
          if (atomicExch(p.class_req + c, stamp) != stamp) p.class_list[atomicAdd(&p.ctl->n_cls, 1u)] = c;
          p.retry[atomicAdd(&p.ctl->n_retry, 1u)] = t;
        } else {
          p.fallback[atomicAdd(&p.ctl->n_fallback, 1u)] = t;
        }
      }
    }
  }
}

// the claim: among the highest bidders of a worker the lowest ask index wins
__global__ void pm_auction_claim(AuctionParams p) {
  if (p.ctl->packed_claim) return;
  const uint32_t n = p.ctl->n_active;
  const uint32_t* __restrict__ active = auc_active(p);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t t = active[i], w = p.bid_w[t];
    if (w != kNone && p.bid_p[t] == p.bid_max[w]) atomicMin(p.winner + w, t);
  }
}

// Winners take their workers; the next round's active list is written on the way: an active ask that did not win and
// did not withdraw stays, and the ask a winner displaces comes back (it held a worker, so it was not active: no
// duplicates).  The block that finishes last advances the round — no pass over all asks, no separate launches.
__global__ void pm_auction_apply(AuctionParams p) {
  const uint32_t n = p.ctl->n_active;
  const uint32_t* __restrict__ active = auc_active(p);
  uint32_t* __restrict__ next = auc_next(p);
  const bool pc = p.ctl->packed_claim != 0u;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t t = active[i], w = p.bid_w[t];
    bool won = false;
    if (w != kNone) won = pc ? (kAucClaimMask - (uint32_t)((unsigned long long)p.bid_max[w] & kAucClaimMask)) == t && p.bid_max[w] >= 0 : p.winner[w] == t;
    if (won) {
      const uint32_t prev = p.owner[w];
      if (prev != kNone) {
        p.assigned[prev] = kNone;   // prev holds a worker, so it did not bid this round
        next[atomicAdd(&p.ctl->n_next, 1u)] = prev;
      }
      p.owner[w] = t;
      p.assigned[t] = w;
      p.price[w] = p.bid_p[t];
      p.price_s[p.pos_of[w]] = p.bid_p[t];
      p.bid_max[w] = kAucNeg;
      p.winner[w] = kNone;
    } else if (!p.withdrawn[t]) {
      next[atomicAdd(&p.ctl->n_next, 1u)] = t;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&p.ctl->ticket, 1u) == gridDim.x - 1u) {
      __threadfence();
      auc_advance(p.ctl, 0);
    }
  }
}

// the first active list of an eps phase: every ask that holds no worker and has not withdrawn
__global__ void pm_auction_compact(AuctionParams p, uint32_t n_asks) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  if (p.assigned[t] == kNone && !p.withdrawn[t]) auc_next(p)[atomicAdd(&p.ctl->n_next, 1u)] = t;
}
__global__ void pm_auction_advance(AuctionCtl* ctl, int first) { auc_advance(ctl, first); }

// Can (value, worker) be sorted as one 64-bit key?  A bid never exceeds (cap + 1) * S + eps (an ask pays at most its outside
// option), so every cost ask_price * S + price stays below (max ask_price + max cap + 2) * S + eps.
__global__ void pm_auction_limits(const uint4* __restrict__ wb, uint32_t n_workers, const uint32_t* __restrict__ cap, uint32_t n_asks,
                                  AuctionCtl* ctl) {
  uint32_t ma = 0, mc = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_workers; i += gridDim.x * blockDim.x) ma = max(ma, wb[i].w);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_asks; i += gridDim.x * blockDim.x) mc = max(mc, cap[i]);
  ma = __reduce_max_sync(0xffffffffu, ma);
  mc = __reduce_max_sync(0xffffffffu, mc);
  if ((threadIdx.x & 31u) == 0u) { atomicMax(&ctl->max_ask_price, ma); atomicMax(&ctl->max_cap, mc); }
}
__global__ void pm_auction_decide_packed(AuctionCtl* ctl, uint32_t n_workers, uint32_t n_asks, unsigned long long scale,
                                         unsigned long long eps_start, uint32_t dbg) {
  const unsigned long long lim = 1ull << 40;
  bool ok = n_workers < (1u << kAucPackShift) && scale < lim && eps_start < lim;
  if (ok) ok = ((unsigned long long)ctl->max_ask_price + ctl->max_cap + 2ull) < (lim - eps_start) / scale;
  ctl->packed = ok ? 1u : 0u;
  ctl->packed_claim = (ok && n_asks <= kAucClaimMask && !(dbg & 128u)) ? 1u : 0u;
}

// ---- ask classes -----------------------------------------------------------------------------
__device__ __forceinline__ uint64_t auc_mix(uint64_t h, uint32_t v) {
  h ^= v;
  h *= 0x9E3779B97F4A7C15ull;
  return h ^ (h >> 29);
}
__global__ void pm_auction_ask_hash(const DevAsk* __restrict__ asks, const DevOpt* __restrict__ opts, const uint32_t* __restrict__ min_rep,
                                    uint32_t n_asks, uint64_t* __restrict__ key, uint32_t* __restrict__ idx) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  const DevAsk a = asks[t];
  uint64_t h = 0x243F6A8885A308D3ull;
  if (min_rep) h = auc_mix(h, min_rep[t]);
  h = auc_mix(h, a.need); h = auc_mix(h, a.n_opts); h = auc_mix(h, a.cpu_cores); h = auc_mix(h, a.ram_mb); h = auc_mix(h, a.storage_gb);
  for (uint32_t o = 0; o < a.n_opts; ++o) {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(opts + a.opt_off + o);
#pragma unroll
    for (int j = 0; j < 8; ++j) h = auc_mix(h, q[j]);
  }
  key[t] = h;
  idx[t] = t;
}
__device__ __forceinline__ bool auc_same_ask(const DevAsk* asks, const DevOpt* opts, const uint32_t* min_rep, uint32_t x, uint32_t y) {
  const DevAsk a = asks[x], b = asks[y];
  if (min_rep && min_rep[x] != min_rep[y]) return false;
  if (a.need != b.need || a.n_opts != b.n_opts || a.cpu_cores != b.cpu_cores || a.ram_mb != b.ram_mb ||
      a.storage_gb != b.storage_gb)
    return false;
  for (uint32_t o = 0; o < a.n_opts; ++o) {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(opts + a.opt_off + o);
    const uint32_t* r = reinterpret_cast<const uint32_t*>(opts + b.opt_off + o);
    for (int j = 0; j < 8; ++j)
      if (q[j] != r[j]) return false;
  }
  return true;
}
// flag[i] = 1 where the i-th ask in hash order starts a new class (content compared, not the hash)
__global__ void pm_auction_class_flags(const DevAsk* __restrict__ asks, const DevOpt* __restrict__ opts, const uint32_t* __restrict__ min_rep,
                                       const uint32_t* __restrict__ sorted, uint32_t n_asks, uint32_t* __restrict__ flag) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_asks) return;
  flag[i] = (i == 0 || !auc_same_ask(asks, opts, min_rep, sorted[i - 1], sorted[i])) ? 1u : 0u;
}
__global__ void pm_auction_class_assign(const uint32_t* __restrict__ sorted, const uint32_t* __restrict__ flag,
                                        const uint32_t* __restrict__ incl, uint32_t n_asks, uint32_t* __restrict__ class_of,
                                        uint32_t* __restrict__ class_rep) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_asks) return;
  const uint32_t c = incl[i] - 1u;
  class_of[sorted[i]] = c;
  if (flag[i]) class_rep[c] = sorted[i];   // stable sort: the lowest ask of the run
}

// ---- price-sorted worker copy ------------------------------------------------------------------
__global__ void pm_auction_cost_keys(const uint4* __restrict__ wb, const long long* __restrict__ price, long long scale,
                                     uint32_t n, unsigned long long* __restrict__ key, uint32_t* __restrict__ idx) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  key[i] = (unsigned long long)((long long)wb[i].w * scale + price[i]);
  idx[i] = i;
}
__global__ void pm_auction_gather_sorted(const uint4* __restrict__ wa, const uint4* __restrict__ wb,
                                         const uint32_t* __restrict__ perm, const long long* __restrict__ price, uint32_t n,
                                         uint4* __restrict__ wa_s, uint4* __restrict__ wb_s, uint32_t* __restrict__ pos_of,
                                         long long* __restrict__ price_s, const uint32_t* __restrict__ rep, uint32_t* __restrict__ rep_s) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t w = perm[i];
  wa_s[i] = wa[w];
  wb_s[i] = wb[w];
  pos_of[w] = i;
  price_s[i] = price[w];
  if (rep_s) rep_s[i] = rep[w];
}

// ---- warm start (PM_AUCTION_WARM) --------------------------------------------------------------
// The stored state of the last pass (price, owner, assigned) is released where the changes since disturb it, then the
// rounds run from what is left.  Every reset worker, and every changed row, joins the list R (`raised`) once; all of
// them have price 0, so value(w) = -(ask_price[w] * S) on the whole list.
__device__ __forceinline__ void auc_release(const AuctionParams& p, uint32_t t) {
  const uint32_t w = atomicExch(p.assigned + t, kNone);   // an ask may be named twice (changed, and owner of a changed row)
  if (w == kNone) return;
  if (w < p.ev.n_workers) p.owner[w] = kNone;   // its price goes to 0 in pm_auction_warm_reset
  atomicAdd(&p.ctl->n_released, 1u);
}
// the initial release: every ask holding a worker at or past n_kept (a row a shrink cut off since the stored state),
// every owner of a changed row, every changed ask
__global__ void pm_auction_warm_seed(AuctionParams p, const uint32_t* __restrict__ rows, uint32_t n_rows,
                                     const uint32_t* __restrict__ changed_asks, uint32_t n_changed, uint32_t n_kept) {
  const uint32_t T = p.n_asks, n = T + n_rows + n_changed;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < T) {
      const uint32_t w = p.assigned[i];
      if (w != kNone && w >= n_kept) auc_release(p, i);
    } else if (i < T + n_rows) {
      const uint32_t t = p.owner[rows[i - T]];
      if (t != kNone) auc_release(p, t);
    } else {
      auc_release(p, changed_asks[i - T - n_rows]);
    }
  }
}
// every unowned worker with a positive price (the released ones, and what an eps-scaled pass left inflated) goes to 0
// and joins R; mark[w] says whether it did
__global__ void pm_auction_warm_reset(AuctionParams p, uint32_t* __restrict__ raised, uint32_t* __restrict__ mark) {
  const uint32_t W = p.ev.n_workers;
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < W; w += gridDim.x * blockDim.x) {
    uint32_t m = 0u;
    if (p.owner[w] == kNone && p.price[w] != 0) {
      p.price[w] = 0;
      raised[atomicAdd(&p.ctl->n_raised, 1u)] = w;
      m = 1u;
    }
    mark[w] = m;
  }
}
// ... and every changed row (the listed ones below n_kept, every row from n_kept on) that is not on R yet
__global__ void pm_auction_warm_rows(AuctionParams p, const uint32_t* __restrict__ rows, uint32_t n_rows, uint32_t n_kept,
                                     uint32_t* __restrict__ raised, uint32_t* __restrict__ mark) {
  const uint32_t W = p.ev.n_workers, n = n_rows + (W > n_kept ? W - n_kept : 0u);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t w = i < n_rows ? rows[i] : n_kept + (i - n_rows);   // distinct rows: no two threads share a mark
    if (!mark[w]) {
      mark[w] = 1u;
      raised[atomicAdd(&p.ctl->n_raised, 1u)] = w;
    }
  }
}
// Does class c accept worker w (compatibility and the reputation floor, both part of the class; the cap is per ask)?
// rep: the `reputation` column in worker order, or null when no floor was given.
__device__ __forceinline__ bool auc_class_accepts(const AuctionParams& p, uint32_t c, const WorkerReg& wr, uint32_t w,
                                                  const uint32_t* __restrict__ rep) {
  const uint32_t t = p.class_rep[c];
  const DevAsk ask = p.ev.asks[t];
  const DevOpt opt0 = p.ev.opts[ask.n_opts ? ask.opt_off : 0u];
  return (!rep || rep[w] >= p.min_rep[t]) && auc_meets(ask, opt0, p.ev.opts, wr, p.ev.bits, p.ev.words);
}
// Closure, step 1: C x |R_new| predicate evaluations.  cmin[c] = the lowest ask_price among the newly raised workers
// class c accepts (reputation floor included): with every raised price at 0 that worker is, for each ask of the class
// whose cap reaches it, its best raised worker.  One CTA per (class, 256 raised workers).
__global__ void __launch_bounds__(256) pm_auction_release_classes(AuctionParams p, const uint32_t* __restrict__ raised, uint32_t lo,
                                                                  uint32_t hi, const uint32_t* __restrict__ rep,
                                                                  uint32_t* __restrict__ cmin) {
  const uint32_t c = blockIdx.x;
  const uint32_t i = lo + blockIdx.y * 256u + threadIdx.x;
  uint32_t ap = 0xFFFFFFFFu;
  if (i < hi) {
    const uint32_t w = raised[i];
    const WorkerReg wr = make_worker(p.ev.wa[w], p.ev.wb[w]);
    if (auc_class_accepts(p, c, wr, w, rep)) ap = wr.price;
  }
  ap = __reduce_min_sync(0xffffffffu, ap);
  if ((threadIdx.x & 31u) == 0u && ap != 0xFFFFFFFFu) atomicMin(cmin + c, ap);
}
// Closure, step 2: an ask still holding w_t is released when its best affordable raised worker beats w_t by more than
// eps (its eps-complementary slackness no longer holds); w_t goes to price 0 and joins R for the next iteration.
__global__ void pm_auction_release_asks(AuctionParams p, const uint32_t* __restrict__ cmin, uint32_t* __restrict__ raised) {
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < p.n_asks; t += gridDim.x * blockDim.x) {
    const uint32_t w = p.assigned[t];
    if (w == kNone) continue;
    const uint32_t m = cmin[p.class_of[t]];
    if (m == 0xFFFFFFFFu || m > p.price_cap[t]) continue;
    const long long v_raised = -((long long)m * p.scale);
    const long long v_held = -((long long)p.ev.wb[w].w * p.scale) - p.price[w];
    if (v_raised - p.eps > v_held) {
      p.assigned[t] = kNone;
      p.owner[w] = kNone;
      p.price[w] = 0;
      raised[atomicAdd(&p.ctl->n_raised, 1u)] = w;
      atomicAdd(&p.ctl->n_released, 1u);
    }
  }
}

// ---- reverse rounds (PM_AUCTION_REVERSE) -----------------------------------------------------------
// Every eps phase ends with them: the unowned workers whose price is still positive (what a coarser phase left
// stranded) bid for asks, synchronously, until none is left.  With a(w) = -(ask_price[w] * S) and the ask's profit
// pi(t) = a(w_t) - price[w_t] when it holds w_t, else outside(t): a bidder w takes the gains g(t) = a(w) - pi(t) over
// its feasible asks, best beta on t* (lowest ask among equals), second value omega of the multiset; beta <= eps (or no
// feasible ask) sends its price to 0, else it offers itself to t* at p' = max(0, omega - eps).  Each ask takes the
// offer of highest profit a(w) - p' (ties: lowest worker); its previous worker becomes unowned at its price.
// All of a round reads the state of its start: the collect step writes the asks' profits before anyone bids.
constexpr uint32_t kRevChunk = 8192;   // classes per chunk of the bid's class mask (1 KB of shared memory)
constexpr unsigned long long kRevPackLim = 1ull << 40;   // packed offer: (2^40 - 1 - cost) << 24 | (2^24 - 1 - worker)

struct AuctionRev {
  uint32_t* bidders;           // [W] this round's bidders (ctl->n_bid of them)
  uint32_t* offer_t;           // [W] per bidder: the ask it offers itself to, or kNone (its price went to 0)
  long long* offer_p;          // [W] ... the price it offers at
  long long* best;             // [T] per ask: the best packed offer key (0: none), or unpacked the best profit
  uint32_t* win;               // [T] unpacked: the lowest worker among the ask's best offers
  long long* pi_s;             // [T] profit of the ask at sorted position i, at the start of the round
  const uint32_t* cap_s;       // [T] cap of the ask at sorted position i
  const uint32_t* sorted;      // [T] asks in class order (the class build's sort): each class is one run
  const uint32_t* cls_s;       // [T] class of sorted position i, plus one (the class build's inclusive scan)
  const uint32_t* cstart;      // [C + 1] first sorted position of each class
  const uint32_t* rep;         // [W] `reputation` in worker order, or null (no floor given)
  uint32_t n_classes;
};

__device__ __forceinline__ bool auc_rev_packed(const AuctionParams& p) { return p.ctl->packed != 0u && !(p.dbg & 128u); }

// once per pass: the run of each class in sorted order, and the caps in that order
__global__ void pm_auction_rev_classes(const uint32_t* __restrict__ sorted, const uint32_t* __restrict__ incl,
                                       const uint32_t* __restrict__ cap, uint32_t n_asks, uint32_t n_classes,
                                       uint32_t* __restrict__ cstart, uint32_t* __restrict__ cap_s) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_asks) return;
  cap_s[i] = cap[sorted[i]];
  if (i == 0 || incl[i] != incl[i - 1]) cstart[incl[i] - 1u] = i;
  if (i == n_asks - 1u) cstart[n_classes] = n_asks;
}

// Start of a round: the bidder list, every ask's profit (in sorted order), no offers yet.
__global__ void pm_auction_rev_collect(AuctionParams p, AuctionRev r) {
  const uint32_t W = p.ev.n_workers, T = p.n_asks, n = max(W, T);
  const bool pk = auc_rev_packed(p);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < W && p.owner[i] == kNone && p.price[i] > 0) r.bidders[atomicAdd(&p.ctl->n_bid, 1u)] = i;
    if (i < T) {
      const uint32_t wt = p.assigned[r.sorted[i]];
      r.pi_s[i] = wt != kNone ? -((long long)p.ev.wb[wt].w * p.scale) - p.price[wt] : -(((long long)r.cap_s[i] + 1) * p.scale);
      r.best[i] = pk ? 0ll : kAucNeg;   // (indexed by ask: i runs over all of them)
      r.win[i] = kNone;
    }
  }
}

// (best gain, its ask, second value) of two parts of the multiset
__device__ __forceinline__ void auc_rev_merge(long long& g1, uint32_t& t1, long long& g2, long long o1, uint32_t ot1, long long o2) {
  if (o1 > g1 || (o1 == g1 && ot1 < t1)) { g2 = max(g1, o2); g1 = o1; t1 = ot1; }
  else g2 = max(g2, o1);
}

struct AuctionRevSmem {   // shared memory of one bidder's gain walk
  uint32_t mask[kRevChunk / 32];
  long long red_g1[kAucWarps], red_g2[kAucWarps];
  uint32_t red_t1[kAucWarps];
};

// The gains of worker w (all threads of the CTA): C predicate evaluations against the class representatives give a class
// mask in shared memory (kRevChunk classes at a time), then a walk over the asks of those classes in sorted order —
// class bit, cap, gain — keeps the best two.  HELD_ONLY (the warm repair's raise) also skips every ask that holds no
// worker.  (g1, t1, g2) = (beta, t*, omega) is valid on thread 0 (t1 = kNone: no ask counted); the caller puts a barrier
// between two calls (red_* are rewritten).
template <bool HELD_ONLY>
__device__ __forceinline__ void auc_rev_gains(const AuctionParams& p, const AuctionRev& r, AuctionRevSmem& sm, uint32_t w,
                                              const WorkerReg& wr, long long a, long long& g1, uint32_t& t1, long long& g2) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t C = r.n_classes;
  g1 = kAucNeg; g2 = kAucNeg; t1 = kNone;
  for (uint32_t c0 = 0; c0 < C; c0 += kRevChunk) {
    const uint32_t nc = min(C - c0, kRevChunk);
    const uint32_t kmax = (nc + kAucThreads - 1u) / kAucThreads * kAucThreads;   // the same trip count on every thread
    for (uint32_t k = threadIdx.x; k < kmax; k += kAucThreads) {
      const bool ok = k < nc && auc_class_accepts(p, c0 + k, wr, w, r.rep);
      const uint32_t m = __ballot_sync(0xffffffffu, ok);   // warp-aligned k: one mask word per warp
      if (lane == 0) sm.mask[k >> 5] = m;
    }
    __syncthreads();
    // four positions per thread and step, their class loads issued together (the walk is latency-bound)
    const uint32_t i1 = r.cstart[c0 + nc];
    for (uint32_t i = r.cstart[c0] + threadIdx.x; i < i1; i += 4u * kAucThreads) {
      uint32_t cs[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t j = i + (uint32_t)u * kAucThreads;
        cs[u] = j < i1 ? r.cls_s[j] - 1u - c0 : kNone;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t j = i + (uint32_t)u * kAucThreads, c = cs[u];
        if (c != kNone && ((sm.mask[c >> 5] >> (c & 31u)) & 1u) && r.cap_s[j] >= wr.price) {
          const uint32_t t = r.sorted[j];
          if (HELD_ONLY && p.assigned[t] == kNone) continue;   // an ask that holds no worker bids in the rounds instead
          const long long g = a - r.pi_s[j];
          if (g > g1 || (g == g1 && t < t1)) { g2 = g1; g1 = g; t1 = t; }
          else g2 = max(g2, g);
        }
      }
    }
    __syncthreads();   // the mask is rewritten by the next chunk
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const long long o1 = __shfl_xor_sync(0xffffffffu, g1, off), o2 = __shfl_xor_sync(0xffffffffu, g2, off);
    const uint32_t ot = __shfl_xor_sync(0xffffffffu, t1, off);
    auc_rev_merge(g1, t1, g2, o1, ot, o2);
  }
  if (lane == 0) { sm.red_g1[warp] = g1; sm.red_g2[warp] = g2; sm.red_t1[warp] = t1; }
  __syncthreads();
  if (threadIdx.x == 0)
    for (uint32_t k = 1; k < (uint32_t)kAucWarps; ++k) auc_rev_merge(g1, t1, g2, sm.red_g1[k], sm.red_t1[k], sm.red_g2[k]);
}

// One CTA per bidder: its gains, then thread 0 drops the price to 0 or posts the offer.
__global__ void __launch_bounds__(kAucThreads, 4) pm_auction_rev_bid(AuctionParams p, AuctionRev r) {
  __shared__ AuctionRevSmem sm;
  const uint32_t n = p.ctl->n_bid;
  const bool pk = auc_rev_packed(p);
  for (uint32_t slot = blockIdx.x; slot < n; slot += gridDim.x) {
    const uint32_t w = r.bidders[slot];
    const WorkerReg wr = make_worker(p.ev.wa[w], p.ev.wb[w]);
    const long long a = -((long long)wr.price * p.scale);
    long long g1, g2;
    uint32_t t1;
    auc_rev_gains<false>(p, r, sm, w, wr, a, g1, t1, g2);
    if (threadIdx.x == 0) {
      if (t1 == kNone || g1 <= p.eps) {   // nothing worth offering: the price goes to 0, the worker stays unowned
        p.price[w] = 0;
        p.price_s[p.pos_of[w]] = 0;
        r.offer_t[slot] = kNone;
        p.ctl->rev_lowered = 1u;
      } else {
        const long long pn = max(0ll, g2 - p.eps);   // no second value: kAucNeg, so 0
        const long long profit = a - pn;
        r.offer_t[slot] = t1;
        r.offer_p[slot] = pn;
        // packed: the highest profit, among equal ones the lowest worker, is the largest key (every cost < 2^40, W < 2^24)
        if (pk) atomicMax(reinterpret_cast<unsigned long long*>(r.best) + t1,
                          ((kRevPackLim - 1ull - (unsigned long long)(-profit)) << kAucPackShift) | (unsigned long long)(((1u << kAucPackShift) - 1u) - w));
        else atomicMax(r.best + t1, profit);
      }
    }
    __syncthreads();   // red_* are reused by the CTA's next bidder
  }
}

// Warm repair (PM_AUCTION_WARM | PM_AUCTION_REPAIR), step 2: one CTA per raised row w (the changed rows, all unowned
// after the release), the bid's gains over the asks that still hold a worker, read from pi_s as pm_auction_rev_collect
// wrote it after the release; price[w] = max(0, beta - eps), or 0 when no held ask is feasible for w.  No offer: the
// forward rounds and the reverse stage take it from here.  A raised row holds no ask, so it changes no profit any other
// raised row reads: the result does not depend on the order.
__global__ void __launch_bounds__(kAucThreads, 4) pm_auction_repair_raise(AuctionParams p, AuctionRev r,
                                                                           const uint32_t* __restrict__ raised) {
  __shared__ AuctionRevSmem sm;
  const uint32_t n = p.ctl->n_raised;
  for (uint32_t slot = blockIdx.x; slot < n; slot += gridDim.x) {
    const uint32_t w = raised[slot];
    const WorkerReg wr = make_worker(p.ev.wa[w], p.ev.wb[w]);
    const long long a = -((long long)wr.price * p.scale);
    long long g1, g2;
    uint32_t t1;
    auc_rev_gains<true>(p, r, sm, w, wr, a, g1, t1, g2);
    if (threadIdx.x == 0) p.price[w] = t1 == kNone ? 0ll : max(0ll, g1 - p.eps);
    __syncthreads();   // red_* are reused by the CTA's next row
  }
}

// unpacked offers: among the best offers on an ask the lowest worker wins
__global__ void pm_auction_rev_claim(AuctionParams p, AuctionRev r) {
  if (auc_rev_packed(p)) return;
  const uint32_t n = p.ctl->n_bid;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t t = r.offer_t[i];
    if (t == kNone) continue;
    const uint32_t w = r.bidders[i];
    if (-((long long)p.ev.wb[w].w * p.scale) - r.offer_p[i] == r.best[t]) atomicMin(r.win + t, w);
  }
}

// The winners take their asks; an ask's previous worker becomes unowned at its price (it bids next round if that is
// positive).  Asks only gain or trade up here: nobody is pushed back into the forward rounds.
__global__ void pm_auction_rev_apply(AuctionParams p, AuctionRev r) {
  const uint32_t n = p.ctl->n_bid;
  const bool pk = auc_rev_packed(p);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t t = r.offer_t[i];
    if (t == kNone) continue;
    const uint32_t w = r.bidders[i];
    const bool won = pk ? (uint32_t)((1u << kAucPackShift) - 1u) - (uint32_t)((unsigned long long)r.best[t] & ((1ull << kAucPackShift) - 1ull)) == w
                        : r.win[t] == w;
    if (!won) continue;
    const uint32_t prev = p.assigned[t];
    if (prev != kNone) p.owner[prev] = kNone;
    p.owner[w] = t;
    p.assigned[t] = w;
    p.withdrawn[t] = 0u;
    const long long pn = r.offer_p[i];
    if (pn < p.price[w]) p.ctl->rev_lowered = 1u;
    p.price[w] = pn;
    p.price_s[p.pos_of[w]] = pn;
  }
}
__global__ void pm_auction_rev_advance(AuctionCtl* ctl) {
  const uint32_t n = ctl->n_bid;
  if (n) { ++ctl->rev_rounds; ctl->rev_bids += n; }
  ctl->rev_last = n;
  ctl->n_bid = 0;
}

// result in the engine's group form: one solo group per assigned ask, in ask order
__global__ void pm_auction_flags(const uint32_t* __restrict__ assigned, uint32_t n_asks, uint32_t* __restrict__ flag) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_asks) flag[t] = assigned[t] != kNone ? 1u : 0u;
  if (t == n_asks) flag[t] = 0u;
}
__global__ void pm_auction_emit(const uint32_t* __restrict__ assigned, const uint32_t* __restrict__ gidx,
                                const uint4* __restrict__ wb, uint32_t n_asks, uint32_t* __restrict__ worker_group,
                                uint32_t* __restrict__ worker_ask, uint32_t* __restrict__ group_ask,
                                uint32_t* __restrict__ group_off, uint32_t* __restrict__ members,
                                long long* __restrict__ ask_best, uint32_t* __restrict__ ask_count) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  const uint32_t w = assigned[t];
  if (w == kNone) { ask_best[t] = kInf; ask_count[t] = 0; return; }
  const uint32_t g = gidx[t];
  worker_group[w] = g;
  worker_ask[w] = t;
  group_ask[g] = t;
  group_off[g] = g;
  members[g] = w;
  ask_best[t] = ((long long)wb[w].w << 32) | (long long)w;
  ask_count[t] = 1;
}

// ---- ask demands (pm_set_ask_demand) -------------------------------------------------------------------
// Ask t with demand d[t] is d[t] bidders, its SLOTS off[t] .. off[t + 1] - 1 (off: the exclusive scan of the demands):
// the ask's row repeated d[t] times at consecutive priorities.  The auction runs on the slots as on any ask table, over
// per-slot copies of the row, the cap and the floor; only the result is folded back per ask.
__device__ __forceinline__ uint32_t auc_ask_of_slot(const uint32_t* __restrict__ off, uint32_t n_asks, uint32_t s) {
  uint32_t lo = 0, hi = n_asks;   // off[lo] <= s < off[hi]; every demand is >= 1, so off is strictly increasing
  while (hi - lo > 1u) {
    const uint32_t mid = (lo + hi) >> 1;
    if (off[mid] <= s) lo = mid;
    else hi = mid;
  }
  return lo;
}
// the slot table: each slot's ask, and its copies of the ask's converted row, cap and floor (floor: null without one)
__global__ void pm_auction_slot_table(const uint32_t* __restrict__ off, uint32_t n_asks, uint32_t n_slots, const DevAsk* __restrict__ asks,
                                      const uint32_t* __restrict__ cap, const uint32_t* __restrict__ floor, uint32_t* __restrict__ slot_ask,
                                      DevAsk* __restrict__ slot_row, uint32_t* __restrict__ slot_cap, uint32_t* __restrict__ slot_floor) {
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_slots; s += gridDim.x * blockDim.x) {
    const uint32_t t = auc_ask_of_slot(off, n_asks, s);
    slot_ask[s] = t;
    slot_row[s] = asks[t];
    slot_cap[s] = cap[t];
    if (floor) slot_floor[s] = floor[t];
  }
}
// A demand change or an ask-table splice under a stored state: old slot k of ask t keeps its hold as slot k of ask
// map[t] (map null: t) while that ask is kept and k < its new demand; otherwise the slot is gone and its worker becomes
// unowned at its stored price, counted in `count` when it is a kept row.  Offsets null: one slot per ask (no demands).
// n_asks: the old table's.  new_assigned is all PM_NONE before: added and inserted slots hold nothing.
__global__ void pm_auction_slot_remap(const uint32_t* __restrict__ old_off, const uint32_t* __restrict__ new_off,
                                      const uint32_t* __restrict__ map, uint32_t n_asks, uint32_t n_old,
                                      const uint32_t* __restrict__ old_assigned, uint32_t* __restrict__ new_assigned,
                                      uint32_t* __restrict__ owner, uint32_t n_rows, uint32_t* __restrict__ count) {
  uint32_t freed = 0;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_old; s += gridDim.x * blockDim.x) {
    const uint32_t t = old_off ? auc_ask_of_slot(old_off, n_asks, s) : s, k = old_off ? s - old_off[t] : 0u;
    const uint32_t nt = map ? map[t] : t;
    const uint32_t w = old_assigned[s];
    if (nt != kNone && k < (new_off ? new_off[nt + 1] - new_off[nt] : 1u)) {
      const uint32_t ns = (new_off ? new_off[nt] : nt) + k;
      new_assigned[ns] = w;
      if (w < n_rows) owner[w] = ns;
    } else if (w < n_rows) {
      owner[w] = kNone;
      ++freed;
    }
  }
  if (freed) atomicAdd(count, freed);
}
// Grouped result (demands set): held[s] for the slots' exclusive scan `spos` (members in slot order) ...
__global__ void pm_auction_slot_flags(const uint32_t* __restrict__ assigned, uint32_t n_slots, uint32_t* __restrict__ flag) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n_slots) flag[s] = assigned[s] != kNone ? 1u : 0u;
  if (s == n_slots) flag[s] = 0u;
}
// ... per ask over its slot segment: the held count, ask_best, and whether it forms a group (for the groups' scan) ...
__global__ void pm_auction_group_counts(const uint32_t* __restrict__ off, const uint32_t* __restrict__ spos,
                                        const uint32_t* __restrict__ assigned, const uint4* __restrict__ wb, uint32_t n_asks,
                                        uint32_t* __restrict__ flag, long long* __restrict__ ask_best, uint32_t* __restrict__ ask_count) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == n_asks) flag[t] = 0u;
  if (t >= n_asks) return;
  const uint32_t s0 = off[t], s1 = off[t + 1], n = spos[s1] - spos[s0];
  long long best = kInf;
  for (uint32_t s = s0; s < s1 && n; ++s) {
    const uint32_t w = assigned[s];
    if (w != kNone) best = min(best, ((long long)wb[w].w << 32) | (long long)w);
  }
  flag[t] = n ? 1u : 0u;
  ask_best[t] = best;
  ask_count[t] = n;
}
// ... and one group per ask holding a worker, in ask order; its members in slot order (the engine sorts each group's
// members by worker index afterwards)
__global__ void pm_auction_group_emit(const uint32_t* __restrict__ off, const uint32_t* __restrict__ spos,
                                      const uint32_t* __restrict__ gidx, const uint32_t* __restrict__ assigned, uint32_t n_asks,
                                      uint32_t* __restrict__ worker_group, uint32_t* __restrict__ worker_ask,
                                      uint32_t* __restrict__ group_ask, uint32_t* __restrict__ group_off, uint32_t* __restrict__ members) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_asks) return;
  const uint32_t s0 = off[t], s1 = off[t + 1];
  uint32_t j = spos[s0];
  if (spos[s1] == j) return;
  const uint32_t g = gidx[t];
  group_ask[g] = t;
  group_off[g] = j;
  for (uint32_t s = s0; s < s1; ++s) {
    const uint32_t w = assigned[s];
    if (w == kNone) continue;
    members[j++] = w;
    worker_group[w] = g;
    worker_ask[w] = t;
  }
}

}  // namespace pm
