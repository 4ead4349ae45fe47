"""An exact reference for the benchmark's full sizes, built on the CPU oracle's predicate alone.

Whether ask t accepts worker w depends on w only through its predicate fields (flags without HAS_LOC, gpu count, gpu
memory, the acceptance class of its model id, cores, ram, storage) and on t only through its row and its option rows.
Price and worker index only order the feasible workers.  So the workers collapse into *profiles* and the asks into
*distinct rows*; orc.soa_eval_matrix evaluates one representative of each profile against each distinct row, and the
results are expanded back.  Nothing is sampled and nothing is approximated: every array pm_fetch_result returns for a
solo table (min = max = 1, or max = 0), the per-shard arrays of pm_match_local, and every field of
pm_auction_certificate follow exactly.

The model clause reads only bits[pattern][model], so model ids with the same column of the acceptance table over all
patterns are interchangeable; each id maps to the first id of its column, and the profile count stays small however
many model strings the catalogue has.  Non-candidate workers keep their own profiles: the oracle reports them
infeasible everywhere, so they need no special case here.

Everything here calls oracle.pm_oracle and numpy only; nothing reads the engine.
"""
from __future__ import annotations

import os

import numpy as np

from oracle import pm_oracle as orc
from protocol_b200 import abi

NONE = abi.PM_NONE
INF = abi.PM_COST_INF
CHUNK_BYTES = 256 << 20   # the int64 cost block one soa_eval_matrix call fills, and the int64 scratch of the reductions


def threads() -> int:
    return max(1, len(os.sched_getaffinity(0)))


def _unique_rows(m: np.ndarray):
    """(first index, inverse) of the distinct rows of a 2-D uint8 matrix, distinct rows in sorted order."""
    m = np.ascontiguousarray(m)
    v = m.view(np.dtype((np.void, m.shape[1]))).ravel() if m.shape[1] else np.zeros(len(m), dtype="V1")
    _, first, inv = np.unique(v, return_index=True, return_inverse=True)
    return first.astype(np.int64), inv.reshape(-1).astype(np.int64)


def model_classes(bits, n_patterns: int, n_models: int, words: int) -> np.ndarray:
    """int64[n_models]: for each model id, the first id whose acceptance column over every pattern is the same."""
    if n_models == 0:
        return np.zeros(0, dtype=np.int64)
    b = np.asarray(bits, dtype=np.uint32)[:n_patterns * words].reshape(n_patterns, words)
    m = np.arange(n_models)
    col = ((b[:, m >> 5] >> (m & 31).astype(np.uint32)) & 1).astype(bool)       # [pattern, model]
    first, inv = _unique_rows(np.packbits(col.T, axis=1))
    return first[inv]


def worker_profiles(wa, wb, classes, extra=None):
    """(profile of every worker int64[W], one representative row index per profile int64[P]).  extra: further
    uint32 columns that join the key (the reputation column)."""
    W = len(wa)
    mid = wa["model_id"].astype(np.int64)
    known = mid < len(classes)
    # an id outside the table keeps its own value, offset past every class id so that the two never meet
    model = np.where(known, classes[np.minimum(mid, len(classes) - 1)] if len(classes) else 0, len(classes) + mid)
    cols = [wa["flags"] & np.uint32(~abi.PM_W_HAS_LOC & 0xFFFFFFFF), wa["gpu_count"], wa["gpu_mem_mb"], model,
            wb["cpu_cores"], wb["ram_mb"], wb["storage_gb"]]
    if extra is not None:
        cols.append(np.asarray(extra, dtype=np.uint32))
    key = np.stack([np.asarray(c).astype(np.uint64) for c in cols], axis=1)
    first, inv = _unique_rows(key.view(np.uint8).reshape(W, 8 * len(cols)))
    return inv, first


def ask_rows(asks, opts, max_at_least_one=False):
    """(distinct row of every ask int64[T], the distinct rows ASK[U], their option rows GPU_OPT).  The key is the row
    without opt_off, plus the bytes of its option rows."""
    asks = np.ascontiguousarray(asks, dtype=abi.ASK)
    opts = np.ascontiguousarray(opts, dtype=abi.GPU_OPT)
    T = len(asks)
    k = asks.copy()
    k["opt_off"] = 0
    if max_at_least_one:
        k["max_group_size"] = np.maximum(k["max_group_size"], 1)
    K = int(asks["n_opts"].max()) if T else 0
    key = np.zeros((T, 32 + 32 * K), dtype=np.uint8)
    key[:, :32] = k.view(np.uint8).reshape(T, 32)
    ov = opts.view(np.uint8).reshape(-1, 32)
    for j in range(K):
        has = asks["n_opts"] > j
        key[has, 32 + 32 * j:64 + 32 * j] = ov[asks["opt_off"][has].astype(np.int64) + j]
    first, inv = _unique_rows(key)
    rep = k[first].copy()
    n = rep["n_opts"].astype(np.int64)
    off = np.zeros(len(rep) + 1, dtype=np.int64)
    np.cumsum(n, out=off[1:])
    rep["opt_off"] = off[:-1]
    src = np.concatenate([np.arange(int(asks["opt_off"][f]), int(asks["opt_off"][f]) + int(c)) for f, c in zip(first, n)]) \
        if off[-1] else np.zeros(0, dtype=np.int64)
    return inv, rep, opts[src.astype(np.int64)].copy() if len(src) else np.zeros(0, dtype=abi.GPU_OPT)


def feasibility(rep_wa, rep_wb, rep_asks, rep_opts, bits, words) -> np.ndarray:
    """bool[U, P]: candidate(profile) and compatible(row, profile), the oracle's soa_eval_matrix in bounded blocks."""
    U, P = len(rep_asks), len(rep_wa)
    F = np.zeros((U, P), dtype=bool)
    if U == 0 or P == 0:
        return F
    wb = rep_wb.copy()
    wb["ext_ask_price"] = 0
    step = max(1, CHUNK_BYTES // (8 * P))
    for u0 in range(0, U, step):
        u1 = min(U, u0 + step)
        ev = orc.soa_eval_matrix(rep_wa, wb, rep_asks, rep_opts, bits, words, u0, u1, 0, P, threads=threads(),
                                 want_cost=True, want_rows=False, want_cols=False)
        F[u0:u1] = ev["cost"] != INF
    return F


def _row_chunks(U, P):
    step = max(1, CHUNK_BYTES // (8 * max(P, 1)))
    return [(u0, min(U, u0 + step)) for u0 in range(0, U, step)]


def packed_cost(wb, w0=0):
    """(ext_ask_price << 32) | w as the oracle packs it, signed."""
    w = np.arange(w0, w0 + len(wb), dtype=np.uint64)
    return ((wb["ext_ask_price"].astype(np.uint64) << np.uint64(32)) | w).view(np.int64)


class Reference:
    """The collapsed first-fit reference of one table.  enabled (bool[T], optional): a disabled ask is absent."""

    def __init__(self, wa, wb, asks, opts, bits, n_patterns, n_models, words, enabled=None):
        mn, mx = asks["min_group_size"], asks["max_group_size"]
        if not np.all((mn == 1) & (mx <= 1)):
            raise ValueError("the collapsed reference covers solo tables only (min_group_size 1, max_group_size 0 or 1)")
        self.wa, self.wb, self.T, self.W = wa, wb, len(asks), len(wa)
        self.enabled = np.ones(self.T, dtype=bool) if enabled is None else np.asarray(enabled, dtype=bool)
        self.classes = model_classes(bits, n_patterns, n_models, words)
        self.prof, rep_w = worker_profiles(wa, wb, self.classes)
        self.row, rep_a, rep_o = ask_rows(asks, opts)
        self.P, self.U = len(rep_w), len(rep_a)
        self.F = feasibility(wa[rep_w], wb[rep_w], rep_a, rep_o, bits, words)
        # the first enabled ask of each distinct row, then the first ask of each profile
        first_t = np.full(self.U, NONE, dtype=np.int64)
        t_en = np.flatnonzero(self.enabled)
        np.minimum.at(first_t, self.row[t_en], t_en)
        pf = np.full(self.P, NONE, dtype=np.int64)
        for u0, u1 in _row_chunks(self.U, self.P):
            pf = np.minimum(pf, np.where(self.F[u0:u1], first_t[u0:u1, None], NONE).min(axis=0, initial=NONE))
        self.profile_first = pf

    # ---- per-ask statistics over a worker range
    def _ask_stats(self, w0, n):
        prof = self.prof[w0:w0 + n]
        mult = np.bincount(prof, minlength=self.P).astype(np.float64)
        best_p = np.full(self.P, INF, dtype=np.int64)
        if n:
            packed = packed_cost(self.wb[w0:w0 + n], w0)
            order = np.lexsort((packed, prof))
            head = np.ones(n, dtype=bool)
            head[1:] = prof[order][1:] != prof[order][:-1]
            best_p[prof[order][head]] = packed[order][head]
        cnt_u = np.zeros(self.U, dtype=np.int64)
        best_u = np.full(self.U, INF, dtype=np.int64)
        for u0, u1 in _row_chunks(self.U, self.P):
            blk = self.F[u0:u1]
            cnt_u[u0:u1] = np.rint(blk.astype(np.float64) @ mult).astype(np.int64)   # exact: counts < 2^53
            best_u[u0:u1] = np.where(blk, best_p[None, :], INF).min(axis=1, initial=INF)
        cnt = np.where(self.enabled, cnt_u[self.row], 0).astype(np.uint32)
        best = np.where(self.enabled, best_u[self.row], INF).astype(np.int64)
        return best, cnt

    def worker_ask(self):
        return self.profile_first[self.prof].astype(np.uint32)

    def result(self, ask_stats=True) -> dict:
        """Every array pm_fetch_result returns after a first-fit pass (PM_NO_ASK_STATS: ask_stats=False)."""
        wk = self.worker_ask()
        assigned = np.flatnonzero(wk != NONE)
        order = assigned[np.argsort(wk[assigned], kind="stable")].astype(np.uint32)   # creation order: (ask, worker)
        wg = np.full(self.W, NONE, dtype=np.uint32)
        wg[order] = np.arange(len(order), dtype=np.uint32)
        if ask_stats:
            best, cnt = self._ask_stats(0, self.W)
        else:
            best, cnt = np.full(self.T, INF, dtype=np.int64), np.zeros(self.T, dtype=np.uint32)
        return dict(worker_group=wg, worker_ask=wk, group_ask=wk[order], group_off=np.arange(len(order) + 1, dtype=np.uint32),
                    group_members=order, ask_best=best, ask_count=cnt)

    def local(self, w0, n, ask_stats=True) -> dict:
        """One shard's arrays after pm_match_local over workers [w0, w0 + n): first_ask over the whole table (NONE
        outside the range), and the per-ask minimum and count over the range."""
        fa = np.full(self.W, NONE, dtype=np.uint32)
        fa[w0:w0 + n] = self.profile_first[self.prof[w0:w0 + n]]
        if ask_stats:
            best, cnt = self._ask_stats(w0, n)
        else:
            best, cnt = np.full(self.T, INF, dtype=np.int64), np.zeros(self.T, dtype=np.uint32)
        return dict(first_ask=fa, ask_best=best, ask_count=cnt)


FIELDS = ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count")
CERT_FIELDS = ("cost", "bound", "gap", "n_held", "n_bad_holds", "n_shared", "n_priced_unowned", "priced_unowned_sum",
               "n_slack_over", "max_slack", "evals")


def certificate(wa, wb, asks, opts, bits, n_patterns, n_models, words, cap, S, price, assigned, reputation=None,
                floors=None) -> dict:
    """pm_auction_certificate's fields (tests/auction_certificate.certificate) without the dense matrix.

    feasible(t, w) = candidate, compatible (max_group_size is a reference-mode clause, ignored here), ask_price[w] <=
    cap[t], reputation[w] >= floor[t].  key(w) = ask_price[w] * S + price[w]; row(t) = min((cap[t] + 1) * S, min over
    feasible w of key(w)).  Within a profile the members are sorted by ask price and keep prefix minima of key, so a
    profile's term for ask t is the prefix minimum over its members with ask_price <= cap[t].  Sums are Python ints."""
    T, W, S = len(asks), len(wa), int(S)
    cap = np.asarray(cap, dtype=np.int64)
    ap = wb["ext_ask_price"].astype(np.int64)
    pr = np.asarray(price, dtype=np.int64)[:W]
    assigned = np.asarray(assigned, dtype=np.uint32)
    rep_col = None if floors is None else (np.zeros(W, dtype=np.uint32) if reputation is None else np.asarray(reputation, dtype=np.uint32))
    fl = np.zeros(T, dtype=np.int64) if floors is None else np.asarray(floors, dtype=np.int64)
    classes = model_classes(bits, n_patterns, n_models, words)
    prof, rep_w = worker_profiles(wa, wb, classes, extra=rep_col)
    row, rep_a, rep_o = ask_rows(asks, opts, max_at_least_one=True)
    P = len(rep_w)
    F = feasibility(wa[rep_w], wb[rep_w], rep_a, rep_o, bits, words)
    rep_rep = (rep_col[rep_w] if rep_col is not None else np.zeros(P, dtype=np.uint32)).astype(np.int64)
    key = ap * S + pr
    assert W == 0 or (key.min() >= 0), "negative prices are outside the certificate's domain"
    # members by (profile, ask price, key): prefix minima of key within each profile
    order = np.lexsort((key, ap, prof))
    sp, sa, sk = prof[order], ap[order], key[order]
    starts = np.searchsorted(sp, np.arange(P + 1))
    pmin = np.empty(W, dtype=np.int64)
    for p in range(P):
        s, e = starts[p], starts[p + 1]
        np.minimum.accumulate(sk[s:e], out=pmin[s:e])
    comp = sp.astype(np.int64) * (1 << 33) + sa          # ask prices are u32: one composite sort key
    outside = (cap + 1) * S
    row_t = np.empty(T, dtype=np.int64)
    big = np.iinfo(np.int64).max
    for (c, f) in sorted(set(zip(cap.tolist(), fl.tolist()))):
        ts = np.flatnonzero((cap == c) & (fl == f))
        last = np.searchsorted(comp, np.arange(P, dtype=np.int64) * (1 << 33) + c, side="right") - 1
        q = np.where(last >= starts[:P], pmin[np.maximum(last, 0)], big)
        q = np.where(rep_rep >= f, q, big)
        us, inv = np.unique(row[ts], return_inverse=True)
        best = np.empty(len(us), dtype=np.int64)
        for u0, u1 in _row_chunks(len(us), P):
            best[u0:u1] = np.where(F[us[u0:u1]], q[None, :], big).min(axis=1, initial=big)
        row_t[ts] = np.minimum(outside[ts], best[inv.reshape(-1)])
    held = (assigned != NONE) & (assigned < W)
    th = np.flatnonzero(held)
    wh = assigned[th].astype(np.int64)
    ok = F[row[th], prof[wh]] & (ap[wh] <= cap[th]) & (rep_rep[prof[wh]] >= fl[th])
    own = np.bincount(wh, minlength=W)
    slack = [int(x) for x in (outside - row_t)]
    for t, w in zip(th.tolist(), wh.tolist()):
        slack[t] = int(key[w]) - int(row_t[t])
    free = (own == 0) & (pr > 0)
    cost = sum(int(x) for x in ap[wh]) * S + sum(int(x) for x in outside[~held])
    bound = sum(int(x) for x in row_t) - sum(int(x) for x in pr)
    return dict(cost=cost, bound=bound, gap=cost - bound, n_held=len(th), n_bad_holds=int((~ok).sum()),
                n_shared=int((own > 1).sum()), n_priced_unowned=int(free.sum()),
                priced_unowned_sum=sum(int(x) for x in pr[free]), n_slack_over=sum(1 for s in slack if s > 1),
                max_slack=max(slack) if T else 0, evals=T * W, ask_bound=row_t, slack=slack)
