"""The audit of pm_auction_restore (prime_match.h "Auction state restore", DESIGN 4) restated in numpy.

Written from the rule, independently of the engine: feasibility is auction_warm_checker.feasible (the oracle's
predicate with the cap and floor clauses), the row terms are auction_certificate's, and ownership is recounted from the
given assignment.  Each hold is checked in order: infeasible (bad), then its worker named by more than one ask (shared,
every naming counts), then slack key(w_t) - row(t) > 1.  A failing hold is dropped; no price changes.
"""
from __future__ import annotations

import numpy as np

import auction_certificate as ac
import auction_warm_checker as wc

NONE = wc.NONE


def price_bound(cap, S, eps_start=1):
    """The largest price a restore takes: (K + 1) * S + max(E, 1), K the largest cap."""
    K = int(np.max(cap)) if len(cap) else 0
    return (K + 1) * int(S) + max(int(eps_start), 1)


def audit(F, ask_price, cap, S, price, assigned):
    """Returns dict(assigned=the kept assignment (uint32[T]), n_held, n_dropped_bad, n_dropped_shared,
    n_dropped_slack, evals)."""
    T, W = F.shape
    assigned = np.asarray(assigned, dtype=np.uint32)
    assert np.all((assigned == NONE) | (assigned < W))
    row = ac.certificate(F, ask_price, cap, S, price, assigned)["ask_bound"]
    held = np.flatnonzero(assigned != NONE)
    own = np.bincount(assigned[held].astype(np.int64), minlength=W)
    ap = np.asarray(ask_price, dtype=np.int64)[:W]
    pr = np.asarray(price, dtype=np.int64)
    kept = np.full(T, NONE, dtype=np.uint32)
    n = dict(n_held=0, n_dropped_bad=0, n_dropped_shared=0, n_dropped_slack=0)
    for t in held:
        w = int(assigned[t])
        if not F[t, w]:
            n["n_dropped_bad"] += 1
        elif own[w] > 1:
            n["n_dropped_shared"] += 1
        elif int(ap[w]) * int(S) + int(pr[w]) - int(row[t]) > 1:
            n["n_dropped_slack"] += 1
        else:
            kept[t] = w
            n["n_held"] += 1
    return dict(assigned=kept, evals=T * W, **n)


def market_audit(m: wc.Market, S, price, assigned):
    """audit() over a warm-checker market's current tables."""
    return audit(m.F(), m.wb["ext_ask_price"], m.cap, S, price, assigned)


def adversarial_state(F, ask_price, cap, S, rng, eps_start=1):
    """A state an outside caller might hand over: prices anywhere in [0, price_bound] (many 0, some at the bound), and
    an assignment that mixes feasible holds, infeasible ones, workers named by two or three asks, and holds on costly
    workers (over-slack); priced workers that nobody holds come with it."""
    T, W = F.shape
    top = price_bound(cap, S, eps_start)
    price = rng.integers(0, top + 1, W).astype(np.int64)
    price[rng.random(W) < 0.4] = 0
    price[rng.random(W) < 0.05] = top
    assigned = np.full(T, NONE, dtype=np.uint32)
    if W == 0:
        return price, assigned
    for t in range(T):
        r = rng.random()
        ws = np.flatnonzero(F[t])
        if r < 0.45 and len(ws):
            assigned[t] = ws[np.argmin(np.asarray(ask_price, dtype=np.int64)[ws] * S + price[ws])]   # a low-slack hold
        elif r < 0.6 and len(ws):
            assigned[t] = rng.choice(ws)
        elif r < 0.75:
            assigned[t] = rng.integers(0, W)
    held = np.flatnonzero(assigned != NONE)
    if len(held) >= 3:   # a few workers named more than once
        for _ in range(max(1, len(held) // 10)):
            a, b = rng.choice(held, 2, replace=False)
            assigned[b] = assigned[a]
    return price, assigned
