"""Sequential checker of the auction's reverse rounds (PM_AUCTION_REVERSE, DESIGN 4).

Self-oracle like the cold and warm auctions' (no reference counterpart).  Written from the rule in prime_match.h,
independently of the engine: the forward rounds of each eps phase are the warm checker's `rounds()` (orc_soa_auction's
synchronous rounds over the whole feasibility matrix), and a reverse round is one whole-round numpy step over the
bidders.  `reverse_gs` restates the stage with one bidder at a time (Gauss-Seidel), to show that the bound does not
rest on the synchronous order.
"""
from __future__ import annotations

import numpy as np

import auction_warm_checker as wc

NONE = wc.NONE
NEG = wc.NEG


def _owner(assigned, W):
    owner = np.full(W, NONE, dtype=np.uint32)
    held = np.flatnonzero(assigned != NONE)
    owner[assigned[held]] = held
    return owner


def profits(assigned, price, base, outside):
    """pi(t): value of the held worker a(w_t) - price[w_t], else the outside option."""
    pi = np.array(outside, dtype=np.int64)
    held = np.flatnonzero(assigned != NONE)
    pi[held] = base[assigned[held]] - price[assigned[held]]
    return pi


def check_eps_cs(F, ask_price, cap, S, price, assigned, eps):
    """eps-complementary slackness over the whole matrix: a(w) - price[w] <= pi(t) + eps for every feasible (t, w)."""
    base = -(np.asarray(ask_price, dtype=np.int64) * S)
    outside = -((np.asarray(cap, dtype=np.int64) + 1) * S)
    pi = profits(assigned, np.asarray(price, dtype=np.int64), base, outside)
    slack = (base - price)[None, :] - pi[:, None]
    bad = F & (slack > eps)
    assert not bad.any(), f"eps-CS violated on {int(bad.sum())} pairs"


def reverse(F, ask_price, cap, S, price, assigned, eps, check=False):
    """Reverse rounds from (price, assigned) until no unowned worker has a positive price.  check: assert eps-CS after
    every round.  Returns (assigned, price, rounds, bids)."""
    T, W = F.shape
    price = np.array(price, dtype=np.int64)
    assigned = np.array(assigned, dtype=np.uint32)
    owner = _owner(assigned, W)
    base = -(np.asarray(ask_price, dtype=np.int64) * S)
    outside = -((np.asarray(cap, dtype=np.int64) + 1) * S)
    n_rounds = n_bids = 0
    while True:
        B = np.flatnonzero((owner == NONE) & (price > 0))
        if len(B) == 0:
            break
        n_rounds += 1
        n_bids += len(B)
        pi = profits(assigned, price, base, outside)          # the state at the start of the round
        FB = F[:, B].T
        G = np.where(FB, base[B][:, None] - pi[None, :], NEG)
        r = np.arange(len(B))
        ts = G.argmax(axis=1)                                 # ties: the lowest ask index
        beta = G[r, ts].copy()
        G[r, ts] = NEG
        omega = G.max(axis=1)                                 # the second value of the multiset
        drop = ~FB.any(axis=1) | (beta <= eps)
        price[B[drop]] = 0
        bw, bt = B[~drop], ts[~drop].astype(np.uint32)
        pn = np.maximum(0, omega[~drop] - eps)
        profit = base[bw] - pn
        # each ask takes the highest profit; ties go to the lowest worker
        order = np.lexsort((bw, -profit, bt))
        bw, bt, pn = bw[order], bt[order], pn[order]
        first = np.ones(len(bt), dtype=bool)
        first[1:] = bt[1:] != bt[:-1]
        bw, bt, pn = bw[first], bt[first], pn[first]
        prev = assigned[bt]
        owner[prev[prev != NONE]] = NONE                      # keeps its price: it bids next round if that is positive
        owner[bw] = bt
        assigned[bt] = bw
        price[bw] = pn
        if check:
            check_eps_cs(F, ask_price, cap, S, price, assigned, eps)
    return assigned, price, n_rounds, n_bids


def reverse_gs(F, ask_price, cap, S, price, assigned, eps):
    """The same rule, one bidder at a time (the lowest unowned worker with a positive price), each bid seeing every
    earlier one.  Returns (assigned, price, bids)."""
    T, W = F.shape
    price = np.array(price, dtype=np.int64)
    assigned = np.array(assigned, dtype=np.uint32)
    owner = _owner(assigned, W)
    base = -(np.asarray(ask_price, dtype=np.int64) * S)
    outside = -((np.asarray(cap, dtype=np.int64) + 1) * S)
    n_bids = 0
    while True:
        B = np.flatnonzero((owner == NONE) & (price > 0))
        if len(B) == 0:
            break
        w = int(B[0])
        n_bids += 1
        pi = profits(assigned, price, base, outside)
        g = np.where(F[:, w], base[w] - pi, NEG)
        t = int(g.argmax())
        beta = g[t]
        g[t] = NEG
        omega = g.max()
        if not F[:, w].any() or beta <= eps:
            price[w] = 0
            continue
        prev = assigned[t]
        if prev != NONE:
            owner[prev] = NONE
        owner[w] = t
        assigned[t] = w
        price[w] = max(0, int(omega) - eps)
    return assigned, price, n_bids


def scaled(F, ask_price, cap, S, eps_start, eps_div, reverse_rounds=True, check=False, gauss_seidel=False):
    """An eps-scaled pass: per phase the forward rounds from cleared assignment and kept prices, then (reverse_rounds)
    the reverse stage.  Returns (assigned, price, forward rounds, reverse rounds, reverse bids, phases)."""
    T, W = F.shape
    eps = max(1, int(eps_start))
    div = max(2, int(eps_div))
    price = np.zeros(W, dtype=np.int64)
    n_fwd = n_rev = n_bids = n_phases = 0
    while True:
        a, price, n = wc.rounds(F, ask_price, cap, S, price, np.full(T, NONE, dtype=np.uint32), eps)
        n_fwd += n
        n_phases += 1
        if check:
            check_eps_cs(F, ask_price, cap, S, price, a, eps)
        if reverse_rounds:
            if gauss_seidel:
                a, price, nb = reverse_gs(F, ask_price, cap, S, price, a, eps)
                nr = 0
            else:
                a, price, nr, nb = reverse(F, ask_price, cap, S, price, a, eps, check=check)
            n_rev += nr
            n_bids += nb
        if eps == 1:
            break
        eps = max(1, eps // div)
    return a, price, n_fwd, n_rev, n_bids, n_phases


def optimum(F, ask_price, cap, S=1):
    """Minimum over injective partial assignments inside F of sum(ask_price * S held, (cap + 1) * S unheld): scipy's
    linear_sum_assignment on the masked matrix, an anchor that is not this repository's code."""
    from scipy.optimize import linear_sum_assignment

    T, W = F.shape
    BIG = 1 << 50
    ap = np.asarray(ask_price, dtype=np.int64)
    M = np.full((T, W + T), BIG, dtype=np.int64)
    M[:, :W] = np.where(F, ap[None, :] * S, BIG)
    M[np.arange(T), W + np.arange(T)] = (np.asarray(cap, dtype=np.int64) + 1) * S
    r, c = linear_sum_assignment(M)
    return int(M[r, c].sum())
