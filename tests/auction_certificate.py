"""The auction certificate (pm_auction_certificate, DESIGN 4) restated in exact Python integers.

Written from the rule, independently of the engine: feasibility is the oracle's evaluation matrix with the cap and
floor clauses (auction_warm_checker.feasible), the row terms are masked minima over the whole matrix, ownership is
recounted from the assignment, and every sum is a Python int (nothing wraps).  For any prices >= 0,

    bound = sum_t min((cap[t] + 1) * S, min over feasible w of ask_price[w] * S + price[w]) - sum_w price[w]

is a lower bound on the optimal total cost (weak LP duality), and gap = cost - bound bounds the stored assignment's
distance from the optimum.
"""
from __future__ import annotations

import numpy as np

import auction_warm_checker as wc

NONE = wc.NONE


def certificate(F, ask_price, cap, S, price, assigned):
    """Every field of pm_auction_cert, as Python ints, plus ask_bound (int64[T]) and slack (Python ints per ask)."""
    T, W = F.shape
    S = int(S)
    ap = [int(x) for x in np.asarray(ask_price)[:W]]
    pr = [int(x) for x in np.asarray(price)[:W]]
    key = [ap[w] * S + pr[w] for w in range(W)]
    assert all(0 <= k < (1 << 63) for k in key)   # exact as int64 below
    key64 = np.array(key, dtype=np.int64)
    outside = [(int(c) + 1) * S for c in cap]
    big = np.iinfo(np.int64).max
    rowmin = np.where(F, key64[None, :], big).min(axis=1) if W else np.full(T, big, dtype=np.int64)
    row = [min(outside[t], int(rowmin[t])) for t in range(T)]
    own = [0] * W
    cost, slack = 0, []
    n_held = n_bad = 0
    for t in range(T):
        a = int(assigned[t])
        if a != NONE and a < W:
            n_held += 1
            own[a] += 1
            n_bad += int(not F[t, a])
            cost += ap[a] * S
            slack.append(key[a] - row[t])
        else:
            cost += outside[t]
            slack.append(outside[t] - row[t])
    bound = sum(row) - sum(pr)
    free = [w for w in range(W) if own[w] == 0 and pr[w] > 0]
    return dict(cost=cost, bound=bound, gap=cost - bound, n_held=n_held, n_bad_holds=n_bad,
                n_shared=sum(1 for o in own if o > 1), n_priced_unowned=len(free),
                priced_unowned_sum=sum(pr[w] for w in free), n_slack_over=sum(1 for s in slack if s > 1),
                max_slack=max(slack) if T else 0, evals=T * W, ask_bound=np.array(row, dtype=np.int64), slack=slack)


def market_certificate(m: wc.Market, S, price, assigned):
    """certificate() over a warm-checker market's current tables."""
    return certificate(m.F(), m.wb["ext_ask_price"], m.cap, S, price, assigned)


FIELDS = ("cost", "bound", "gap", "n_held", "n_bad_holds", "n_shared", "n_priced_unowned", "priced_unowned_sum",
          "n_slack_over", "max_slack", "evals")
