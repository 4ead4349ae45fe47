"""Exact-integer restatement of the price-capped auction (PM_MODE_AUCTION): the cold rounds and eps phases, the reverse
rounds of PM_AUCTION_REVERSE and the warm release of PM_AUCTION_WARM, written from the rules in prime_match.h.

Every number is a Python int, so nothing wraps whatever the prices, caps and scales, and "no worker" is None rather
than a sentinel value that a real value could equal.  Feasibility arrives as one list of workers per ask (ascending;
an ask left out has none), taken from the oracle's predicate: an instance with millions of infeasible rows or asks
costs only its feasible pairs.  Every entry point takes max_rounds and raises RoundLimit past it, so an instance that
would run an O(cost_scale) price war fails here, on the CPU, and never reaches a device.

Independent on purpose of auction_warm_checker / auction_reverse_checker (numpy int64 over a dense matrix, with
INT64_MIN / 4 as "no worker"): the two restatements are pinned to each other inside the int64-safe range only.
"""
from __future__ import annotations

import numpy as np

NONE = 0xFFFFFFFF
DOMAIN = 1 << 61   # (P + K + 2) * S + E must stay below this (prime_match.h)


class RoundLimit(RuntimeError):
    pass


def in_domain(max_ask_price: int, max_cap: int, cost_scale: int, eps_start: int) -> bool:
    return (int(max_ask_price) + int(max_cap) + 2) * max(1, int(cost_scale)) + max(1, int(eps_start)) < DOMAIN


def lists_from_matrix(F) -> dict[int, list[int]]:
    """Per-ask feasible lists from a dense bool[T, W]."""
    F = np.asarray(F, dtype=bool)
    return {t: np.flatnonzero(F[t]).tolist() for t in range(F.shape[0]) if F[t].any()}


class Auction:
    """One instance: n_asks asks, feasible lists, ask prices (indexable by worker), caps (indexable by ask), S.

    State: price (worker -> int, absent = 0), assigned (ask -> worker), owner (worker -> ask)."""

    def __init__(self, n_asks, feas, ask_price, cap, cost_scale=1):
        self.n_asks = int(n_asks)
        self.feas = {int(t): [int(w) for w in ws] for t, ws in feas.items() if len(ws)}
        self.S = max(1, int(cost_scale))
        self.a = {}                                   # a(w) = -(ask_price[w] * S), over the workers some ask may take
        self.asks_of = {}                             # worker -> asks feasible for it, ascending
        for t in sorted(self.feas):
            for w in self.feas[t]:
                if w not in self.a:
                    self.a[w] = -(int(ask_price[w]) * self.S)
                    self.asks_of[w] = []
                self.asks_of[w].append(t)
        self.outside = {t: -((int(cap[t]) + 1) * self.S) for t in self.feas}
        self.price: dict[int, int] = {}
        self.assigned: dict[int, int] = {}
        self.owner: dict[int, int] = {}

    def value(self, w):
        return self.a[w] - self.price.get(w, 0)

    def profit(self, t):
        w = self.assigned.get(t)
        return self.outside[t] if w is None else self.value(w)

    def _take(self, t, w, price):
        prev = self.owner.get(w)
        if prev is not None:
            del self.assigned[prev]
        old = self.assigned.get(t)
        if old is not None and self.owner.get(old) == t:
            del self.owner[old]
        self.owner[w] = t
        self.assigned[t] = w
        self.price[w] = price

    # ---- forward rounds
    def forward(self, eps, max_rounds):
        """Synchronous rounds at eps, every ask that holds no worker active (the asks without a feasible worker too:
        they withdraw in the first round).  Returns the rounds run."""
        withdrawn = set()
        n_empty = self.n_asks - len(self.feas)      # never hold a worker: active in the first round only
        n = 0
        while True:
            act = [t for t in sorted(self.feas) if t not in self.assigned and t not in withdrawn]
            if not act and not (n == 0 and n_empty):
                return n
            n += 1
            if n > max_rounds:
                raise RoundLimit(f"more than {max_rounds} forward rounds at eps = {eps}")
            best = {}                                 # worker -> (bid, ask): the highest bid, the lowest ask among equals
            for t in act:
                b1 = b2 = w1 = None
                for w in self.feas[t]:                # ascending: strict compares keep the lowest worker
                    v = self.value(w)
                    if b1 is None or v > b1:
                        b2, b1, w1 = b1, v, w
                    elif b2 is None or v > b2:
                        b2 = v
                out = self.outside[t]
                if b1 < out:
                    withdrawn.add(t)
                    continue
                second = out if b2 is None else max(b2, out)
                bid = self.price.get(w1, 0) + (b1 - second) + eps
                if w1 not in best or bid > best[w1][0]:
                    best[w1] = (bid, t)
            for w, (bid, t) in best.items():
                self._take(t, w, bid)

    # ---- reverse rounds
    def reverse(self, eps, max_rounds):
        """PM_AUCTION_REVERSE's stage: rounds until no unowned worker has a positive price.  Returns (rounds, bids)."""
        n_rounds = n_bids = 0
        while True:
            bidders = sorted(w for w, p in self.price.items() if p > 0 and w not in self.owner)
            if not bidders:
                return n_rounds, n_bids
            n_rounds += 1
            n_bids += len(bidders)
            if n_rounds > max_rounds:
                raise RoundLimit(f"more than {max_rounds} reverse rounds at eps = {eps}")
            pi = {t: self.profit(t) for t in self.feas}   # the state at the round's start
            offers = {}                                   # ask -> (profit, worker, price): highest profit, lowest worker
            for w in bidders:
                beta = omega = t_star = None
                for t in self.asks_of.get(w, ()):         # ascending: strict compares keep the lowest ask
                    g = self.a[w] - pi[t]
                    if beta is None or g > beta:
                        omega, beta, t_star = beta, g, t
                    elif omega is None or g > omega:
                        omega = g
                if beta is None or beta <= eps:
                    self.price[w] = 0
                    continue
                pn = 0 if omega is None else max(0, omega - eps)
                prof = self.a[w] - pn
                if t_star not in offers or prof > offers[t_star][0]:
                    offers[t_star] = (prof, w, pn)
            for t, (_, w, pn) in offers.items():
                prev = self.assigned.get(t)
                if prev is not None:
                    del self.owner[prev]                  # unowned at its price: it bids next round if that is positive
                self.owner[w] = t
                self.assigned[t] = w
                self.price[w] = pn

    # ---- passes
    def scaled(self, eps_start=1, eps_div=4, reverse=False, max_rounds=20000):
        """A cold pass: per eps phase the assignment is cleared, prices kept, forward rounds, then (reverse) the reverse
        stage.  Returns dict(fwd, rev, bids, phases)."""
        eps, div = max(1, int(eps_start)), max(2, int(eps_div))
        self.price, self.assigned, self.owner = {}, {}, {}
        st = dict(fwd=0, rev=0, bids=0, phases=0)
        while True:
            self.assigned, self.owner = {}, {}
            st["fwd"] += self.forward(eps, max_rounds - st["fwd"])
            st["phases"] += 1
            if reverse:
                r, b = self.reverse(eps, max_rounds - st["rev"])
                st["rev"] += r
                st["bids"] += b
            if eps == 1:
                return st
            eps = max(1, eps // div)

    def warm(self, price, assigned, n_kept, n_workers, changed_rows, changed_asks, max_rounds=20000):
        """A warm pass from the stored state (price over its rows, assigned per ask; NONE = no worker): the release
        (steps 1-3 of the warm start in prime_match.h), then rounds at eps = 1.  n_kept: the stored rows no shrink has
        cut off since; changed_rows, changed_asks: R0 and A0.  Returns dict(fwd, released)."""
        keep = min(int(n_kept), int(n_workers))
        assigned = [int(x) for x in assigned]
        self.assigned = {t: w for t, w in enumerate(assigned) if w != NONE}
        self.owner = {w: t for t, w in self.assigned.items() if w < keep}
        self.price = {w: int(price[w]) for w in range(keep) if int(price[w]) != 0}
        released = set()

        def give_up(t):
            w = self.assigned.pop(t, None)
            if w is None:
                return
            released.add(t)
            self.owner.pop(w, None)

        # step 2: every ask of A0, every owner of a changed row, every holder of a row cut off by a shrink
        for t, w in list(self.assigned.items()):
            if w >= keep:
                give_up(t)
        for w in changed_rows:
            if w < n_workers and w in self.owner:
                give_up(self.owner[w])
        for t in changed_asks:
            give_up(int(t))
        R = set()
        for w in list(self.price):                    # every unowned worker with a positive price goes to 0
            if w not in self.owner and self.price[w] > 0:
                self.price[w] = 0
                R.add(w)
        R |= {int(w) for w in changed_rows if w < n_workers} | set(range(keep, int(n_workers)))
        # step 3: the closure (monotone: R only grows and a raised worker's value is fixed, so any order gives it)
        changed = True
        while changed:
            changed = False
            for t in sorted(self.assigned):
                wt = self.assigned[t]
                best = None
                for w in self.feas.get(t, ()):
                    if w in R and (best is None or self.a[w] > best):
                        best = self.a[w]                # price 0 on R
                if best is not None and best - 1 > self.value(wt):
                    give_up(t)
                    self.price[wt] = 0
                    R.add(wt)
                    changed = True
        fwd = self.forward(1, max_rounds)
        return dict(fwd=fwd, released=len(released))

    # ---- results
    def assignment(self):
        out = np.full(self.n_asks, NONE, dtype=np.uint32)
        for t, w in self.assigned.items():
            out[t] = w
        return out

    def prices(self, n_workers):
        """int64[n_workers]; asserts every price fits (inside the domain they all do)."""
        out = np.zeros(n_workers, dtype=np.int64)
        for w, p in self.price.items():
            assert -(1 << 63) <= p < (1 << 63)
            if w < n_workers:
                out[w] = p
        return out

    def total_cost(self):
        """sum over the asks with a feasible worker of ask_price held * S, or the outside option (cap + 1) * S."""
        return sum(-self.a[self.assigned[t]] if t in self.assigned else -self.outside[t] for t in self.feas)
