"""Sequential checker of the auction's warm repair (PM_AUCTION_WARM | PM_AUCTION_REPAIR, DESIGN 4).

Self-oracle like the other auction checkers (no reference counterpart), written from the rule in prime_match.h:
  1. release: the warm start's give-ups (every ask of A0, every owner of a row of R0, every holder of a row a shrink cut
     off), without its price reset: a released worker becomes unowned at its stored price;
  2. raise: every row of R0 and every row added since gets price max(0, beta - eps), beta the largest a(w) - pi(t) over
     the asks t that still hold a worker and are feasible for w (0 when there is none), all read from the state after 1;
  3. the forward rounds at eps = 1 (auction_warm_checker.rounds), every unassigned ask active;
  4. one reverse stage at eps = 1 (auction_reverse_checker.reverse).
`Repair` restates the same rule in Python integers on top of auction_exact.Auction, for the edges of the domain.
"""
from __future__ import annotations

import numpy as np

import auction_exact as ex
import auction_reverse_checker as rc
import auction_warm_checker as wc

NONE = wc.NONE
NEG = wc.NEG


def release(price, assigned, W, n_kept, changed_rows, changed_asks):
    """Step 1.  price / assigned: the stored state (over the rows of its pass); n_kept: the stored rows no shrink has cut
    off since; changed_rows, changed_asks: R0 and A0.  Returns (price[W], assigned, released asks sorted, the raised
    rows R0 + [n_kept, W) sorted)."""
    keep = min(n_kept, W)
    p = np.zeros(W, dtype=np.int64)
    p[:keep] = np.asarray(price, dtype=np.int64)[:keep]
    assigned = np.array(assigned, dtype=np.uint32)
    T = len(assigned)
    owner = np.full(W, NONE, dtype=np.uint32)
    for t in range(T):
        if assigned[t] != NONE and assigned[t] < keep:
            owner[assigned[t]] = t
    released = set()

    def give_up(t):
        w = int(assigned[t])
        if w == NONE:
            return
        assigned[t] = NONE
        released.add(t)
        if w < W:
            owner[w] = NONE

    for t in range(T):
        if assigned[t] != NONE and assigned[t] >= keep:
            give_up(t)
    for w in changed_rows:
        if w < W and owner[w] != NONE:
            give_up(int(owner[w]))
    for t in changed_asks:
        give_up(int(t))
    rows = sorted(set(int(x) for x in changed_rows if x < W) | set(range(keep, W)))
    return p, assigned, np.array(sorted(released), dtype=np.int64), np.array(rows, dtype=np.int64)


def raise_rows(F, ask_price, cap, S, price, assigned, rows, eps=1, held_only=True):
    """Step 2 over the rows `rows`, every beta from the state (price, assigned) given.  held_only=False also counts the
    asks that hold no worker (pi = their outside option): not the rule, only there to show that it differs."""
    price = np.array(price, dtype=np.int64)
    rows = np.asarray(rows, dtype=np.int64)
    if len(rows) == 0:
        return price
    base = -(np.asarray(ask_price, dtype=np.int64) * S)
    outside = -((np.asarray(cap, dtype=np.int64) + 1) * S)
    pi = rc.profits(assigned, price, base, outside)
    asks = np.flatnonzero(assigned != NONE) if held_only else np.arange(len(assigned))
    FR = F[asks][:, rows]
    G = np.where(FR, base[rows][None, :] - pi[asks][:, None], NEG)
    beta = G.max(axis=0) if len(asks) else np.full(len(rows), NEG, dtype=np.int64)
    has = FR.any(axis=0) if len(asks) else np.zeros(len(rows), dtype=bool)
    out = price.copy()
    out[rows] = np.where(has, np.maximum(0, beta - eps), 0)
    return out


def check_held_eps_cs(F, ask_price, cap, S, price, assigned, eps=1):
    """eps-CS over every held ask against every worker (the unassigned asks still bid)."""
    held = np.flatnonzero(assigned != NONE)
    rc.check_eps_cs(F[held], ask_price, np.asarray(cap)[held], S, price, assigned[held], eps)


def repair(F, ask_price, cap, S, price, assigned, n_kept, changed_rows, changed_asks, check=False):
    """A repair pass.  Returns dict(assigned, price, fwd, rev, bids, released, raised)."""
    T, W = F.shape
    p, a, rel, rows = release(price, assigned, W, n_kept, changed_rows, changed_asks)
    p = raise_rows(F, ask_price, cap, S, p, a, rows)
    if check:
        check_held_eps_cs(F, ask_price, cap, S, p, a)
    a, p, n_fwd = wc.rounds(F, ask_price, cap, S, p, a, eps=1)
    if check:
        rc.check_eps_cs(F, ask_price, cap, S, p, a, 1)
    a, p, n_rev, n_bids = rc.reverse(F, ask_price, cap, S, p, a, 1, check=check)
    return dict(assigned=a, price=p, fwd=n_fwd, rev=n_rev, bids=n_bids, released=rel, raised=rows)


def market_repair(m: wc.Market, S=1, check=False):
    """repair() over a warm-checker market: its current tables and the changes since its stored state."""
    return repair(m.F(), m.wb["ext_ask_price"], m.cap, S, m.price, m.assigned, m.n_kept, m.changed_rows(),
                  m.changed_asks(), check=check)


class Repair(ex.Auction):
    """The repair pass in Python integers (no sentinel, nothing wraps)."""

    def repair(self, price, assigned, n_kept, n_workers, changed_rows, changed_asks, max_rounds=20000):
        """From the stored state (price over its rows, assigned per ask; NONE = no worker).  Returns dict(fwd, rev,
        bids, released)."""
        keep = min(int(n_kept), int(n_workers))
        self.assigned = {t: int(w) for t, w in enumerate(assigned) if int(w) != NONE}
        self.owner = {w: t for t, w in self.assigned.items() if w < keep}
        self.price = {w: int(price[w]) for w in range(keep) if int(price[w]) != 0}
        released = set()

        def give_up(t):
            w = self.assigned.pop(t, None)
            if w is None:
                return
            released.add(t)
            self.owner.pop(w, None)

        for t, w in list(self.assigned.items()):
            if w >= keep:
                give_up(t)
        for w in changed_rows:
            if w < n_workers and w in self.owner:
                give_up(self.owner[w])
        for t in changed_asks:
            give_up(int(t))
        rows = {int(w) for w in changed_rows if w < n_workers} | set(range(keep, int(n_workers)))
        pi = {t: self.profit(t) for t in self.assigned}          # the held asks, after the release
        raised = {}
        for w in rows:
            gains = [self.a[w] - pi[t] for t in self.asks_of.get(w, ()) if t in pi]
            raised[w] = max(0, max(gains) - 1) if gains else 0
        for w, p in raised.items():
            if p:
                self.price[w] = p
            else:
                self.price.pop(w, None)
        fwd = self.forward(1, max_rounds)
        rev, bids = self.reverse(1, max_rounds)
        return dict(fwd=fwd, rev=rev, bids=bids, released=len(released))
