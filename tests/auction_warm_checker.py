"""Sequential checker of the auction's warm start (PM_AUCTION_WARM, DESIGN 4), and the random table histories the
warm-start tests drive through it and through the engine.

Self-oracle like the cold auction's (no reference counterpart).  The checker is written from the rule, independently
of the engine: feasibility comes from the oracle's own predicate, the release is a worklist over one raised worker at a
time, and the rounds restate orc_soa_auction's synchronous rounds over the whole feasibility matrix.  It computes the
release closure itself from the stored state and the changes it is told about; nobody hands it the released set.
"""
from __future__ import annotations

import numpy as np

from oracle import pm_oracle as orc
from protocol_b200 import abi

NONE = 0xFFFFFFFF
NEG = np.iinfo(np.int64).min // 4


def feasible(wa, wb, asks, opts, bits, words, cap, reputation=None, floors=None):
    """bool[T, W]: candidate(w) and compatible(t, w) (the oracle's predicate), ask_price[w] <= cap[t] and
    reputation[w] >= floor[t] (a missing column is a column of zeros)."""
    T, W = len(asks), len(wa)
    if T == 0 or W == 0:
        return np.zeros((T, W), dtype=bool)
    k = np.ascontiguousarray(asks).copy()
    k["max_group_size"] = np.maximum(k["max_group_size"], 1)   # that clause belongs to the reference modes only
    ev = orc.soa_eval_matrix(wa, wb, k, opts, bits, words, 0, T, 0, W, threads=8, want_cost=True, want_rows=False,
                             want_cols=False)
    F = ev["cost"] != abi.PM_COST_INF
    F &= wb["ext_ask_price"][None, :] <= np.asarray(cap)[:, None]
    if floors is not None:
        rep = np.zeros(W, dtype=np.uint32) if reputation is None else np.asarray(reputation)
        F &= rep[None, :] >= np.asarray(floors)[:, None]
    return F


def rounds(F, ask_price, cap, S, price, assigned, eps=1):
    """Synchronous rounds from (price, assigned), every unassigned ask active: orc_soa_auction's inner loop.
    Returns (assigned, price, number of rounds)."""
    T, W = F.shape
    price = np.array(price, dtype=np.int64)
    assigned = np.array(assigned, dtype=np.uint32)
    owner = np.full(W, NONE, dtype=np.uint32)
    held = np.flatnonzero(assigned != NONE)
    owner[assigned[held]] = held
    withdrawn = np.zeros(T, dtype=bool)
    base = -(np.asarray(ask_price, dtype=np.int64) * S)
    outside = -((np.asarray(cap, dtype=np.int64) + 1) * S)
    n = 0
    while True:
        act = np.flatnonzero((assigned == NONE) & ~withdrawn)
        if len(act) == 0:
            break
        n += 1
        if W == 0:
            withdrawn[act] = True
            continue
        V = np.where(F[act], (base - price)[None, :], NEG)
        r = np.arange(len(act))
        w1 = V.argmax(axis=1)                        # ties: the lowest worker index
        b1 = V[r, w1].copy()
        V[r, w1] = NEG
        b2 = V.max(axis=1)                            # the second best of the multiset
        out = b1 == NEG
        out |= b1 < outside[act]
        withdrawn[act[out]] = True
        keep = ~out
        bt, bw = act[keep], w1[keep]
        bp = price[bw] + (b1[keep] - np.maximum(b2[keep], outside[bt])) + eps
        # a worker takes the highest bid; ties go to the lowest ask index
        order = np.lexsort((bt, -bp, bw))
        bt, bw, bp = bt[order], bw[order], bp[order]
        first = np.ones(len(bw), dtype=bool)
        first[1:] = bw[1:] != bw[:-1]
        bt, bw, bp = bt[first], bw[first], bp[first]
        prev = owner[bw]
        assigned[prev[prev != NONE]] = NONE
        owner[bw] = bt
        assigned[bt] = bw
        price[bw] = bp
    return assigned, price, n


def cold(F, ask_price, cap, S):
    T, W = F.shape
    return rounds(F, ask_price, cap, S, np.zeros(W, dtype=np.int64), np.full(T, NONE, dtype=np.uint32))


def release(F, ask_price, S, price, assigned, n_kept, changed_rows, changed_asks, eps=1):
    """Steps 1-3 of the warm start.  price / assigned: the stored state (over the rows of its pass); n_kept: the stored
    rows no shrink has cut off since; changed_rows, changed_asks: R0 and A0 (rows from n_kept on are changed rows too).
    Returns (price[W], assigned, released asks sorted, R in the order it was built)."""
    T, W = F.shape
    keep = min(n_kept, W)
    p = np.zeros(W, dtype=np.int64)
    p[:keep] = np.asarray(price, dtype=np.int64)[:keep]
    assigned = np.array(assigned, dtype=np.uint32)
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
        if assigned[t] != NONE and assigned[t] >= keep:      # its worker was cut off by a shrink
            give_up(t)
    for w in changed_rows:
        if w < W and owner[w] != NONE:
            give_up(int(owner[w]))
    for t in changed_asks:
        give_up(int(t))
    R, in_r = [], np.zeros(W, dtype=bool)
    for w in range(W):                                       # every unowned worker goes to price 0
        if owner[w] == NONE and p[w] != 0:
            p[w] = 0
            R.append(w)
            in_r[w] = True
    for w in sorted(set(int(x) for x in changed_rows if x < W) | set(range(keep, W))):
        if not in_r[w]:
            R.append(w)
            in_r[w] = True
    ap = np.asarray(ask_price, dtype=np.int64)
    i = 0
    while i < len(R):                                        # closure: one raised worker at a time
        w = R[i]
        i += 1
        v = -(ap[w] * S) - p[w]
        for t in np.flatnonzero(assigned != NONE):
            wt = int(assigned[t])
            if F[t, w] and v - eps > -(ap[wt] * S) - p[wt]:
                give_up(int(t))
                p[wt] = 0
                R.append(wt)
    return p, assigned, np.array(sorted(released), dtype=np.int64), R


def warm(F, ask_price, cap, S, price, assigned, n_kept, changed_rows, changed_asks):
    """A warm pass: the release, then one phase of rounds at eps = 1.  Returns (assigned, price, rounds, released)."""
    p, a, rel, _ = release(F, ask_price, S, price, assigned, n_kept, changed_rows, changed_asks)
    a, p, n = rounds(F, ask_price, cap, S, p, a)
    return a, p, n, rel


def total_cost(assigned, ask_price, cap):
    """sum over asks of ask_price of its worker, or cap + 1 (the outside option) when it holds none."""
    held = assigned != NONE
    return int(np.asarray(ask_price, dtype=np.int64)[assigned[held]].sum() + (np.asarray(cap, dtype=np.int64)[~held] + 1).sum())


def check_feasible_injective(F, assigned):
    held = np.flatnonzero(assigned != NONE)
    assert len(np.unique(assigned[held])) == len(held)
    assert F[held, assigned[held]].all()


# ---------------------------------------------------------------- random histories
class Market:
    """The current tables and the changes since the stored state, as the engine tracks them."""

    def __init__(self, t, cap, reputation=None, floors=None):
        self.wa, self.wb = t["wa"].copy(), t["wb"].copy()
        self.asks, self.opts, self.bits, self.words = t["asks"], t["opts"], t["bits"], t["words"]
        self.cap = np.array(cap, dtype=np.uint32)
        self.reputation = None if reputation is None else np.array(reputation, dtype=np.uint32)
        self.floors = None if floors is None else np.array(floors, dtype=np.uint32)
        self.store(None, None)

    @property
    def n_workers(self):
        return len(self.wa)

    def F(self):
        return feasible(self.wa, self.wb, self.asks, self.opts, self.bits, self.words, self.cap, self.reputation, self.floors)

    def floors_or_zero(self):
        return np.zeros(len(self.asks), dtype=np.uint32) if self.floors is None else self.floors

    def store(self, price, assigned):
        """A pass ran: its state is the stored one, and nothing has changed since."""
        self.price, self.assigned = price, assigned
        self.rows, self.toggled, self.n_kept = set(), set(), self.n_workers
        self.cap0, self.floors0 = self.cap.copy(), self.floors_or_zero().copy()

    def changed_rows(self):
        return sorted(self.rows)

    def changed_asks(self):
        d = (self.cap != self.cap0) | (self.floors_or_zero() != self.floors0)
        return sorted(set(np.flatnonzero(d).tolist()) | self.toggled)

    def n_changes(self):
        return len(self.rows) + (self.n_workers - self.n_kept) + len(self.changed_asks())

    def warm(self, S=1):
        F = self.F()
        return warm(F, self.wb["ext_ask_price"], self.cap, S, self.price, self.assigned, self.n_kept,
                    self.changed_rows(), self.changed_asks())

    def cold(self, S=1):
        return cold(self.F(), self.wb["ext_ask_price"], self.cap, S)

    # ---- changes, applied to the market and (when given) to an engine
    def write(self, idx, a, b, eng=None):
        idx = np.asarray(idx, dtype=np.uint32)
        self.wa[idx], self.wb[idx] = a, b
        self.rows |= {int(i) for i in idx if i < self.n_kept}
        if eng is not None:
            eng.update_workers(idx, a, b)

    def set_flags(self, idx, flags, eng=None):
        idx = np.asarray(idx, dtype=np.uint32)
        self.wa["flags"][idx] = flags
        self.rows |= {int(i) for i in idx if i < self.n_kept}
        if eng is not None:
            eng.set_flags(idx, np.asarray(flags, dtype=np.uint32))

    def resize(self, n, a=None, b=None, eng=None):
        """Shrink to n rows, or grow to n and write the new rows (a, b)."""
        W = self.n_workers
        if n < W:
            self.wa, self.wb = self.wa[:n].copy(), self.wb[:n].copy()
            if self.reputation is not None:
                self.reputation = self.reputation[:n].copy()
            self.n_kept = min(self.n_kept, n)
            self.rows = {r for r in self.rows if r < n}
        else:
            self.wa = np.concatenate([self.wa, a]).astype(abi.WORKER_A)
            self.wb = np.concatenate([self.wb, b]).astype(abi.WORKER_B)
            if self.reputation is not None:
                self.reputation = np.concatenate([self.reputation, np.zeros(n - W, dtype=np.uint32)])
        if eng is not None:
            eng.resize_workers(n)
            if n > W:
                eng.upsert_workers(np.ascontiguousarray(a, dtype=abi.WORKER_A), np.ascontiguousarray(b, dtype=abi.WORKER_B), W)

    def set_caps(self, cap, eng=None):
        self.cap = np.array(cap, dtype=np.uint32)
        if eng is not None:
            eng.set_price_caps(self.cap)

    def set_floors(self, floors, eng=None):
        self.floors = np.array(floors, dtype=np.uint32)
        if eng is not None:
            eng.set_min_reputation(self.floors)

    def set_reputation(self, first, values, eng=None):
        if self.reputation is None:
            self.reputation = np.zeros(self.n_workers, dtype=np.uint32)
        values = np.asarray(values, dtype=np.uint32)
        self.reputation[first:first + len(values)] = values
        self.rows |= {i for i in range(first, first + len(values)) if i < self.n_kept}
        if eng is not None:
            eng.set_worker_reputation(values, first)

    def toggle(self, idx, eng=None):
        """Switch the asks off and on again (the auction refuses disabled asks; a toggle still counts as a change)."""
        self.toggled |= {int(i) for i in idx}
        if eng is not None:
            eng.set_ask_enabled(idx, False)
            eng.set_ask_enabled(idx, True)


def random_step(m: Market, rng, n_rows=None, eng=None, kinds=None):
    """One random change: writes to owned or unowned rows (price up or down, flags off and on, another row's spec),
    a resize that grows or shrinks the table, cap or floor changes, or toggles."""
    W, T = m.n_workers, len(m.asks)
    kinds = kinds or ("price", "flags", "spec", "resize", "caps", "floors", "toggle", "reputation")
    kind = kinds[rng.integers(len(kinds))]
    held = m.assigned[m.assigned != NONE] if m.assigned is not None else np.zeros(0, dtype=np.uint32)
    held = held[held < W]
    k = n_rows or int(rng.integers(1, max(2, W // 50)))

    def pick(k):
        owned = rng.random() < 0.5 and len(held)
        pool = held if owned else np.arange(W)
        return np.unique(rng.choice(pool, size=min(k, len(pool)), replace=False)).astype(np.uint32)

    if kind == "price":
        idx = pick(k)
        a, b = m.wa[idx].copy(), m.wb[idx].copy()
        p = b["ext_ask_price"].astype(np.int64)
        b["ext_ask_price"] = np.clip(np.where(rng.random(len(idx)) < 0.5, p // 2, p * 2 + 1), 1, 1 << 20)
        m.write(idx, a, b, eng)
    elif kind == "flags":
        idx = pick(k)
        m.set_flags(idx, m.wa["flags"][idx] ^ abi.PM_W_HEALTHY, eng)
    elif kind == "spec":
        idx = pick(k)
        src = rng.integers(0, W, len(idx))
        m.write(idx, m.wa[src].copy(), m.wb[src].copy(), eng)
    elif kind == "resize":
        if rng.random() < 0.5 and W > 4:
            m.resize(W - int(rng.integers(1, max(2, W // 20))), eng=eng)
        else:
            n = int(rng.integers(1, max(2, W // 20)))
            src = rng.integers(0, W, n)
            m.resize(W + n, m.wa[src].copy(), m.wb[src].copy(), eng)
    elif kind == "caps":
        cap = m.cap.copy()
        idx = rng.choice(T, size=min(T, int(rng.integers(1, max(2, T // 10)))), replace=False)
        cap[idx] = np.clip(cap[idx].astype(np.int64) + rng.integers(-100, 100, len(idx)), 0, None)
        m.set_caps(cap, eng)
    elif kind == "floors":
        fl = m.floors_or_zero().copy()
        idx = rng.choice(T, size=min(T, int(rng.integers(1, max(2, T // 10)))), replace=False)
        fl[idx] = rng.integers(0, 3, len(idx))
        m.set_floors(fl, eng)
    elif kind == "toggle":
        m.toggle(rng.choice(T, size=min(T, int(rng.integers(1, 4))), replace=False).astype(np.uint32), eng)
    elif kind == "reputation":
        first = int(rng.integers(0, W))
        m.set_reputation(first, rng.integers(0, 4, min(k, W - first)), eng)
    return kind
