"""Removing and inserting worker rows anywhere in the table (pm_remove_workers / pm_insert_workers) on the CPU.

The engine moves every row on the device without a W-entry map: the new index of a kept old row i is
i - |{removed r < i}| + |{before <= i}|, and inserted row k lands at before[k] - |{removed r < before[k]}| + k.  Here
that formula is checked against np.delete / np.insert, and the stored auction state is remapped on the host the way
the engine remaps it: prices and owners move with their rows, a hold on a removed row (or on a row an earlier shrink
cut off) is released by the next warm pass as a shrink's is, inserted rows are changed rows at price 0.  A warm pass
from that state keeps eps-CS on every held pair, stays within T of the optimum and is exact with cost_scale = T + 1;
removing the tail and inserting at the end are the checker's shrink and grow."""
import numpy as np
import pytest

import auction_repair_checker as rp
import auction_warm_checker as wc
from protocol_b200 import abi
from test_auction_warm_formulation import lsa_optimum, market

NONE = wc.NONE
CUT = 0xFFFFFFFE   # a hold on a row that is gone: released in step 1 of the next warm pass, exported as PM_NONE


class Splice:
    """The index arithmetic of one splice: `removed` old rows (any order, repeats once), `before` per inserted row."""

    def __init__(self, n_old, removed=(), before=()):
        self.n_old = n_old
        self.removed = np.unique(np.asarray(removed, dtype=np.int64))
        self.before = np.asarray(before, dtype=np.int64)
        assert np.all(np.diff(self.before) >= 0) and np.all(self.before <= n_old)
        self.n_new = n_old - len(self.removed) + len(self.before)

    def is_removed(self, i):
        i = np.asarray(i, dtype=np.int64)
        k = np.searchsorted(self.removed, i)
        return (k < len(self.removed)) & (self.removed[np.minimum(k, max(len(self.removed) - 1, 0))] == i) if len(self.removed) else np.zeros(i.shape, bool)

    def map(self, i):
        """the new index of kept old rows i"""
        i = np.asarray(i, dtype=np.int64)
        return i - np.searchsorted(self.removed, i, "left") + np.searchsorted(self.before, i, "right")

    def at(self):
        """the new index of every inserted row"""
        b = self.before
        return b - np.searchsorted(self.removed, b, "left") + np.arange(len(b))

    def edge(self, x):
        """the new index of the boundary in front of old row x, ahead of the rows inserted before x"""
        return int(x - np.searchsorted(self.removed, x, "left") + np.searchsorted(self.before, x, "left"))

    def apply(self, col, new_rows, fill=0):
        """a per-row column moved with its rows, new_rows (or fill) at the inserted positions"""
        kept = np.delete(np.asarray(col), self.removed)
        if len(self.before) == 0:
            return kept
        vals = np.full(len(self.before), fill, dtype=np.asarray(col).dtype) if new_rows is None else new_rows
        return np.insert(kept, self.before - np.searchsorted(self.removed, self.before, "left"), vals)


class SpliceMarket(wc.Market):
    """wc.Market with the worker splices, remapping the stored state as the engine does."""

    def splice(self, removed=(), before=(), a=None, b=None, eng=None):
        sp = Splice(self.n_workers, removed, before)
        assert not (len(sp.removed) and len(sp.before)), "one kind per call, as the engine's calls take them"
        if eng is not None:
            if len(sp.removed):
                eng.remove_workers(np.asarray(removed, dtype=np.uint32))
            if len(sp.before):
                eng.insert_workers(sp.before.astype(np.uint32), a, b)
        ins_a = None if a is None else np.asarray(a, dtype=abi.WORKER_A)
        ins_b = None if b is None else np.asarray(b, dtype=abi.WORKER_B)
        self.wa = sp.apply(self.wa, ins_a).astype(abi.WORKER_A)
        self.wb = sp.apply(self.wb, ins_b).astype(abi.WORKER_B)
        if self.reputation is not None:
            self.reputation = sp.apply(self.reputation, None).astype(np.uint32)
        if self.assigned is not None:
            keep = min(self.n_kept, sp.n_old)
            self.price = remap_prices(sp, self.price, keep)
            self.assigned = remap_holds(sp, self.assigned, keep)
            rows = np.array(sorted(self.rows), dtype=np.int64)
            rows = rows[~sp.is_removed(rows)] if len(rows) else rows
            self.rows = {int(r) for r in sp.map(rows)} | {int(j) for j, bf in zip(sp.at(), sp.before) if bf < keep}
            self.n_kept = sp.edge(keep)
        return sp


def remap_prices(sp, price, keep):
    """the stored prices over the new rows: kept rows below keep keep theirs, every other row is 0"""
    old = np.zeros(sp.n_old, dtype=np.int64)
    old[:keep] = np.asarray(price, dtype=np.int64)[:keep]
    return sp.apply(old, None).astype(np.int64)


def remap_holds(sp, assigned, keep):
    """the stored assignment renamed: a hold on a removed row, or on a row at or past keep, becomes CUT"""
    a = np.array(assigned, dtype=np.int64)
    out = np.full(len(a), NONE, dtype=np.int64)
    held = a != NONE
    gone = held & ((a >= keep) | sp.is_removed(np.where(held, a, 0)))
    out[gone] = CUT
    ok = held & ~gone
    out[ok] = sp.map(a[ok])
    return out.astype(np.uint32)


def exported(assigned):
    """pm_auction_assignment's view: a CUT hold reads PM_NONE"""
    a = np.array(assigned, dtype=np.uint32)
    a[a == CUT] = NONE
    return a


# ------------------------------------------------------------------ the index formula
@pytest.mark.parametrize("seed", range(8))
def test_index_formula_matches_delete_and_insert(seed):
    rng = np.random.default_rng(seed)
    for _ in range(50):
        W = int(rng.integers(0, 40))
        rm = rng.integers(0, W, int(rng.integers(0, W + 1))) if W and rng.random() < 0.7 else np.zeros(0, np.int64)
        n_kept = W - len(np.unique(rm))
        k = int(rng.integers(0, 6))
        bf = np.sort(rng.integers(0, W + 1, k))
        if rng.random() < 0.2:
            bf = np.full(k, W)                     # every row at n_workers
        elif rng.random() < 0.2:
            bf = np.zeros(k, np.int64)             # every row at position 0
        ids = np.arange(W)
        sp = Splice(W, rm, bf)
        want = np.insert(np.delete(ids, np.unique(rm)), bf - np.searchsorted(np.unique(rm), bf), -1 - np.arange(k))
        assert len(want) == sp.n_new == n_kept + k
        kept = np.setdiff1d(ids, rm)
        got = np.full(sp.n_new, -999)
        got[sp.map(kept)] = kept
        got[sp.at()] = -1 - np.arange(k)
        assert np.array_equal(got, want)
        assert np.array_equal(sp.apply(ids, -1 - np.arange(k)), want)


def test_repeated_indices_remove_once_and_empty_result():
    sp = Splice(5, [4, 1, 4, 1, 1])
    assert list(sp.removed) == [1, 4] and sp.n_new == 3
    assert list(sp.map([0, 2, 3])) == [0, 1, 2]
    sp = Splice(4, [3, 2, 1, 0, 0])
    assert sp.n_new == 0 and len(sp.apply(np.arange(4), None)) == 0
    sp = Splice(0, (), [0, 0, 0])
    assert list(sp.at()) == [0, 1, 2]


# ------------------------------------------------------------------ the auction from the remapped state
def _held_eps_cs(m, a, p, S):
    F = m.F()
    ap = m.wb["ext_ask_price"].astype(np.int64)
    rp.check_held_eps_cs(F, ap, m.cap, S, p, a)


def splice_history(seed, steps, S=1, floors=False, repair=False):
    m = SpliceMarket.__new__(SpliceMarket)
    base = market(14, 60, seed, floors=floors)
    m.__dict__.update(base.__dict__)
    rng = np.random.default_rng(seed)
    a, p, _ = m.cold(S)
    m.store(p, a)
    T = len(m.asks)
    for step in range(steps):
        W = m.n_workers
        held = m.assigned[(m.assigned != NONE) & (m.assigned < W)]
        kind = ("remove", "insert", "both", "other")[step % 4]
        if kind in ("remove", "both") and W > 8:
            pool = held if len(held) and rng.random() < 0.7 else np.arange(W)
            m.splice(rng.choice(pool, min(len(pool), int(rng.integers(1, 4))), replace=False))
        if kind in ("insert", "both"):
            k = int(rng.integers(1, 5))
            src = rng.integers(0, m.n_workers, k)
            m.splice((), np.sort(rng.integers(0, m.n_workers + 1, k)), m.wa[src].copy(), m.wb[src].copy())
        if kind == "other":
            wc.random_step(m, rng)
        F = m.F()
        ap = m.wb["ext_ask_price"].astype(np.int64)
        if repair:
            out = rp.market_repair(m, S)
            a, p = out["assigned"], out["price"]
        else:
            a, p, _, rel = m.warm(S)
        wc.check_feasible_injective(F, a)
        rp.check_held_eps_cs(F, ap, m.cap, S, p, a)
        opt = lsa_optimum(ap, m.cap.astype(np.int64), F, S)
        cost = wc.total_cost(a, ap * S, m.cap.astype(np.int64) * S + (S - 1))
        if S == 1:
            assert cost - opt <= T, (step, cost, opt)
        else:
            assert cost == opt, (step, cost, opt)
        m.store(p, a)


@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_warm_from_the_remapped_state_keeps_the_bound(seed, repair):
    splice_history(900 + seed, 12, repair=repair)


@pytest.mark.parametrize("seed", [4, 5])
def test_warm_from_the_remapped_state_is_exact_with_scale_t_plus_1(seed):
    splice_history(900 + seed, 10, S=15)


def test_warm_from_the_remapped_state_under_reputation_floors():
    splice_history(911, 10, floors=True)


def test_removed_holders_are_released_and_counted():
    m = SpliceMarket.__new__(SpliceMarket)
    m.__dict__.update(market(10, 50, 21).__dict__)
    a, p, _ = m.cold()
    m.store(p, a)
    held = np.flatnonzero(m.assigned != NONE)[:3]
    gone = m.assigned[held]
    m.splice(gone)
    assert np.all(m.assigned[held] == CUT) and np.all(exported(m.assigned)[held] == NONE)
    _, _, _, rel = m.warm()
    assert set(held.tolist()) <= set(rel.tolist())


# ------------------------------------------------------------------ the tail cases are the checker's shrink and grow
@pytest.mark.parametrize("seed", [6, 7, 8])
def test_tail_splices_are_shrink_and_grow(seed):
    rng = np.random.default_rng(seed)
    x = SpliceMarket.__new__(SpliceMarket)
    x.__dict__.update(market(12, 60, 930 + seed).__dict__)
    a, p, _ = x.cold()
    x.store(p, a)
    y = SpliceMarket.__new__(SpliceMarket)
    y.__dict__.update({k: (v.copy() if isinstance(v, (np.ndarray, set)) else v) for k, v in x.__dict__.items()})
    for step in range(8):
        W = x.n_workers
        if step % 2 == 0:
            n = int(rng.integers(1, 6))
            x.splice(np.arange(W - n, W)[::-1])
            y.resize(W - n)
        else:
            n = int(rng.integers(1, 6))
            src = rng.integers(0, W, n)
            x.splice((), np.full(n, W), x.wa[src].copy(), x.wb[src].copy())
            y.resize(W + n, y.wa[src].copy(), y.wb[src].copy())
        assert np.array_equal(x.wa, y.wa) and np.array_equal(x.wb, y.wb)
        assert x.n_kept == y.n_kept and x.rows == y.rows
        ax, px, nx, rx = x.warm()
        ay, py, ny, ry = y.warm()
        assert np.array_equal(ax, ay) and np.array_equal(px, py) and nx == ny and np.array_equal(rx, ry), step
        x.store(px, ax)
        y.store(py, ay)
