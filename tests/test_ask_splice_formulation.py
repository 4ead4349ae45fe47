"""Removing and inserting asks anywhere in the table (pm_remove_asks / pm_insert_asks) restated on the CPU.

Part 1 extends the Incremental mirror of test_ask_deltas_formulation.  Every stored first ask f moves with its row:
f - (removed rows below f) + (rows inserted before a position <= f).  A removed f lands on the next kept row (its
"heir"), or NONE when no row is kept after it.  The heir is listed in D with the replaced bit whatever its own state,
so the removed ask's workers are walked again from the heir itself.  Listing it in E alone is not enough: the E-pass
skips the ask a worker already stores.  Inserted rows are in E, like appended ones.  Over random histories of removals,
insertions, replacements, appends, shrinks, toggles and written rows, the stored first ask equals a from-scratch
recomputation, and the traps a wrong rule falls into are pinned one by one.

Part 2 extends AskMarket the same way.  Kept asks keep their workers under their new indices.  A removed ask's worker
becomes unowned at its stored price, and inserted asks hold nothing and join A0.  Warm and repair passes from the
remapped state end within T of scipy's optimum and keep eps-CS over the held asks.  The lemma the full-size GPU test
relies on is proved here: while no pass crosses the cutoff, a warm or repair pass from the remapped state equals the
same pass after pm_set_asks of the current rows and a restore of the remapped export, in assignment, prices and rounds.
"""
import numpy as np
import pytest

import auction_repair_checker as rp
import auction_restore_checker as rc
import auction_warm_checker as wc
from test_ask_deltas_formulation import NONE, AskMarket, Incremental, first_ask, optimum, rand_rows, small_tables


# ================================================================== part 1: the incremental rule
def _rename(s, new):
    return {int(new[t]) for t in s if new[t] >= 0}


class Splice(Incremental):
    """Incremental with remove / insert; `heirs` are the kept rows the workers of a removed ask landed on."""

    def full(self):
        super().full()
        self.heirs = set()

    def remove(self, idx):
        T = len(self.F)
        rm = np.unique(np.asarray(idx, dtype=np.int64))
        keep = np.setdiff1d(np.arange(T), rm)
        new = np.full(T, -1, np.int64)
        new[keep] = np.arange(len(keep))
        heirs = set()
        for t in rm:
            s = int(np.searchsorted(keep, t))            # the next kept row's new index
            if (self.eval_on[t] or int(t) in self.heirs) and s < len(keep):
                heirs.add(s)
        f = self.stored.astype(np.int64)
        g = f - np.searchsorted(rm, f, side="left")
        self.stored = np.where((f == NONE) | (g >= len(keep)), NONE, g).astype(np.uint32)
        self.F, self.on, self.eval_on = self.F[keep], self.on[keep], self.eval_on[keep]
        self.touched = _rename(self.touched, new) | heirs
        self.replaced = _rename(self.replaced, new)
        self.heirs = _rename(self.heirs, new) | heirs

    def shrink(self, n):
        super().shrink(n)
        self.heirs = {t for t in self.heirs if t < n}   # the marks go with their rows, as every per-ask column does

    def insert(self, before, rows):
        T = len(self.F)
        before = np.asarray(before, dtype=np.int64)
        assert np.all(np.diff(before) >= 0) and np.all(before <= T)
        new = np.arange(T) + np.searchsorted(before, np.arange(T), side="right")
        at = before + np.arange(len(before))
        self.F = np.insert(self.F, before, rows, axis=0)
        self.on = np.insert(self.on, before, True)
        self.eval_on = np.insert(self.eval_on, before, False)
        f = self.stored.astype(np.int64)
        self.stored = np.where(f == NONE, NONE, f + np.searchsorted(before, f, side="right")).astype(np.uint32)
        self.touched = _rename(self.touched, new) | {int(a) for a in at}
        self.replaced = _rename(self.replaced, new)
        self.heirs = _rename(self.heirs, new)
        return at

    def lists(self, as_disable=False, heirs_in_d=True):
        E, D = [], []
        for t in sorted(self.touched):
            heir = heirs_in_d and t in self.heirs
            if t in self.replaced:
                if self.on[t]:
                    E.append(t)
                if self.eval_on[t] or heir:
                    D.append((t, True))
            else:
                if self.on[t] and not self.eval_on[t]:
                    E.append(t)
                if heir:
                    D.append((t, True))
                elif self.eval_on[t] and not self.on[t]:
                    D.append((t, False))
        return E, D

    def run(self, heirs_in_d=True):
        real = self.lists
        self.lists = lambda as_disable=False: real(heirs_in_d=heirs_in_d)
        try:
            out = super().run()
        finally:
            self.lists = real
        self.heirs = set()
        return out


def check(inc, what=""):
    want = first_ask(inc.F, inc.on)
    got = inc.run()
    assert np.array_equal(got, want), what


def wrong_and_right(F, on, steps):
    """The pass after `steps` with the heir listed in E only (wrong) and in D (right)."""
    out = []
    for heirs_in_d in (False, True):
        x = Splice(F, on)
        steps(x)
        out.append(x.run(heirs_in_d=heirs_in_d).copy())
        assert heirs_in_d or not np.array_equal(out[0], first_ask(x.F, x.on)), "the wrong rule should fail here"
        if heirs_in_d:
            assert np.array_equal(out[1], first_ask(x.F, x.on))
    return out


def test_trap_the_heir_is_in_e():
    """Worker 0 stores ask 1; ask 2 was disabled at the evaluation and is enabled since (in E), and rejects it; ask 1
    is removed.  The worker now stores new index 1 (ask 2): the E-pass skips it, so only the walk from the heir moves
    it on to ask 3."""
    F = np.zeros((4, 1), bool)
    F[1, 0] = F[3, 0] = True
    on = np.array([True, True, False, True])

    def steps(x):
        x.toggle([2], [True])
        x.remove([1])

    wrong, right = wrong_and_right(F, on, steps)
    assert wrong.tolist() == [1] and right.tolist() == [2]


def test_trap_the_heir_was_appended_since_the_evaluation():
    """The heir was appended after the evaluation (eval_on 0), so a rule that lists only rows enabled at the
    evaluation in D misses it; the heir rejects the worker, the row appended after it accepts it."""
    F = np.zeros((2, 1), bool)
    F[1, 0] = True

    def steps(x):
        x.append(np.array([[False]]))
        x.append(np.array([[True]]))
        x.remove([1])

    wrong, right = wrong_and_right(F, np.ones(2, bool), steps)
    assert wrong.tolist() == [1] and right.tolist() == [2]


def test_trap_the_heir_was_disabled_or_replaced():
    F = np.zeros((4, 2), bool)
    F[1] = True
    F[2, 0] = True
    F[3] = True
    inc = Splice(F, np.ones(4, bool))
    assert inc.stored.tolist() == [1, 1]
    inc.toggle([2], [False])                      # the heir is disabled: its own workers walk on from it
    inc.remove([1])
    check(inc, "disabled heir")
    assert inc.stored.tolist() == [2, 2]
    inc = Splice(F, np.ones(4, bool))
    inc.replace([2], [np.array([False, True])])   # the heir is replaced by a row that accepts worker 1 only
    inc.remove([1])
    check(inc, "replaced heir")
    assert inc.stored.tolist() == [2, 1]


def test_trap_the_whole_tail_is_removed():
    F = np.zeros((5, 3), bool)
    F[2, 0] = F[4, 1] = F[0, 2] = True
    inc = Splice(F, np.ones(5, bool))
    inc.remove([4, 2, 3, 2])                       # any order, a repeated index once
    assert inc.stored.tolist() == [NONE, NONE, 0]
    check(inc)


def test_trap_an_ask_toggled_off_then_removed():
    F = np.zeros((4, 2), bool)
    F[1] = F[3] = True
    F[2, 1] = True
    inc = Splice(F, np.ones(4, bool))
    inc.toggle([1], [False])
    inc.remove([1])
    check(inc)
    assert inc.stored.tolist() == [2, 1]


def test_trap_a_row_inserted_just_before_a_workers_first_ask():
    F = np.zeros((3, 2), bool)
    F[2] = True
    inc = Splice(F, np.ones(3, bool))
    at = inc.insert([2, 2], np.array([[False, True], [True, True]]))
    assert at.tolist() == [2, 3] and inc.stored.tolist() == [4, 4]
    check(inc)
    assert inc.stored.tolist() == [3, 2]


def test_trap_a_removal_chain_before_the_pass():
    """The heir of a removed ask is removed in turn: its heir inherits the walk."""
    F = np.zeros((5, 1), bool)
    F[1, 0] = F[4, 0] = True
    inc = Splice(F, np.ones(5, bool))
    inc.append(np.array([[False]]))
    inc.remove([1])                                # heir: old 2
    inc.remove([1])                                # old 2 goes too: heir old 3, which rejects; old 4 accepts
    check(inc)
    assert inc.stored.tolist() == [2]


def test_removing_the_tail_is_a_shrink_and_appending_is_inserting_at_the_end():
    rng = np.random.default_rng(5)
    F, on = rand_rows(rng, 20, 50), rng.random(20) < 0.8
    a, b = Splice(F, on), Splice(F, on)
    a.toggle([3, 17], [True, False])
    b.toggle([3, 17], [True, False])
    a.remove(range(14, 20))
    b.shrink(14)
    assert np.array_equal(a.stored, b.stored) and a.lists() == b.lists()
    rows = rand_rows(rng, 3, 50)
    a.insert([14, 14, 14], rows)
    b.append(rows)
    assert np.array_equal(a.stored, b.stored) and a.lists() == b.lists()
    assert np.array_equal(a.run(), b.run())


def test_a_shrink_drops_the_heirs_past_the_new_end():
    """A heir cut off by a shrink goes with its row: a row appended later at its index is no heir (the engine moves
    its marks with the rows, orph_mark included)."""
    F = np.zeros((5, 1), bool)
    F[2, 0] = True
    inc = Splice(F, np.ones(5, bool))
    inc.remove([2])                                 # heir: old 3, new index 2
    assert inc.heirs == {2}
    inc.shrink(2)
    assert inc.heirs == set()
    inc.append(np.array([[True]]))
    assert inc.lists() == ([2], [])
    check(inc)
    assert inc.stored.tolist() == [2]


def test_insert_takes_one_row_per_position():
    from protocol_b200 import abi
    from protocol_b200.engine import _insert_args

    rows = np.zeros(2, dtype=abi.ASK)
    with pytest.raises(ValueError):
        _insert_args([0, 1, 1], rows, None)
    before, asks, opts = _insert_args([0, 1], rows, None)
    assert len(before) == len(asks) == 2 and len(opts) == 0


@pytest.mark.parametrize("seed", range(16))
def test_random_histories(seed):
    rng = np.random.default_rng(1000 + seed)
    T, W = int(rng.integers(5, 40)), int(rng.integers(20, 120))
    inc = Splice(rand_rows(rng, T, W), rng.random(T) < 0.8)
    kinds = set()
    for step in range(25):
        for _ in range(int(rng.integers(1, 4))):
            T = len(inc.F)
            kind = str(rng.choice(["remove", "insert", "replace", "append", "shrink", "toggle", "write"]))
            if kind == "remove" and T > 2:
                inc.remove(rng.integers(0, T, int(rng.integers(1, min(5, T)))))
            elif kind == "insert":
                k = int(rng.integers(1, 4))
                inc.insert(np.sort(rng.integers(0, T + 1, k)), rand_rows(rng, k, W))
            elif kind == "replace" and T:
                k = int(rng.integers(1, 4))
                inc.replace(rng.integers(0, T, k), rand_rows(rng, k, W))
            elif kind == "append":
                inc.append(rand_rows(rng, int(rng.integers(1, 4)), W))
            elif kind == "shrink" and T > 1:
                inc.shrink(T - int(rng.integers(1, min(4, T))))
            elif kind == "toggle" and T:
                k = int(rng.integers(1, 4))
                inc.toggle(rng.integers(0, T, k), rng.random(k) < 0.5)
            elif kind == "write":
                inc.write(int(rng.integers(0, W)), rng.random(len(inc.F)) < 0.1)
            kinds.add(kind)
        check(inc, f"seed {seed} step {step}")
    assert {"remove", "insert"} <= kinds


# ================================================================== part 2: the auction from the remapped state
class SpliceMarket(AskMarket):
    """AskMarket with remove / insert, remapped as the engine remaps its stored state."""

    def remove(self, idx, eng=None):
        T = len(self.asks)
        rm = np.unique(np.asarray(idx, dtype=np.int64))
        keep = np.setdiff1d(np.arange(T), rm)
        new = np.full(T, -1, np.int64)
        new[keep] = np.arange(len(keep))
        if self.assigned is not None:
            gone = self.assigned[rm]
            self.removed_held += int(((gone != NONE) & (gone < self.n_kept)).sum())
            self.assigned = self.assigned[keep].copy()
        self.asks, self.cap, self.cap0, self.floors0 = self.asks[keep].copy(), self.cap[keep].copy(), self.cap0[keep], self.floors0[keep]
        if self.floors is not None:
            self.floors = self.floors[keep].copy()
        self.toggled = _rename(self.toggled, new)
        if eng is not None:
            eng.remove_asks(np.asarray(idx, dtype=np.uint32))

    def insert(self, before, rows, eng=None):
        from test_ask_deltas_formulation import own_options

        T = len(self.asks)
        before = np.asarray(before, dtype=np.int64)
        new = np.arange(T) + np.searchsorted(before, np.arange(T), side="right")
        at = before + np.arange(len(before))
        self.asks = np.insert(self.asks, before, rows)
        z = np.zeros(len(before), np.uint32)
        self.cap, self.cap0 = np.insert(self.cap, before, z), np.insert(self.cap0, before, z)
        if self.floors is not None:
            self.floors = np.insert(self.floors, before, z)
        self.floors0 = np.insert(self.floors0, before, z)
        if self.assigned is not None:
            self.assigned = np.insert(self.assigned, before, np.full(len(before), NONE, np.uint32))
        self.toggled = _rename(self.toggled, new) | {int(a) for a in at}
        if eng is not None:
            eng.insert_asks(before.astype(np.uint32), *own_options(rows, self.opts))
        return at


def splice_step(m: SpliceMarket, pool, rng, eng=None, held_only=False):
    """Remove 1-3 asks at scattered positions (held ones with held_only) or insert 1-3 rows at random priorities, with
    caps for the inserted rows."""
    T = len(m.asks)
    if rng.random() < 0.5 and T > 6:
        cand = np.flatnonzero(m.assigned != NONE) if held_only and m.assigned is not None else np.arange(T)
        cand = cand if len(cand) else np.arange(T)
        m.remove(rng.choice(cand, min(len(cand), int(rng.integers(1, 4))), replace=False), eng)
        return "remove"
    k = int(rng.integers(1, 4))
    at = m.insert(np.sort(rng.integers(0, T + 1, k)), pool[rng.integers(0, len(pool), k)], eng)
    cap = m.cap.copy()
    cap[at] = rng.integers(50, 1500, k)
    m.set_caps(cap, eng)
    return "insert"


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
def test_auction_from_the_remapped_state(seed, repair):
    t, cap, pool = small_tables(seed)
    m = SpliceMarket(t, cap)
    a, p, _ = m.cold()
    m.store(p, a)
    rng = np.random.default_rng(200 + seed)
    for step in range(6):
        for _ in range(int(rng.integers(1, 3))):
            splice_step(m, pool, rng)
        F, ap = m.F(), m.wb["ext_ask_price"]
        if repair:
            p1, a1, _, rows = rp.release(m.price, m.assigned, m.n_workers, m.n_kept, m.changed_rows(), m.changed_asks())
            p1 = rp.raise_rows(F, ap, m.cap, 1, p1, a1, rows)
            rp.check_held_eps_cs(F, ap, m.cap, 1, p1, a1)
            out = rp.market_repair(m, check=True)
            a, p = out["assigned"], out["price"]
        else:
            p1, a1, _, _ = wc.release(F, ap, 1, m.price, m.assigned, m.n_kept, m.changed_rows(), m.changed_asks())
            rp.check_held_eps_cs(F, ap, m.cap, 1, p1, a1)
            a, p, _, _ = m.warm()
        wc.check_feasible_injective(F, a)
        assert 0 <= wc.total_cost(a, ap, m.cap) - optimum(F, ap, m.cap) <= len(m.asks), f"seed {seed} step {step}"
        m.store(p, a)


def restored_twin(m: SpliceMarket):
    """The route without the splice calls: a market on the current rows and caps (pm_set_asks + caps), its stored
    state the audited restore of m's remapped export."""
    t = dict(asks=m.asks, opts=m.opts, wa=m.wa, wb=m.wb, bits=m.bits, words=m.words)
    r = wc.Market(t, m.cap, m.reputation, m.floors)
    kept = rc.market_audit(r, 1, m.price, m.assigned)["assigned"]
    r.store(m.price, kept)
    return r, kept


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
def test_lemma_remapped_state_equals_a_restore_of_its_export(seed, repair):
    t, cap, pool = small_tables(seed, T=30, W=80)
    m = SpliceMarket(t, cap)
    a, p, _ = m.cold()
    m.store(p, a)
    rng = np.random.default_rng(300 + seed)
    for step in range(5):
        for _ in range(int(rng.integers(1, 3))):
            splice_step(m, pool, rng, held_only=True)
        r, kept = restored_twin(m)
        assert np.array_equal(kept, m.assigned), "the audit keeps every remapped hold"
        if repair:
            x, y = rp.market_repair(m), rp.market_repair(r)
            got, want = (x["assigned"], x["price"], x["fwd"], x["rev"]), (y["assigned"], y["price"], y["fwd"], y["rev"])
        else:
            got, want = m.warm()[:3], r.warm()[:3]
        for g, w in zip(got, want):
            assert np.array_equal(g, w), f"seed {seed} step {step}"
        m.store(got[1], got[0])


def test_removed_asks_free_their_workers_and_inserted_ones_hold_nothing():
    t, cap, pool = small_tables(3)
    m = SpliceMarket(t, cap)
    a, p, _ = m.cold()
    m.store(p, a)
    idx = np.array([2, 9, 15, 20])
    held = int((a[idx] != NONE).sum())
    m.remove(idx)
    assert m.removed_held == held and m.n_changes() == held
    assert not set(a[idx][a[idx] != NONE].tolist()) & set(m.assigned.tolist())
    assert np.array_equal(m.assigned, np.delete(a, idx))
    at = m.insert([0, 5, 5], pool[:3])
    assert (m.assigned[at] == NONE).all() and set(at.tolist()) <= set(m.changed_asks())
