"""Ask-table deltas (pm_update_asks / pm_resize_asks) restated on the CPU.

Part 1 restates the incremental rule of PM_INCREMENTAL in numpy, over a feasibility matrix: a replaced row counts as
disabled and enabled again (in E when it is enabled now, in D when it was enabled at the stored evaluation, its
orphans walked from the ask itself), appended rows are in E, and a shrink sets every stored first ask past the new end
to NONE.  Over random histories of replaced, appended and removed asks mixed with toggles and written worker rows, the
stored first ask equals a from-scratch recomputation; the traps a wrong rule falls into are pinned one by one.

Part 2 pins the auction rule through the existing checkers: the warm start and the warm repair run from the stored
state remapped to the new table (kept asks keep their workers, a removed ask's worker becomes unowned at its stored
price, A0 = replaced + appended + cap or floor changes), and their results are within T * eps of the optimum
scipy.optimize.linear_sum_assignment finds; eps-complementary slackness holds over the held asks after the release.
AskMarket (below) is that remapped market; the GPU tests drive the engine through it.
"""
import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

import auction_repair_checker as rp
import auction_warm_checker as wc

NONE = 0xFFFFFFFF


# ================================================================== part 1: the incremental rule
def first_ask(F, on):
    """The first enabled feasible ask of every worker (F: bool[T, W]), or NONE."""
    G = F & on[:, None]
    hit = G.any(axis=0)
    return np.where(hit, G.argmax(axis=0), NONE).astype(np.uint32)


class Incremental:
    """The engine's bookkeeping between two evaluations, and the incremental pass that consumes it."""

    def __init__(self, F, on):
        self.F, self.on = F.copy(), on.copy()
        self.full()

    def full(self):
        self.stored = first_ask(self.F, self.on)
        self.eval_on = self.on.copy()
        self.touched, self.replaced, self.rows = set(), set(), set()

    # ---- the table calls
    def replace(self, idx, rows):
        for t, r in zip(idx, rows):          # the last entry of an index decides
            self.F[t] = r
            self.touched.add(int(t))
            self.replaced.add(int(t))

    def append(self, rows):
        T = len(self.F)
        self.F = np.concatenate([self.F, rows])
        self.on = np.concatenate([self.on, np.ones(len(rows), bool)])
        self.eval_on = np.concatenate([self.eval_on, np.zeros(len(rows), bool)])
        self.touched |= set(range(T, T + len(rows)))

    def shrink(self, n):
        self.F, self.on, self.eval_on = self.F[:n], self.on[:n], self.eval_on[:n]
        self.stored = np.where((self.stored != NONE) & (self.stored >= n), NONE, self.stored).astype(np.uint32)
        self.touched = {t for t in self.touched if t < n}
        self.replaced = {t for t in self.replaced if t < n}

    def toggle(self, idx, enabled):
        for t, e in zip(idx, enabled):
            self.on[t] = e
            self.touched.add(int(t))

    def write(self, w, col):
        self.F[:, w] = col
        self.rows.add(int(w))

    # ---- the pass
    def lists(self, as_disable=False):
        """E (asks) and D ((ask, walk its orphans from the ask itself)).  as_disable: the wrong rule that treats a
        replaced row that stays enabled as a disabled ask alone (orphans from the ask after it, no E-pass)."""
        E, D = [], []
        for t in sorted(self.touched):
            if t in self.replaced and as_disable and self.on[t] and self.eval_on[t]:
                D.append((t, False))
            elif t in self.replaced:
                if self.on[t]:
                    E.append(t)
                if self.eval_on[t]:
                    D.append((t, True))
            elif self.on[t] and not self.eval_on[t]:
                E.append(t)
            elif self.eval_on[t] and not self.on[t]:
                D.append((t, False))
        return E, D

    def run(self, orphan_from_next=False):
        """The incremental pass; orphan_from_next uses the wrong rule of lists(as_disable=True)."""
        E, D = self.lists(as_disable=orphan_from_next)
        G = self.F & self.on[:, None]
        f = self.stored.copy()
        start = {}
        for w in self.rows:                  # written rows: reset, walked over every ask
            f[w] = NONE
            start[w] = 0
        dmap = dict(D)
        for w in range(len(f)):              # orphans
            if f[w] != NONE and int(f[w]) in dmap and w not in start:
                t = int(f[w])
                start[w] = t if dmap[t] else t + 1
                f[w] = NONE
        self.n_tiles = len(start)            # rows walked in full: the written rows and the orphans
        for w, s in start.items():
            hit = np.flatnonzero(G[s:, w])
            f[w] = s + hit[0] if len(hit) else NONE
        for t in E:                          # the E-pass: min(f, first feasible ask of E)
            for w in np.flatnonzero(G[t]):
                if f[w] == NONE or t < f[w]:
                    f[w] = t
        self.stored = f.astype(np.uint32)
        self.eval_on = self.on.copy()
        self.touched, self.replaced, self.rows = set(), set(), set()
        return self.stored


def rand_rows(rng, k, W, p=0.08):
    return rng.random((k, W)) < p


def check(inc, what=""):
    """The pass equals a recomputation; its E, D and walked rows are those engine_history's mirror plans."""
    import engine_history as eh

    E, D = inc.lists()
    en, dis = eh.split_toggles(inc.on, inc.eval_on, inc.replaced)
    assert (set(E), {t for t, _ in D}) == (en, dis), what
    assert all(from_ask == (t in inc.replaced) for t, from_ask in D), what
    n_tiles = eh.walked_rows(inc.stored, inc.rows, dis)
    want = first_ask(inc.F, inc.on)
    got = inc.run()
    assert np.array_equal(got, want), what
    assert inc.n_tiles == n_tiles, (what, inc.n_tiles, n_tiles)


def test_trap_orphan_the_replaced_row_still_accepts():
    F = np.zeros((4, 3), bool)
    F[1, 0] = F[3, 0] = True
    inc = Incremental(F, np.ones(4, bool))
    assert inc.stored[0] == 1
    row = F[1].copy()                        # the new row 1 still accepts worker 0
    for wrong in (True, False):
        x = Incremental(F, np.ones(4, bool))
        x.replace([1], [row])
        got = x.run(orphan_from_next=wrong)
        assert (got[0] == 3) if wrong else (got[0] == 1)   # a walk from t + 1 loses it


def test_trap_a_worker_beyond_the_replaced_row_now_meets_it():
    F = np.zeros((4, 2), bool)
    F[3, 0] = True
    inc = Incremental(F, np.ones(4, bool))
    row = np.array([True, True])
    inc.replace([1], [row])
    check(inc)
    assert inc.stored.tolist() == [1, 1]


def test_trap_a_disabled_ask_that_is_replaced():
    F = np.zeros((3, 2), bool)
    F[2] = True
    on = np.array([True, False, True])
    inc = Incremental(F, on)
    inc.replace([1], [np.array([True, True])])
    check(inc, "replaced while disabled: still absent")
    assert inc.stored.tolist() == [2, 2]
    inc.toggle([1], [True])
    check(inc, "then enabled")
    assert inc.stored.tolist() == [1, 1]


def test_trap_a_replace_followed_by_a_disable():
    F = np.zeros((3, 2), bool)
    F[1] = F[2] = True
    inc = Incremental(F, np.ones(3, bool))
    inc.replace([1], [np.array([True, False])])
    inc.toggle([1], [False])
    check(inc)
    assert inc.stored.tolist() == [2, 2]


def test_trap_an_append_and_a_shrink_in_one_step():
    F = np.zeros((4, 3), bool)
    F[3, 0] = F[2, 1] = True
    inc = Incremental(F, np.ones(4, bool))
    inc.shrink(2)
    inc.append(np.array([[True, False, True], [False, True, False]]))
    check(inc)
    assert inc.stored.tolist() == [2, 3, 2]


def test_trap_a_shrink_below_a_workers_first_ask():
    F = np.zeros((5, 2), bool)
    F[4, 0] = F[1, 1] = True
    inc = Incremental(F, np.ones(5, bool))
    inc.shrink(3)
    check(inc)
    assert inc.stored.tolist() == [NONE, 1]


@pytest.mark.parametrize("seed", range(12))
def test_random_histories(seed):
    rng = np.random.default_rng(seed)
    T, W = int(rng.integers(5, 40)), int(rng.integers(20, 120))
    inc = Incremental(rand_rows(rng, T, W), rng.random(T) < 0.8)
    for step in range(25):
        for _ in range(int(rng.integers(1, 4))):
            T = len(inc.F)
            kind = rng.choice(["replace", "append", "shrink", "toggle", "write", "replace_held"])
            if kind == "replace" and T:
                k = int(rng.integers(1, 4))
                inc.replace(rng.integers(0, T, k), rand_rows(rng, k, W))
            elif kind == "replace_held" and T:   # a held row replaced by a row that keeps some of its workers
                t = int(rng.integers(0, T))
                inc.replace([t], [inc.F[t] & (rng.random(W) < 0.5)])
            elif kind == "append":
                inc.append(rand_rows(rng, int(rng.integers(1, 4)), W))
            elif kind == "shrink" and T > 1:
                inc.shrink(T - int(rng.integers(1, min(4, T))))
            elif kind == "toggle" and T:
                k = int(rng.integers(1, 4))
                inc.toggle(rng.integers(0, T, k), rng.random(k) < 0.5)
            elif kind == "write":
                w = int(rng.integers(0, W))
                inc.write(w, rng.random(len(inc.F)) < 0.1)
        check(inc, f"seed {seed} step {step}")


# ================================================================== part 2: the auction from the remapped state
def own_options(src, opts):
    """Rows `src` (opt_off into `opts`) with only their own option rows, each row's range after the last, as a caller
    that sends a new task's row sends it."""
    rows = np.ascontiguousarray(src).copy()
    rows["opt_off"] = np.concatenate([[0], np.cumsum(rows["n_opts"])[:-1]]).astype(np.uint32)
    own = np.concatenate([opts[o:o + k] for o, k in zip(src["opt_off"], src["n_opts"])] or [opts[:0]])
    return rows, np.ascontiguousarray(own)


class AskMarket(wc.Market):
    """A warm-checker market whose ask table changes in place: the stored state is remapped as the engine remaps it.
    Kept asks keep their workers; a removed ask's worker becomes unowned at its stored price (removed_held counts the
    kept rows that freed); replaced and appended asks join A0 (toggled); appended asks have cap 0 and floor 0."""

    def __init__(self, t, cap, reputation=None, floors=None):
        super().__init__(t, cap, reputation, floors)
        self.asks = np.ascontiguousarray(t["asks"]).copy()

    def store(self, price, assigned):
        super().store(price, assigned)
        self.removed_held = 0

    def n_changes(self):
        return super().n_changes() + self.removed_held

    def replace(self, idx, rows, eng=None):
        idx = np.atleast_1d(np.asarray(idx, dtype=np.uint32))
        for t, r in zip(idx, rows):
            self.asks[t] = r
        self.toggled |= {int(t) for t in idx}
        if eng is not None:   # the caller sends the new rows with their own option rows only
            eng.update_asks(idx, *own_options(rows, self.opts))

    def append(self, rows, eng=None):
        T, k = len(self.asks), len(rows)
        self.asks = np.concatenate([self.asks, rows])
        self.cap = np.concatenate([self.cap, np.zeros(k, np.uint32)])
        self.cap0 = np.concatenate([self.cap0, np.zeros(k, np.uint32)])
        if self.floors is not None:
            self.floors = np.concatenate([self.floors, np.zeros(k, np.uint32)])
        self.floors0 = np.concatenate([self.floors0, np.zeros(k, np.uint32)])
        if self.assigned is not None:
            self.assigned = np.concatenate([self.assigned, np.full(k, NONE, np.uint32)])
        self.toggled |= set(range(T, T + k))
        if eng is not None:
            eng.resize_asks(T + k, *own_options(rows, self.opts))

    def shrink(self, n, eng=None):
        if self.assigned is not None:
            gone = self.assigned[n:]
            self.removed_held += int(((gone != NONE) & (gone < self.n_kept)).sum())
            self.assigned = self.assigned[:n].copy()
        self.asks, self.cap, self.cap0, self.floors0 = self.asks[:n].copy(), self.cap[:n].copy(), self.cap0[:n], self.floors0[:n]
        if self.floors is not None:
            self.floors = self.floors[:n].copy()
        self.toggled = {t for t in self.toggled if t < n}
        if eng is not None:
            eng.resize_asks(n)


def ask_step(m: AskMarket, pool, rng, eng=None, kinds=("replace", "append", "shrink", "caps", "rows")):
    """One random ask-side change (or a worker-side one from auction_warm_checker.random_step)."""
    T = len(m.asks)
    kind = kinds[rng.integers(len(kinds))]
    if kind == "replace":
        k = int(rng.integers(1, 4))
        m.replace(rng.integers(0, T, k).astype(np.uint32), pool[rng.integers(0, len(pool), k)], eng)
    elif kind == "append":
        k = int(rng.integers(1, 5))
        m.append(pool[rng.integers(0, len(pool), k)], eng)
        cap = m.cap.copy()
        cap[T:] = rng.integers(50, 1500, k)
        m.set_caps(cap, eng)
    elif kind == "shrink" and T > 3:
        m.shrink(T - int(rng.integers(1, 3)), eng)
    elif kind == "caps":
        wc.random_step(m, rng, eng=eng, kinds=("caps",))
    else:
        wc.random_step(m, rng, eng=eng, kinds=("price", "flags", "spec"))
    return kind


def optimum(F, ask_price, cap):
    """The least total cost (each ask a feasible worker at its ask_price, or cap + 1 alone), by linear_sum_assignment."""
    T, W = F.shape
    big = 1 << 40
    C = np.full((T, W + T), big, dtype=np.int64)
    C[:, :W] = np.where(F, np.asarray(ask_price, np.int64)[None, :], big)
    C[np.arange(T), W + np.arange(T)] = np.asarray(cap, np.int64) + 1
    r, c = linear_sum_assignment(C)
    return int(C[r, c].sum())


def small_tables(seed, T=24, W=60):
    from protocol_b200 import synth
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed)
    a = synth.make_asks(T + 40, "mixed", seed=synth.SEED_ASKS + seed)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    rng = np.random.default_rng(seed)
    wb = w.b.copy()
    wb["ext_ask_price"] = rng.integers(10, 1000, W).astype(np.uint32)
    t = dict(asks=a.asks[:T], opts=a.opts, wa=w.a, wb=wb, bits=bits, n_patterns=npat, n_models=nmod, words=words)
    return t, rng.integers(50, 1500, T).astype(np.uint32), a.asks


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("repair", [False, True], ids=["warm", "repair"])
def test_auction_from_the_remapped_state(seed, repair):
    t, cap, pool = small_tables(seed)
    m = AskMarket(t, cap)
    a, p, _ = m.cold()
    m.store(p, a)
    rng = np.random.default_rng(100 + seed)
    for step in range(6):
        for _ in range(int(rng.integers(1, 3))):
            ask_step(m, pool, rng)
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
        T = len(m.asks)
        assert 0 <= wc.total_cost(a, ap, m.cap) - optimum(F, ap, m.cap) <= T, f"seed {seed} step {step}"
        m.store(p, a)


def test_removed_asks_free_their_workers():
    t, cap, pool = small_tables(3)
    m = AskMarket(t, cap)
    a, p, _ = m.cold()
    m.store(p, a)
    held = int((a[len(a) - 5:] != NONE).sum())
    m.shrink(len(a) - 5)
    assert m.removed_held == held and m.n_changes() == held
    freed = set(a[len(a) - 5:][a[len(a) - 5:] != NONE].tolist())
    assert not freed & set(m.assigned.tolist())
