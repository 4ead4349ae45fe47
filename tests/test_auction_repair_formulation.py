"""The auction's warm repair (PM_AUCTION_WARM | PM_AUCTION_REPAIR, DESIGN 4) on the CPU: eps-complementary slackness
over the whole matrix after the raise, after every forward round and after every reverse round; every unowned worker at
price 0 at the end; within T of scipy's optimum (the optimum with cost_scale = T + 1) over random histories, also from
an eps-scaled stored pass without reverse rounds; the released set is the step-1 set and a subset of the warm start's;
no change, no release and no reverse round; the raise ignores row order and counts held asks only; the exact-integer
checker equals the numpy one."""
import numpy as np
import pytest

import auction_repair_checker as rp
import auction_reverse_checker as rc
import auction_warm_checker as wc
from test_auction_exact_checker import open_market
from test_auction_warm_formulation import market

NONE = wc.NONE


def forward_round(F, ask_price, cap, S, price, assigned, withdrawn, eps=1):
    """One synchronous forward round of auction_warm_checker.rounds, so that a test can look between rounds.
    Returns False when no ask was active."""
    act = np.flatnonzero((assigned == NONE) & ~withdrawn)
    if len(act) == 0:
        return False
    base = -(np.asarray(ask_price, dtype=np.int64) * S)
    outside = -((np.asarray(cap, dtype=np.int64) + 1) * S)
    V = np.where(F[act], (base - price)[None, :], wc.NEG)
    r = np.arange(len(act))
    w1 = V.argmax(axis=1)
    b1 = V[r, w1].copy()
    V[r, w1] = wc.NEG
    b2 = V.max(axis=1)
    out = (b1 == wc.NEG) | (b1 < outside[act])
    withdrawn[act[out]] = True
    bt, bw = act[~out], w1[~out]
    bp = price[bw] + (b1[~out] - np.maximum(b2[~out], outside[bt])) + eps
    order = np.lexsort((bt, -bp, bw))
    bt, bw, bp = bt[order], bw[order], bp[order]
    first = np.ones(len(bw), dtype=bool)
    first[1:] = bw[1:] != bw[:-1]
    bt, bw, bp = bt[first], bw[first], bp[first]
    for t, w, b in zip(bt, bw, bp):
        prev = np.flatnonzero(assigned == w)
        assigned[prev] = NONE
        assigned[t] = w
        price[w] = b
    return True


def check_every_step(m: wc.Market, S):
    """The repair pass step by step with eps-CS checked in between; the end state equals the checker's."""
    F, ap = m.F(), m.wb["ext_ask_price"]
    p, a, rel, rows = rp.release(m.price, m.assigned, m.n_workers, m.n_kept, m.changed_rows(), m.changed_asks())
    p = rp.raise_rows(F, ap, m.cap, S, p, a, rows)
    rp.check_held_eps_cs(F, ap, m.cap, S, p, a)
    withdrawn = np.zeros(len(a), dtype=bool)
    n_fwd = 0
    while forward_round(F, ap, m.cap, S, p, a, withdrawn):
        n_fwd += 1
        rp.check_held_eps_cs(F, ap, m.cap, S, p, a)
    rc.check_eps_cs(F, ap, m.cap, S, p, a, 1)
    a, p, n_rev, n_bids = rc.reverse(F, ap, m.cap, S, p, a, 1, check=True)
    want = rp.market_repair(m, S)
    assert np.array_equal(a, want["assigned"]) and np.array_equal(p, want["price"])
    assert (n_fwd, n_rev, n_bids) == (want["fwd"], want["rev"], want["bids"])
    return want


def check_sound(m: wc.Market, S, out):
    F, ap = m.F(), m.wb["ext_ask_price"]
    a, p = out["assigned"], out["price"]
    T, W = F.shape
    wc.check_feasible_injective(F, a)
    owned = np.zeros(W, dtype=bool)
    owned[a[a != NONE]] = True
    assert np.all(p[~owned] == 0) and np.all(p >= 0)
    opt = rc.optimum(F, ap, m.cap, S)
    got = wc.total_cost(a, ap, m.cap) * S
    if S == 1:
        assert opt <= got <= opt + T, (opt, got)
    else:
        assert got == opt, (opt, got)


def history(m: wc.Market, rng, S, steps, start="cold"):
    if start == "cold":
        a, p, _ = m.cold(S)
    else:   # an eps-scaled pass without reverse rounds: unowned workers left at inflated prices
        a, p, *_ = rc.scaled(m.F(), m.wb["ext_ask_price"], m.cap, S, 64, 4, reverse_rounds=False)
    m.store(p, a)
    for _ in range(steps):
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng)
        yield m
        out = rp.market_repair(m, S)
        m.store(out["price"], out["assigned"])


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("S_mode", ["unit", "exact"])
@pytest.mark.parametrize("start", ["cold", "scaled"])
def test_eps_cs_at_every_step_and_the_bound(seed, S_mode, start):
    T, W = 40, 150
    m = market(T, W, 50 + seed, floors=seed == 1)
    S = 1 if S_mode == "unit" else T + 1
    rng = np.random.default_rng(200 + seed)
    for m in history(m, rng, S, 8, start):
        out = check_every_step(m, S)
        check_sound(m, S, out)


@pytest.mark.parametrize("seed", range(3))
def test_released_set_is_step_1_and_inside_the_warm_release(seed):
    m = market(40, 150, 60 + seed, floors=seed == 2)
    rng = np.random.default_rng(300 + seed)
    n_released = 0
    for m in history(m, rng, 1, 10):
        F, ap = m.F(), m.wb["ext_ask_price"]
        out = rp.market_repair(m)
        _, a1, rel1, _ = rp.release(m.price, m.assigned, m.n_workers, m.n_kept, m.changed_rows(), m.changed_asks())
        assert np.array_equal(out["released"], rel1)
        assert np.array_equal(np.flatnonzero((m.assigned != NONE) & (a1 == NONE)), rel1)
        _, _, rel_warm, _ = wc.release(F, ap, 1, m.price, m.assigned, m.n_kept, m.changed_rows(), m.changed_asks())
        assert set(rel1.tolist()) <= set(rel_warm.tolist())
        n_released += len(rel1)
    assert n_released > 0


@pytest.mark.parametrize("seed", range(3))
def test_no_change_releases_nothing_and_runs_no_reverse_round(seed):
    m = market(50, 120, 20 + seed)
    a, p, _ = m.cold(1)
    m.store(p, a)
    out = rp.market_repair(m)
    assert len(out["released"]) == 0 and len(out["raised"]) == 0 and (out["rev"], out["bids"]) == (0, 0)
    assert np.array_equal(out["assigned"], a) and np.array_equal(out["price"], p)
    assert out["fwd"] == int((a == NONE).any())   # the unassigned asks withdraw again in round 1


def test_no_change_after_a_scaled_pass_returns_the_stranded_prices_to_0():
    m = market(60, 200, 31)
    a, p, *_ = rc.scaled(m.F(), m.wb["ext_ask_price"], m.cap, 1, 64, 4, reverse_rounds=False)
    owned = np.zeros(m.n_workers, dtype=bool)
    owned[a[a != NONE]] = True
    assert (p[~owned] > 0).any()
    m.store(p, a)
    out = rp.market_repair(m, check=True)
    assert len(out["released"]) == 0 and out["rev"] > 0
    check_sound(m, 1, out)


@pytest.mark.parametrize("seed", range(3))
def test_the_raise_ignores_row_order(seed):
    m = market(40, 150, 70 + seed)
    rng = np.random.default_rng(400 + seed)
    for m in history(m, rng, 1, 6):
        F, ap = m.F(), m.wb["ext_ask_price"]
        want = rp.market_repair(m)
        for _ in range(3):
            rows = rng.permutation(m.changed_rows()).tolist()
            out = rp.repair(F, ap, m.cap, 1, m.price, m.assigned, m.n_kept, rows, m.changed_asks())
            assert np.array_equal(out["assigned"], want["assigned"]) and np.array_equal(out["price"], want["price"])
            E = rp.Repair(len(m.asks), rp.ex.lists_from_matrix(F), ap, m.cap, 1)
            st = E.repair(m.price, m.assigned, m.n_kept, m.n_workers, rows, m.changed_asks())
            assert np.array_equal(E.assignment(), want["assigned"]) and np.array_equal(E.prices(m.n_workers), want["price"])
            assert (st["fwd"], st["rev"], st["bids"], st["released"]) == (want["fwd"], want["rev"], want["bids"],
                                                                        len(want["released"]))


@pytest.mark.parametrize("seed,S", [(1, 1), (2, 41), (3, 1), (4, 1)])
def test_exact_checker_equals_the_numpy_checker(seed, S):
    m = market(40, 150, 80 + seed, floors=seed == 3)
    rng = np.random.default_rng(500 + seed)
    for m in history(m, rng, S, 6, "scaled" if seed == 4 else "cold"):
        want = rp.market_repair(m, S)
        E = rp.Repair(len(m.asks), rp.ex.lists_from_matrix(m.F()), m.wb["ext_ask_price"], m.cap, S)
        st = E.repair(m.price, m.assigned, m.n_kept, m.n_workers, m.changed_rows(), m.changed_asks())
        assert np.array_equal(E.assignment(), want["assigned"]) and np.array_equal(E.prices(m.n_workers), want["price"])
        assert (st["fwd"], st["rev"], st["bids"], st["released"]) == (want["fwd"], want["rev"], want["bids"],
                                                                    len(want["released"]))


def test_only_held_asks_count_in_the_raise():
    """Ask 0 holds worker 0 (ask_price 10, price 0); ask 1 was released by a cap change, so it holds nothing; worker 1
    (ask_price 5) was rewritten.  Held asks only: beta = -5 - (-10) = 5, price 4.  Counting ask 1 at its outside
    option -(100 + 1) would give beta 96 and price 95."""
    t, cap = open_market(2, 2, np.array([10, 5], dtype=np.uint32), np.array([100, 100], dtype=np.uint32))
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    ap = t["wb"]["ext_ask_price"]
    price = np.zeros(2, dtype=np.int64)
    stored = np.array([0, 1], dtype=np.uint32)
    p, a, rel, rows = rp.release(price, stored, 2, 2, [1], [1])
    assert a.tolist() == [0, NONE] and rel.tolist() == [1] and rows.tolist() == [1]
    assert rp.raise_rows(F, ap, cap, 1, p, a, rows).tolist() == [0, 4]
    assert rp.raise_rows(F, ap, cap, 1, p, a, rows, held_only=False).tolist() == [0, 95]
    E = rp.Repair(2, rp.ex.lists_from_matrix(F), ap, cap, 1)
    st = E.repair(price, stored, 2, 2, [1], [1])
    out = rp.repair(F, ap, cap, 1, price, stored, 2, [1], [1], check=True)
    assert np.array_equal(E.assignment(), out["assigned"]) and np.array_equal(E.prices(2), out["price"])
    assert (st["fwd"], st["rev"], st["bids"]) == (out["fwd"], out["rev"], out["bids"])


def test_history_reaches_every_kind_of_change():
    m = market(40, 150, 7, floors=True)
    rng = np.random.default_rng(7)
    a, p, _ = m.cold(1)
    m.store(p, a)
    kinds = set()
    for _ in range(60):
        kinds.add(wc.random_step(m, rng))
        out = rp.market_repair(m)
        m.store(out["price"], out["assigned"])
    assert kinds == {"price", "flags", "spec", "resize", "caps", "floors", "toggle", "reputation"}
