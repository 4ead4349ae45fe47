"""The auction certificate (auction_certificate.py, DESIGN 4) on the CPU: weak duality on random states (the bound never
exceeds scipy's optimum, which never exceeds the cost of a feasible assignment); the slack identity; the final states
of every sequential checker (cold, eps-scaled with reverse rounds, warm, repair) certify within T, and exactly optimal
with cost_scale = T + 1; and the eps-scaled pass without reverse rounds is flagged."""
import numpy as np
import pytest

import auction_certificate as ac
import auction_repair_checker as rp
import auction_reverse_checker as rc
import auction_warm_checker as wc
from test_auction_warm_formulation import market
from test_gpu_auction_reverse import scipy_instance

NONE = wc.NONE


def random_assignment(F, rng):
    """An injective assignment inside F: asks in random order take a random free feasible worker, or stay unheld."""
    T, W = F.shape
    a = np.full(T, NONE, dtype=np.uint32)
    free = np.ones(W, dtype=bool)
    for t in rng.permutation(T):
        ws = np.flatnonzero(F[t] & free)
        if len(ws) and rng.random() < 0.8:
            w = int(rng.choice(ws))
            a[t] = w
            free[w] = False
    return a


def cost_of(a, ap, cap, S):
    return sum(int(ap[a[t]]) * S if a[t] != NONE else (int(cap[t]) + 1) * S for t in range(len(a)))


@pytest.mark.parametrize("seed", range(4))
def test_weak_duality_on_random_states(seed):
    m = market(30, 120, 10 + seed, floors=seed % 2 == 1)
    F, ap = m.F(), m.wb["ext_ask_price"]
    rng = np.random.default_rng(seed)
    for S in (1, 31):
        opt = rc.optimum(F, ap, m.cap, S)
        for _ in range(6):
            hi = int(rng.choice([1, 50, 5000]))
            price = rng.integers(0, hi, m.n_workers).astype(np.int64)
            price[rng.random(m.n_workers) < 0.5] = 0
            a = random_assignment(F, rng)
            c = ac.certificate(F, ap, m.cap, S, price, a)
            assert c["bound"] <= opt <= c["cost"] == cost_of(a, ap, m.cap, S)
            assert c["gap"] >= c["cost"] - opt


@pytest.mark.parametrize("seed", range(4))
def test_gap_is_the_slack_plus_the_priced_unowned_sum(seed):
    m = market(30, 120, 20 + seed, floors=seed == 2)
    F, ap = m.F(), m.wb["ext_ask_price"]
    rng = np.random.default_rng(100 + seed)
    for _ in range(8):
        price = rng.integers(0, 400, m.n_workers).astype(np.int64) * (rng.random(m.n_workers) < 0.6)
        a = random_assignment(F, rng)
        S = int(rng.choice([1, 7, 31]))
        c = ac.certificate(F, ap, m.cap, S, price, a)
        assert c["n_shared"] == c["n_bad_holds"] == 0
        assert c["gap"] == sum(c["slack"]) + c["priced_unowned_sum"]
        assert c["n_held"] == int((a != NONE).sum()) and c["evals"] == F.size


def test_shared_and_bad_holds_are_counted():
    m = market(20, 80, 3)
    F, ap = m.F(), m.wb["ext_ask_price"]
    a = random_assignment(F, np.random.default_rng(3))
    held = np.flatnonzero(a != NONE)
    assert len(held) >= 3
    a[held[1]] = a[held[0]]                              # two asks on one worker
    bad = [w for w in range(m.n_workers) if not F[held[2], w]]
    a[held[2]] = bad[0]                                  # a hold the tables do not allow
    c = ac.certificate(F, ap, m.cap, 1, np.zeros(m.n_workers, dtype=np.int64), a)
    held = np.flatnonzero(a != NONE)
    assert c["n_shared"] == 1 and c["n_bad_holds"] == int((~F[held, a[held]]).sum()) >= 1


def check_final(F, ap, cap, S, price, a):
    T = F.shape[0]
    c = ac.certificate(F, ap, cap, S, price, a)
    assert (c["n_bad_holds"], c["n_shared"], c["n_priced_unowned"], c["n_slack_over"]) == (0, 0, 0, 0)
    assert c["max_slack"] <= 1 and 0 <= c["gap"] <= T
    assert c["gap"] == sum(c["slack"])
    if S == T + 1:
        opt = rc.optimum(F, ap, cap, S)
        assert c["cost"] == opt and c["gap"] < S
    return c


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("S_mode", ["unit", "exact"])
def test_final_states_of_the_cold_and_scaled_checkers(seed, S_mode):
    m = market(40, 150, 30 + seed, floors=seed == 1)
    T = len(m.asks)
    S = 1 if S_mode == "unit" else T + 1
    F, ap = m.F(), m.wb["ext_ask_price"]
    a, p, _ = m.cold(S)
    check_final(F, ap, m.cap, S, p, a)
    a, p, *_ = rc.scaled(F, ap, m.cap, S, 64, 4, reverse_rounds=True)
    check_final(F, ap, m.cap, S, p, a)


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("S_mode", ["unit", "exact"])
@pytest.mark.parametrize("kind", ["warm", "repair"])
def test_final_states_of_the_warm_and_repair_checkers(seed, S_mode, kind):
    m = market(40, 150, 40 + seed, floors=seed == 2)
    T = len(m.asks)
    S = 1 if S_mode == "unit" else T + 1
    a, p, _ = m.cold(S)
    m.store(p, a)
    rng = np.random.default_rng(600 + seed)
    for _ in range(6):
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng)
        if kind == "warm":
            a, p, _, _ = m.warm(S)
        else:
            out = rp.market_repair(m, S)
            a, p = out["assigned"], out["price"]
        check_final(m.F(), m.wb["ext_ask_price"], m.cap, S, p, a)
        m.store(p, a)


def test_the_scaled_pass_without_reverse_rounds_is_flagged():
    """test_oracle_auction.py's first scipy instance: eps 64 / 4 without reverse rounds ends 54 % above the optimum."""
    t, cap = scipy_instance(60, 200, 1)
    T = len(cap)
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    ap = t["wb"]["ext_ask_price"]
    a, p, *_ = rc.scaled(F, ap, cap, 1, 64, 4, reverse_rounds=False)
    c = ac.certificate(F, ap, cap, 1, p, a)
    opt = rc.optimum(F, ap, cap)
    assert c["cost"] > opt + T and c["bound"] <= opt
    assert c["n_priced_unowned"] > 0 and c["gap"] > T
    assert c["gap"] == sum(c["slack"]) + c["priced_unowned_sum"]
    a, p, *_ = rc.scaled(F, ap, cap, 1, 64, 4, reverse_rounds=True)
    check_final(F, ap, cap, 1, p, a)
