"""The exact-integer auction checker (auction_exact.py) against the numpy checkers and the oracle inside their int64-safe
range, against brute force at prices and caps near 2^32, and the integer domain the oracle and the engine share:
outside it the oracle refuses instead of answering, at its last admitted point it equals the exact checker."""
import itertools

import numpy as np
import pytest

import auction_exact as ex
import auction_reverse_checker as rc
import auction_warm_checker as wc
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth

NONE = ex.NONE
U32 = 0xFFFFFFFF


def tables(n_asks, n_workers, seed, dup=None):
    """The instance shapes of the device auction suites (test_gpu_auction_warm.tables)."""
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed)
    a = synth.make_asks(n_asks, "mixed", seed=synth.SEED_ASKS + seed)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)
    rng = np.random.default_rng(seed)
    wb = t["wb"].copy()
    if dup is None:
        wb["ext_ask_price"] = rng.integers(10, 1000, n_workers).astype(np.uint32)
        cap = rng.integers(50, 1500, n_asks).astype(np.uint32)
    else:             # duplicated asks over a narrow price range: every tie rule
        copies, plo, phi = dup
        idx = rng.permutation(np.repeat(np.arange(n_asks), copies))
        t["asks"] = np.ascontiguousarray(t["asks"][idx])
        wb["ext_ask_price"] = rng.integers(plo, phi + 1, n_workers).astype(np.uint32)
        cap = rng.integers(max(plo - 2, 0), phi + 3, len(idx)).astype(np.uint32)
    t["wb"] = wb
    return t, cap


def open_market(T, W, ask_price, cap, flags=abi.PM_W_HEALTHY | abi.PM_W_P2P):
    """T asks without requirements over W workers: every candidate is compatible with every ask."""
    a = np.zeros(W, dtype=abi.WORKER_A)
    b = np.zeros(W, dtype=abi.WORKER_B)
    a["flags"] = flags
    b["ext_ask_price"] = ask_price
    asks = np.zeros(T, dtype=abi.ASK)
    asks["min_group_size"] = asks["max_group_size"] = 1
    t = dict(asks=asks, opts=np.zeros(0, dtype=abi.GPU_OPT), wa=a, wb=b, bits=np.array([U32], dtype=np.uint32),
             n_patterns=0, n_models=0, words=1)
    return t, np.asarray(cap, dtype=np.uint32)


def feasible(t, cap, reputation=None, floors=None):
    return wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap, reputation, floors)


def exact(t, cap, S, F=None, reputation=None, floors=None):
    F = feasible(t, cap, reputation, floors) if F is None else F
    return ex.Auction(len(cap), ex.lists_from_matrix(F), t["wb"]["ext_ask_price"], cap, S)


def oracle(t, cap, S=1, eps_start=1, eps_div=4, reputation=None, floors=None):
    return orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap, cost_scale=S,
                           eps_start=eps_start, eps_div=eps_div, reputation=reputation, min_reputation=floors)


SHAPES = [(50, 700, 2, None), (64, 1025, 4, None), (300, 2500, 3, None), (12, 3000, 5, (40, 10, 14)),
          (3, 2500, 8, (200, 7, 9))]


# ---------------------------------------------------------------- equal to the existing checkers in their range
@pytest.mark.parametrize("T,W,seed,dup", SHAPES)
def test_cold_pass_equals_the_oracle_and_the_numpy_checker(T, W, seed, dup):
    t, cap = tables(T, W, seed, dup)
    W = len(t["wa"])
    F = feasible(t, cap)
    A = exact(t, cap, 1, F)
    st = A.scaled(max_rounds=20000)
    got, price = A.assignment(), A.prices(W)
    o_got, o_price, o_rounds = oracle(t, cap)
    assert np.array_equal(got, o_got) and np.array_equal(price, o_price) and st["fwd"] == o_rounds
    w_got, w_price, w_rounds = wc.cold(F, t["wb"]["ext_ask_price"], cap, 1)
    assert np.array_equal(got, w_got) and np.array_equal(price, w_price) and st["fwd"] == w_rounds


def test_cold_pass_with_the_exact_scale_and_reputation_floors_equals_the_oracle():
    t, cap = tables(50, 700, 2)
    A = exact(t, cap, 51)
    st = A.scaled(max_rounds=20000)
    o_got, o_price, o_rounds = oracle(t, cap, S=51)
    assert np.array_equal(A.assignment(), o_got) and np.array_equal(A.prices(700), o_price) and st["fwd"] == o_rounds
    t, cap = tables(120, 1500, 31)
    rng = np.random.default_rng(31)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 120).astype(np.uint32)
    A = exact(t, cap, 1, reputation=rep, floors=floors)
    st = A.scaled(max_rounds=20000)
    o_got, o_price, o_rounds = oracle(t, cap, reputation=rep, floors=floors)
    assert np.array_equal(A.assignment(), o_got) and np.array_equal(A.prices(1500), o_price) and st["fwd"] == o_rounds


SCALED = [((50, 700, 2, None), 1, 64, 4), ((50, 700, 2, None), 1, (1 << 41) + 12345, 16),
          ((60, 200, 1, None), 61, 64, 4), ((300, 2500, 3, None), 1, 16, 4),
          ((12, 3000, 5, (40, 10, 14)), 1, 64, 4), ((3, 2500, 8, (200, 7, 9)), 1, 1024, 8)]


@pytest.mark.parametrize("shape,S,eps_start,eps_div", SCALED)
def test_scaled_pass_equals_the_reverse_checker_and_the_oracle(shape, S, eps_start, eps_div):
    t, cap = tables(*shape[:3], dup=shape[3])
    W = len(t["wa"])
    F = feasible(t, cap)
    ap = t["wb"]["ext_ask_price"]
    for reverse in (True, False):
        A = exact(t, cap, S, F)
        st = A.scaled(eps_start, eps_div, reverse=reverse, max_rounds=20000)
        a, p, n_fwd, n_rev, bids, phases = rc.scaled(F, ap, cap, S, eps_start, eps_div, reverse_rounds=reverse)
        assert np.array_equal(A.assignment(), a) and np.array_equal(A.prices(W), p)
        assert (st["fwd"], st["rev"], st["bids"], st["phases"]) == (n_fwd, n_rev, bids, phases)
        if reverse:
            assert n_rev > 0 or eps_start == 1
        else:
            o_got, o_price, o_rounds = oracle(t, cap, S, eps_start, eps_div)
            assert np.array_equal(A.assignment(), o_got) and np.array_equal(A.prices(W), o_price) and st["fwd"] == o_rounds


def test_scaled_pass_with_reputation_floors_equals_the_reverse_checker():
    t, cap = tables(120, 1500, 31)
    rng = np.random.default_rng(31)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 120).astype(np.uint32)
    F = feasible(t, cap, rep, floors)
    A = exact(t, cap, 1, F)
    st = A.scaled(64, 2, reverse=True, max_rounds=20000)
    a, p, n_fwd, n_rev, bids, phases = rc.scaled(F, t["wb"]["ext_ask_price"], cap, 1, 64, 2)
    assert np.array_equal(A.assignment(), a) and np.array_equal(A.prices(1500), p)
    assert (st["fwd"], st["rev"], st["bids"], st["phases"]) == (n_fwd, n_rev, bids, phases)


def exact_warm(m: wc.Market, S=1):
    """The exact checker's warm pass over a warm-checker market (its tables and the changes since its stored state)."""
    A = ex.Auction(len(m.asks), ex.lists_from_matrix(m.F()), m.wb["ext_ask_price"], m.cap, S)
    st = A.warm(m.price, m.assigned, m.n_kept, m.n_workers, m.changed_rows(), m.changed_asks())
    return A.assignment(), A.prices(m.n_workers), st["fwd"], st["released"]


@pytest.mark.parametrize("shape,S,seed", [((50, 700, 2, None), 1, 2), ((64, 1025, 4, None), 1, 4),
                                          ((50, 700, 2, None), 51, 9), ((12, 3000, 5, (40, 10, 14)), 1, 5)])
def test_warm_chain_equals_the_warm_checker(shape, S, seed):
    t, cap = tables(*shape[:3], dup=shape[3])
    m = wc.Market(t, cap)
    a, p, _ = m.cold(S)
    m.store(p, a)
    rng = np.random.default_rng(seed)
    n_released = 0
    for _ in range(6):
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng)
        got, price, rounds, released = exact_warm(m, S)
        a, p, n, rel = m.warm(S)
        assert np.array_equal(got, a) and np.array_equal(price, p) and rounds == n and released == len(rel)
        n_released += released
        m.store(p, a)
    assert n_released > 0


def test_warm_release_of_an_eps_scaled_reverse_pass_equals_the_warm_checker():
    """The stored state of a scaled pass (unowned workers at price 0 after reverse rounds; without them, inflated
    prices that the release resets)."""
    t, cap = tables(50, 700, 2)
    for reverse in (True, False):
        m = wc.Market(t, cap)
        a, p, *_ = rc.scaled(m.F(), t["wb"]["ext_ask_price"], cap, 1, 64, 4, reverse_rounds=reverse)
        m.store(p, a)
        rng = np.random.default_rng(3)
        for _ in range(3):
            wc.random_step(m, rng)
            got, price, rounds, released = exact_warm(m)
            a, p, n, rel = m.warm(1)
            assert np.array_equal(got, a) and np.array_equal(price, p) and rounds == n and released == len(rel)
            m.store(p, a)


# ---------------------------------------------------------------- anchors at extreme values
def brute_force_cost(F, ask_price, cap, S):
    """Minimum over injective partial assignments inside F of sum(ask_price * S held, (cap + 1) * S unheld)."""
    T, W = F.shape
    best = None
    for ws in itertools.product([None, *range(W)], repeat=T):
        held = [w for w in ws if w is not None]
        if len(set(held)) != len(held) or any(w is not None and not F[t, w] for t, w in enumerate(ws)):
            continue
        c = sum((int(ask_price[w]) if w is not None else int(cap[t]) + 1) * S for t, w in enumerate(ws))
        best = c if best is None else min(best, c)
    return best


EDGE_PRICES = [
    [U32, U32 - 1, U32 - 2, U32 - 5, U32 - 3],                     # the top of u32
    [0x7FFFFFFF, 0x80000000, 0x80000001, 0x7FFFFFFE, 0x80000002],  # across 2^31
    [0, 1, U32, 0x80000000, 2],                                    # both ends
]
EDGE_CAPS = [
    [U32, U32 - 1, U32 - 4, U32],
    [0x80000000, 0x7FFFFFFF, 0x80000001, 0x80000002],
    [1, U32, 0, 0x80000000],
]


@pytest.mark.parametrize("case", range(len(EDGE_PRICES)))
@pytest.mark.parametrize("seed", range(3))
def test_extreme_prices_and_caps_reach_the_brute_force_optimum(case, seed):
    """Prices and caps near 2^31 and 2^32 (cap + 1 = 2^32 must not wrap), cost_scale = T + 1: the optimum, and the
    oracle (inside the domain) equals the checker."""
    rng = np.random.default_rng(seed)
    ap = rng.permutation(np.array(EDGE_PRICES[case], dtype=np.uint32))
    cap = rng.permutation(np.array(EDGE_CAPS[case], dtype=np.uint32))
    T, W = len(cap), len(ap)
    t, cap = open_market(T, W, ap, cap)
    S = T + 1
    F = feasible(t, cap)
    A = exact(t, cap, S, F)
    st = A.scaled(max_rounds=5000)
    assert A.total_cost() == brute_force_cost(F, ap, cap, S)
    o_got, o_price, o_rounds = oracle(t, cap, S)
    assert np.array_equal(A.assignment(), o_got) and np.array_equal(A.prices(W), o_price) and st["fwd"] == o_rounds
    A2 = exact(t, cap, S, F)
    A2.scaled(1 << 36, 64, reverse=True, max_rounds=5000)
    assert A2.total_cost() == A.total_cost()


# ---------------------------------------------------------------- the domain
def ladder(ask_price, cap, extra_price=None):
    """One ask per rung: workers in ascending ask_price carry reputation 0, 1, 2, ...; ask t has floor t, so its
    feasible workers are w >= t within its cap and its first choice is w_t — no two asks contend in the first round,
    and there is no price war however large the scale.  extra_price: one more row, not a candidate (no ask takes it),
    that still counts for P."""
    ap = list(ask_price) + ([] if extra_price is None else [extra_price])
    W, T = len(ap), len(cap)
    t, cap = open_market(T, W, np.array(ap, dtype=np.uint32), cap)
    if extra_price is not None:
        t["wa"]["flags"][W - 1] = 0
    rep = np.arange(W, dtype=np.uint32)
    floors = np.arange(T, dtype=np.uint32)
    return t, cap, rep, floors


def probe1():
    """3 identical asks without requirements, 4 workers priced 2^31 .. 2^31 + 3, every cap 0xFFFFFFFF."""
    return open_market(3, 4, (1 << 31) + np.arange(4), np.full(3, U32))


def test_probe_beyond_int64_safety_is_refused_and_the_exact_answer_sells_every_ask():
    t, cap = probe1()
    S = 1 << 30
    assert not ex.in_domain((1 << 31) + 3, U32, S, 1)
    with pytest.raises(ValueError):
        oracle(t, cap, S)
    A = exact(t, cap, S)
    A.scaled(S, 4, reverse=True, max_rounds=1000)   # (eps-scaled: at eps = 1 alone the three asks fight O(S) rounds)
    assert (A.assignment() != NONE).all()       # each value, about -2^61, is above the outside option, -2^62
    assert A.total_cost() == brute_force_cost(feasible(t, cap), t["wb"]["ext_ask_price"], cap, S)


def test_eps_start_beyond_the_domain_is_refused_at_once():
    t, cap = open_market(3, 4, 10 + np.arange(4), np.full(3, 100))
    for eps in ((1 << 63) + 1, 1 << 62, 1 << 61, (1 << 61) - 115):
        with pytest.raises(ValueError):
            oracle(t, cap, 1, eps, 1 << 30)
    E = (1 << 61) - 1 - 115                      # (P + K + 2) * S + E = 2^61 - 1: admitted
    A = exact(t, cap, 1)
    st = A.scaled(E, 1 << 30, max_rounds=2000)
    got, price, rounds = oracle(t, cap, 1, E, 1 << 30)
    assert np.array_equal(A.assignment(), got) and np.array_equal(A.prices(4), price) and st["fwd"] == rounds


def test_a_price_war_stops_at_the_round_limit():
    """Three asks over two equal workers at a large scale: the eps = 1 war takes O(S) rounds, the checker stops."""
    t, cap = open_market(3, 2, [7, 7], [9, 9, 9])
    A = exact(t, cap, 1 << 20)
    with pytest.raises(ex.RoundLimit):
        A.scaled(max_rounds=1000)


def last_admitted_scale(P, K, E=1):
    return ((1 << 61) - 1 - E) // (P + K + 2)


# (worker prices ascending, caps, P = the largest price of any row): the cheapest rung against the largest cap puts a
# value right above -2^61 - (P + 1) * S, the outside option at -(K + 1) * S
DOMAIN_CASES = [
    ([1, 2, (1 << 31) + 3], [U32, U32 - 1, U32], (1 << 31) + 3),
    ([0, 0x7FFFFFFF, 0x80000000, U32 - 1], [U32, 0x80000000, U32, U32 - 1], U32),
    ([5, 6, 1000], [1500, 1499, 1500], 2000),
    ([0, 1, 2], [3, 3, 2], U32),
]


@pytest.mark.parametrize("case", range(len(DOMAIN_CASES)))
def test_last_admitted_scale_equals_the_exact_checker_and_one_more_is_refused(case):
    """The oracle at the largest admitted scale equals the exact checker bit for bit and reaches the optimum; one step
    further it refuses."""
    ap, caps, P = DOMAIN_CASES[case]
    t, cap, rep, floors = ladder(ap, caps, extra_price=P)
    K = max(caps)
    W = len(t["wa"])
    S = last_admitted_scale(P, K)
    assert ex.in_domain(P, K, S, 1) and not ex.in_domain(P, K, S + 1, 1)
    F = feasible(t, cap, rep, floors)
    A = exact(t, cap, S, F)
    st = A.scaled(max_rounds=200)
    got, price, rounds = oracle(t, cap, S, reputation=rep, floors=floors)
    assert np.array_equal(A.assignment(), got) and np.array_equal(A.prices(W), price) and st["fwd"] == rounds
    assert A.total_cost() == brute_force_cost(F, t["wb"]["ext_ask_price"], cap, S)
    with pytest.raises(ValueError):
        oracle(t, cap, S + 1, reputation=rep, floors=floors)


@pytest.mark.parametrize("case", range(len(DOMAIN_CASES)))
def test_last_admitted_eps_start_equals_the_exact_checker(case):
    ap, caps, P = DOMAIN_CASES[case]
    t, cap, rep, floors = ladder(ap, caps, extra_price=P)
    K, S = max(caps), len(caps) + 1
    W = len(t["wa"])
    E = (1 << 61) - 1 - (P + K + 2) * S
    assert ex.in_domain(P, K, S, E) and not ex.in_domain(P, K, S, E + 1)
    A = exact(t, cap, S, feasible(t, cap, rep, floors))
    st = A.scaled(E, 1 << 20, max_rounds=2000)
    got, price, rounds = oracle(t, cap, S, E, 1 << 20, reputation=rep, floors=floors)
    assert np.array_equal(A.assignment(), got) and np.array_equal(A.prices(W), price) and st["fwd"] == rounds
    with pytest.raises(ValueError):
        oracle(t, cap, S, E + 1, 1 << 20, reputation=rep, floors=floors)
