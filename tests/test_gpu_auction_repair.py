"""PM_AUCTION_WARM | PM_AUCTION_REPAIR on the device: chains of repair passes over random table histories equal the
repair checker bit for bit (assignment, prices, forward rounds, reverse rounds and bids, warm, asks released), under
every PM_TUNE_AUCTION setting the warm tests iterate; repairs from an eps-scaled stored state; the cutoff and every call
that discards the stored state give the cold pass; refusals leave the stored state alone; both sides of the packed-key
switch with stored prices at the eps_start-sized top, against the exact-integer checker; scipy's optimum at
2000 x 2000 after a history; and a repair pass at the 100k x 1M size of BASELINE configs[2]."""
import time

import numpy as np
import pytest

import auction_exact as ex
import auction_repair_checker as rp
import auction_reverse_checker as rc
import auction_warm_checker as wc
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from test_auction_exact_checker import feasible, ladder
from test_gpu_auction_reverse import scipy_instance
from test_gpu_auction_warm import cfg3, engine, tables

pytestmark = pytest.mark.gpu

NONE = wc.NONE
AUC = abi.PM_MODE_AUCTION
WARM = AUC | abi.PM_AUCTION_WARM
REPAIR = WARM | abi.PM_AUCTION_REPAIR
TUNES = [1, 2, 8, 16, 32, 64, 128, 8 | 32, 64 | 32, 1 | 64, 128 | 32, 0x200, 0x100 | 16]   # test_gpu_auction_warm's
MAX_ROUNDS = 20000
RESULT_LAUNCHES = 2


def run(eng, T, mode=REPAIR):
    eng.match(mode)
    res = eng.fetch()
    got = np.full(T, NONE, dtype=np.uint32)
    for ask, members in res.groups():
        assert len(members) == 1
        got[ask] = members[0]
    price, warm, released = eng.auction_state()
    return got, price, res.stats, warm, released, eng.auction_reverse_stats()


def check_pass(eng, m, S, want_warm, cold=None):
    """One repair pass against the checker (want_warm), or the cold pass it falls back to (cold: that pass's
    (assignment, prices, rounds); default the eps = 1 checker)."""
    T = len(m.asks)
    got, price, st, warm, released, rs = run(eng, T)
    if want_warm:
        out = rp.market_repair(m, S)
        a, p = out["assigned"], out["price"]
        assert warm and released == len(out["released"])
        assert rs == (1, out["rev"], out["bids"])
        assert st["n_rounds"] == out["fwd"]
    else:
        a, p, n = m.cold(S) if cold is None else cold
        assert not warm and released == 0 and rs == (0, 0, 0)
        assert st["n_rounds"] == n
    assert np.array_equal(got, a)
    assert np.array_equal(price, p)
    m.store(p, a)
    return rs


def chain(t, cap, seed, steps, tune=0, S=1, floors=None, reputation=None, scaled=False):
    """A cold pass, then `steps` repair passes, each after one or two random changes.  scaled: the first pass is eps
    64 / 4 without reverse rounds (it strands unowned workers at inflated prices)."""
    m = wc.Market(t, cap, reputation, floors)
    eng = engine(t, cap, tune=tune, floors=floors, reputation=reputation, S=S)
    if scaled:
        eng.set_auction_params(cost_scale=S, eps_start=64, eps_div=4)
        a, p, n, *_ = rc.scaled(m.F(), t["wb"]["ext_ask_price"], cap, S, 64, 4, reverse_rounds=False)
        check_pass(eng, m, S, want_warm=False, cold=(a, p, n))
    else:
        check_pass(eng, m, S, want_warm=False)
    rng = np.random.default_rng(seed)
    n_released = n_rev = 0
    for _ in range(steps):
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng, eng=eng)
        n_rev += check_pass(eng, m, S, want_warm=True)[1]
        n_released += eng.auction_state()[2]
    eng.close()
    return n_released, n_rev


@pytest.mark.parametrize("n_asks,n_workers,seed", [(50, 700, 2), (300, 2500, 3), (64, 1025, 4)])
def test_repair_chain_matches_checker(n_asks, n_workers, seed):
    t, cap = tables(n_asks, n_workers, seed)
    n_released, n_rev = chain(t, cap, seed, 8)
    assert n_released > 0 and n_rev > 0


def test_repair_chain_with_reputation_floors_and_scale():
    t, cap = tables(120, 1500, 31)
    rng = np.random.default_rng(31)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 120).astype(np.uint32)
    chain(t, cap, 31, 8, floors=floors, reputation=rep)
    chain(t, cap, 32, 6, S=121)


@pytest.mark.parametrize("n_base,copies,n_workers,plo,phi,seed", [(12, 40, 3000, 10, 14, 5), (3, 200, 2500, 7, 9, 8)])
def test_repair_chain_identical_bidders_and_ties(n_base, copies, n_workers, plo, phi, seed):
    t, cap = tables(n_base, n_workers, seed, dup=(copies, plo, phi))
    chain(t, cap, seed, 6)


@pytest.mark.parametrize("tune", TUNES)
def test_repair_chain_every_shortcut_can_be_switched_off(tune):
    t, cap = tables(25, 6000, 7, dup=(20, 5, 120))
    chain(t, cap, 70 + tune, 4, tune=tune)


@pytest.mark.parametrize("tune", [0, 128])
@pytest.mark.parametrize("S", [1, 301])
def test_repair_from_an_eps_scaled_state(tune, S):
    t, cap = tables(300, 2500, 3)
    n_released, n_rev = chain(t, cap, 13, 4, tune=tune, S=S, scaled=True)
    assert n_rev > 0


def test_no_change_after_an_eps_scaled_pass():
    """Stored eps 64 / 4 without reverse rounds: a repair pass with nothing changed releases nothing and returns every
    stranded price to 0 through its reverse stage; within T of scipy's optimum."""
    t, cap = scipy_instance(60, 200, 1)
    T = len(cap)
    m = wc.Market(t, cap)
    eng = engine(t, cap)
    eng.set_auction_params(eps_start=64, eps_div=4)
    a, p, n, *_ = rc.scaled(m.F(), t["wb"]["ext_ask_price"], cap, 1, 64, 4, reverse_rounds=False)
    check_pass(eng, m, 1, want_warm=False, cold=(a, p, n))
    rs = check_pass(eng, m, 1, want_warm=True)
    assert eng.auction_state()[2] == 0 and rs[1] > 0
    F, ap = m.F(), t["wb"]["ext_ask_price"]
    opt = rc.optimum(F, ap, cap)
    assert opt <= wc.total_cost(m.assigned, ap, cap) <= opt + T
    rs = check_pass(eng, m, 1, want_warm=True)   # nothing stranded any more: no reverse round
    assert rs == (1, 0, 0)
    eng.close()


def test_cutoff_exceeded_runs_cold():
    t, cap = tables(64, 1025, 4)
    m = wc.Market(t, cap)
    eng = engine(t, cap, incr=5)
    check_pass(eng, m, 1, want_warm=False)
    rng = np.random.default_rng(4)
    wc.random_step(m, rng, n_rows=3, eng=eng, kinds=("price",))
    check_pass(eng, m, 1, want_warm=True)      # 3 rows: within the cutoff
    wc.random_step(m, rng, n_rows=10, eng=eng, kinds=("price",))
    assert m.n_changes() > 5
    check_pass(eng, m, 1, want_warm=False)     # 10 rows: the cold pass, equal to the cold checker on the current tables
    eng.close()


def test_discarding_calls_give_a_cold_pass():
    t, cap = tables(50, 700, 2)
    calls = [
        lambda e: (e.set_asks(t["asks"], t["opts"]), e.set_price_caps(cap)),
        lambda e: e.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"]),
        lambda e: e.set_workers(t["wa"], t["wb"]),
        lambda e: e.set_auction_params(),
        lambda e: e.set_shard(0, 0),
        lambda e: e.attach_comm(None),
    ]
    m = wc.Market(t, cap)
    eng = engine(t, cap)
    check_pass(eng, m, 1, want_warm=False)
    for call in calls:
        assert check_pass(eng, m, 1, want_warm=True) == (1, 0, 0)   # nothing changed: warm, nothing released or stranded
        call(eng)
        check_pass(eng, m, 1, want_warm=False)
    eng.close()


def test_refusals_leave_the_stored_state():
    t, cap = tables(50, 700, 2)
    m = wc.Market(t, cap)
    eng = engine(t, cap)
    check_pass(eng, m, 1, want_warm=False)
    wc.random_step(m, np.random.default_rng(2), n_rows=4, eng=eng, kinds=("price",))
    check_pass(eng, m, 1, want_warm=True)
    state, rs = eng.auction_state(), eng.auction_reverse_stats()

    def unchanged():
        after = eng.auction_state()
        assert np.array_equal(after[0], state[0]) and after[1:] == state[1:] and eng.auction_reverse_stats() == rs

    R = abi.PM_AUCTION_REPAIR
    for mode in (AUC | R, REPAIR | abi.PM_AUCTION_REVERSE, AUC | abi.PM_AUCTION_REVERSE | R,
                 abi.PM_MODE_FIRST_FIT | R, abi.PM_MODE_FIRST_FIT | abi.PM_AUCTION_WARM | R,
                 abi.PM_MODE_PROXIMITY | abi.PM_AUCTION_WARM | R, abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | R,
                 REPAIR | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_INCREMENTAL):
        with pytest.raises(PrimeMatchError) as exc:
            eng.match(mode)
        assert exc.value.status == abi.PM_E_INVALID, hex(mode)
        unchanged()
    for call in (eng.match_local, eng.match_finish):
        for mode in (abi.PM_MODE_FIRST_FIT | R, abi.PM_MODE_FIRST_FIT | abi.PM_AUCTION_WARM | R):
            with pytest.raises(PrimeMatchError) as exc:
                call(mode)
            assert exc.value.status == abi.PM_E_INVALID, hex(mode)
            unchanged()
    eng.set_ask_enabled([3], False)
    with pytest.raises(PrimeMatchError) as exc:
        eng.match(REPAIR)
    assert exc.value.status == abi.PM_E_UNSUPPORTED
    unchanged()
    eng.set_ask_enabled([3], True)
    m.toggle([3])
    check_pass(eng, m, 1, want_warm=True)      # the toggle counts as a change; the state was kept
    eng.set_shard(0, 350)                      # (discards the state)
    for _ in range(2):
        with pytest.raises(PrimeMatchError) as exc:
            eng.auction_state()
        assert exc.value.status == abi.PM_E_STATE
        with pytest.raises(PrimeMatchError) as exc:
            eng.match(REPAIR)
        assert exc.value.status == abi.PM_E_UNSUPPORTED
    eng.close()


# ---------------------------------------------------------------- the packed-key switch at the eps_start-sized top
def packed_ok(P, K, S, E):
    """pm_auction_decide_packed's rule, restated: every reachable cost below 2^40."""
    lim = 1 << 40
    return S < lim and E < lim and P + K + 2 < (lim - E) // S


def last_packed_eps(P, K, S):
    E = (1 << 40) - (P + K + 2) * S - 1
    while packed_ok(P, K, S, E + 1):
        E += 1
    while not packed_ok(P, K, S, E):
        E -= 1
    return E


PACKED_CASES = [([1, 2, 3, 5, 8], [100, 100, 90, 100]), ([0, 5, 1000, 1001, 1002], [1500, 1001, 1500, 2000])]


def packed_plan(ap, caps, E):
    """On the CPU: the stored pass (eps E, eps_div 2^20, no reverse rounds: every ask withdraws and the ladder's
    rungs end at E-sized prices), one rewritten row, the exact repair.  Both round counts bounded before any device
    runs it."""
    t, cap, rep, floors = ladder(ap, caps)
    W = len(t["wa"])
    F = ex.lists_from_matrix(feasible(t, cap, rep, floors))
    A = ex.Auction(len(cap), F, t["wb"]["ext_ask_price"], cap, 1)
    st = A.scaled(E, 1 << 20, reverse=False, max_rounds=MAX_ROUNDS)
    assert (A.assignment() == NONE).all() and (A.prices(W) >= E).sum() >= len(cap)
    B = rp.Repair(len(cap), F, t["wb"]["ext_ask_price"], cap, 1)
    rst = B.repair(A.prices(W), A.assignment(), W, W, [1], [], max_rounds=MAX_ROUNDS)
    assert st["fwd"] + rst["fwd"] + rst["rev"] < MAX_ROUNDS and rst["rev"] > 0
    return t, cap, rep, floors, A, st, B, rst


@pytest.mark.parametrize("case", range(len(PACKED_CASES)))
def test_packed_key_switch_with_stored_prices_at_the_top(case):
    ap, caps = PACKED_CASES[case]
    P, K = max(ap), max(caps)
    E = last_packed_eps(P, K, 1)
    for e, want_packed in ((E, True), (E + 1, False)):
        t, cap, rep, floors, A, st, B, rst = packed_plan(ap, caps, e)
        W = len(t["wa"])
        for tune in (0, 128):
            eng = engine(t, cap, tune=tune, reputation=rep, floors=floors)
            eng.set_auction_params(eps_start=e, eps_div=1 << 20)
            got, price, stats, warm, released, rs = run(eng, len(cap), AUC)
            assert np.array_equal(got, A.assignment()) and np.array_equal(price, A.prices(W))
            assert stats["n_rounds"] == st["fwd"]
            eng.update_workers(np.array([1], dtype=np.uint32), t["wa"][1:2], t["wb"][1:2])
            got, price, stats, warm, released, rs = run(eng, len(cap))
            eng.close()
            assert warm and released == rst["released"] and rs == (1, rst["rev"], rst["bids"])
            assert np.array_equal(got, B.assignment()) and np.array_equal(price, B.prices(W))
            assert stats["n_rounds"] == rst["fwd"]
            per_round = 6 if (want_packed and tune == 0) else 7   # the packed claim needs no pm_auction_claim
            assert stats["n_launches"] == per_round * stats["n_rounds"] + RESULT_LAUNCHES, (e, tune)


# ---------------------------------------------------------------- the bound
def test_2000_x_2000_within_T_of_scipy_after_a_history():
    t, cap = scipy_instance(2000, 2000, 4)
    T = len(cap)
    for S in (1, T + 1):
        m = wc.Market(t, cap)
        eng = engine(t, cap)
        eng.set_auction_params(cost_scale=S, eps_start=64, eps_div=4)
        eng.match(AUC | abi.PM_AUCTION_REVERSE)    # the stored state: a sound scaled pass
        rng = np.random.default_rng(S)
        for _ in range(3 if S == 1 else 1):
            for _ in range(2):
                wc.random_step(m, rng, eng=eng, kinds=("price", "flags", "spec", "resize", "caps", "floors"))
            got, price, st, warm, released, rs = run(eng, T)
            assert warm and rs[0] == 1
            F, ap = m.F(), m.wb["ext_ask_price"]
            wc.check_feasible_injective(F, got)
            owned = np.zeros(m.n_workers, dtype=bool)
            owned[got[got != NONE]] = True
            assert np.all(price[~owned] == 0) and np.all(price >= 0)
            opt = rc.optimum(F, ap, m.cap, S)
            cost = wc.total_cost(got, ap, m.cap) * S
            assert (opt <= cost <= opt + T) if S == 1 else (cost == opt), (S, opt, cost)
            m.store(price, got)
        eng.close()


def test_repair_pass_at_cfg3_size():
    """100k asks x 1M workers: one cold pass, 1 000 owned rows rewritten, one repair pass.  Injective, caps and
    requirements respected on a sample (the oracle's predicate), every unowned worker at price 0, and eps-complementary
    slackness on 300 sampled asks against every worker.  The time is printed, not asserted."""
    t, cap = cfg3()
    T, W = len(cap), len(t["wa"])
    eng = engine(t, cap)
    got, price, st, warm, _, _ = run(eng, T, AUC)
    assert not warm
    rng = np.random.default_rng(7)
    held = got[got != NONE]
    idx = np.sort(rng.choice(held, 1000, replace=False)).astype(np.uint32)
    a, b = t["wa"][idx].copy(), t["wb"][idx].copy()
    b["ext_ask_price"] = np.maximum(1, (b["ext_ask_price"] * rng.uniform(0.5, 1.5, len(idx))).astype(np.uint32))
    t["wa"][idx], t["wb"][idx] = a, b
    eng.update_workers(idx, a, b)
    t0 = time.perf_counter()
    got, price, st, warm, released, rs = run(eng, T)
    ms = (time.perf_counter() - t0) * 1e3
    print(f"\nrepair pass at 100k x 1M after 1000 owned rows: {ms:.1f} ms (with the fetch), released {released}, "
          f"forward rounds {st['n_rounds']}, reverse rounds {rs[1]}, reverse bids {rs[2]}")
    eng.close()
    assert warm and released == 1000 and rs[0] == 1
    ap = t["wb"]["ext_ask_price"].astype(np.int64)
    sold = np.flatnonzero(got != NONE)
    assert len(np.unique(got[sold])) == len(sold) and np.all(ap[got[sold]] <= cap[sold])
    owned = np.zeros(W, dtype=bool)
    owned[got[sold]] = True
    assert np.all(price[~owned] == 0) and np.all(price >= 0)
    value = -ap - price
    for tk in rng.choice(T, 300, replace=False):
        F = wc.feasible(t["wa"], t["wb"], t["asks"][tk:tk + 1], t["opts"], t["bits"], t["words"], cap[tk:tk + 1])[0]
        pi = value[got[tk]] if got[tk] != NONE else -(int(cap[tk]) + 1)
        if got[tk] != NONE:
            assert F[got[tk]]
        if F.any():
            assert value[F].max() <= pi + 1
