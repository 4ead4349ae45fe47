"""The auction's reverse rounds (PM_AUCTION_REVERSE, DESIGN 4) on the CPU: the reverse checker's phases without the
reverse stage equal orc_soa_auction; with eps_start = 1 the stage has no bidders; with it, every eps-scaled pass is
feasible, injective, leaves every unowned worker at price 0, keeps eps-complementary slackness over the whole matrix,
and is within T of scipy's optimum (equal to it with cost_scale = T + 1) — on the instance where scaling without the
stage ends 54 % above the optimum too, and with one bidder at a time as well as synchronously."""
import numpy as np
import pytest

import auction_reverse_checker as rc
import auction_warm_checker as wc
from oracle import pm_oracle as orc
from protocol_b200 import synth

NONE = wc.NONE


def scipy_instance(T, W, seed):
    """test_oracle_auction.py's instances: loguniform worker prices, caps between 20 and 1200."""
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed, price="loguniform")
    a = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS + seed)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, words=words)
    cap = np.exp(np.log(20) + synth._unit(synth.SEED_EXT + seed, T, 3) * np.log(60)).astype(np.uint32)
    return t, cap


def random_instance(T, W, seed, dup=False):
    """synth tables with uniform prices and caps; dup: few distinct asks over a narrow price range (ties everywhere)."""
    t, _ = scipy_instance(T, W, seed)
    rng = np.random.default_rng(seed)
    wb = t["wb"].copy()
    if dup:
        t["asks"] = np.ascontiguousarray(t["asks"][rng.integers(0, 4, T)])
        wb["ext_ask_price"] = rng.integers(5, 9, W)
        cap = rng.integers(3, 11, T).astype(np.uint32)
    else:
        wb["ext_ask_price"] = rng.integers(10, 1000, W)
        cap = rng.integers(50, 1500, T).astype(np.uint32)
    t["wb"] = wb
    return t, cap


def F_of(t, cap):
    return wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)


def check_sound(F, ap, cap, out, S):
    a, price = out[0], out[1]
    T, W = F.shape
    wc.check_feasible_injective(F, a)
    owned = np.zeros(W, dtype=bool)
    owned[a[a != NONE]] = True
    assert np.all(price[~owned] == 0) and np.all(price >= 0)
    rc.check_eps_cs(F, ap, cap, S, price, a, 1)
    opt = rc.optimum(F, ap, cap, S)
    got = wc.total_cost(a, ap, cap) * S
    assert opt <= got <= opt + T * 1, (opt, got)
    return got, opt


@pytest.mark.parametrize("eps_start,eps_div", [(4, 2), (64, 4), (1024, 8), (1 << 20, 4)])
@pytest.mark.parametrize("T,W,seed", [(60, 200, 1), (300, 2000, 2), (500, 300, 3)])
def test_checker_without_the_stage_is_the_oracle(T, W, seed, eps_start, eps_div):
    t, cap = scipy_instance(T, W, seed)
    out = rc.scaled(F_of(t, cap), t["wb"]["ext_ask_price"], cap, 1, eps_start, eps_div, reverse_rounds=False)
    a, p, n = orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap, cost_scale=1,
                              eps_start=eps_start, eps_div=eps_div)
    assert np.array_equal(out[0], a) and np.array_equal(out[1], p) and out[2] == n
    assert out[3:] == (0, 0, out[5])


@pytest.mark.parametrize("seed", range(4))
def test_eps_start_1_has_no_bidders(seed):
    t, cap = random_instance(200, 900, 40 + seed, dup=seed % 2 == 1)
    F, ap = F_of(t, cap), t["wb"]["ext_ask_price"]
    with_stage = rc.scaled(F, ap, cap, 1, 1, 4)
    without = rc.scaled(F, ap, cap, 1, 1, 4, reverse_rounds=False)
    assert with_stage[3:] == (0, 0, 1)
    assert np.array_equal(with_stage[0], without[0]) and np.array_equal(with_stage[1], without[1])


def test_the_54_percent_instance():
    t, cap = scipy_instance(60, 200, 1)
    F, ap = F_of(t, cap), t["wb"]["ext_ask_price"]
    T = len(cap)
    opt = rc.optimum(F, ap, cap)
    forward_only = rc.scaled(F, ap, cap, 1, 64, 4, reverse_rounds=False)
    assert wc.total_cost(forward_only[0], ap, cap) > 1.5 * opt     # what the stage repairs
    out = rc.scaled(F, ap, cap, 1, 64, 4, check=True)
    assert out[3] > 0 and out[4] > 0 and out[5] == 4
    check_sound(F, ap, cap, out, 1)
    out = rc.scaled(F, ap, cap, T + 1, 64, 4, check=True)
    got, opt_s = check_sound(F, ap, cap, out, T + 1)
    assert got == opt_s


@pytest.mark.parametrize("eps_div", [2, 4, 8])
@pytest.mark.parametrize("eps_start", [4, 64, 1 << 20])
@pytest.mark.parametrize("seed,dup", [(11, False), (12, True), (13, False)])
def test_scaled_passes_are_sound(seed, dup, eps_start, eps_div):
    t, cap = random_instance(120, 400, seed, dup=dup)
    F, ap = F_of(t, cap), t["wb"]["ext_ask_price"]
    T = len(cap)
    check_sound(F, ap, cap, rc.scaled(F, ap, cap, 1, eps_start, eps_div, check=True), 1)
    got, opt = check_sound(F, ap, cap, rc.scaled(F, ap, cap, T + 1, eps_start, eps_div), T + 1)
    assert got == opt


@pytest.mark.parametrize("T,W,seed", [(60, 200, 1), (300, 2000, 2), (500, 300, 3)])
def test_scipy_instances_are_sound(T, W, seed):
    t, cap = scipy_instance(T, W, seed)
    F, ap = F_of(t, cap), t["wb"]["ext_ask_price"]
    check_sound(F, ap, cap, rc.scaled(F, ap, cap, 1, 64, 4), 1)
    got, opt = check_sound(F, ap, cap, rc.scaled(F, ap, cap, T + 1, 64, 4), T + 1)
    assert got == opt


@pytest.mark.parametrize("seed,dup", [(1, None), (21, False), (22, True)])
def test_one_bidder_at_a_time_meets_the_bound(seed, dup):
    """Gauss-Seidel: every bid sees the ones before it.  The bound holds all the same: it rests on eps-CS and on the
    unowned workers' prices, not on the synchronous order."""
    t, cap = scipy_instance(60, 200, 1) if dup is None else random_instance(150, 500, seed, dup=dup)
    F, ap = F_of(t, cap), t["wb"]["ext_ask_price"]
    T = len(cap)
    check_sound(F, ap, cap, rc.scaled(F, ap, cap, 1, 64, 4, gauss_seidel=True), 1)
    got, opt = check_sound(F, ap, cap, rc.scaled(F, ap, cap, T + 1, 64, 4, gauss_seidel=True), T + 1)
    assert got == opt


def test_a_round_reads_the_state_at_its_start():
    """Two workers stranded at positive prices, both best for the same ask: one round, both bid on it, the ask takes
    the higher profit; the loser bids again in the next round against the new profit."""
    F = np.ones((1, 2), dtype=bool)
    ap = np.array([3, 5], dtype=np.uint32)
    cap = np.array([10], dtype=np.uint32)
    price = np.array([4, 4], dtype=np.int64)
    a, p, n, bids = rc.reverse(F, ap, cap, 1, price, np.full(1, NONE, dtype=np.uint32), 1, check=True)
    # round 1: pi = -11; gains 8 and 6, no second value: both offer at 0; profits -3 and -5: worker 0 wins.
    # round 2: pi = -3; worker 1's gain -2 <= eps: its price goes to 0.
    assert a.tolist() == [0] and p.tolist() == [0, 0] and (n, bids) == (2, 3)
