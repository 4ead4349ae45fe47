"""PM_AUCTION_REVERSE on the device: eps-scaled passes equal the reverse checker bit for bit (assignment, prices,
forward and reverse rounds, bids, phases) under every PM_TUNE_AUCTION setting; eps_start = 1 equals the pass without
the bit; the result is within T of scipy's optimum; a warm pass may start from the stored state; refusals; and a
scaled pass at the 100k x 1M size of BASELINE configs[2]."""
import numpy as np
import pytest

import auction_reverse_checker as rc
import auction_warm_checker as wc
from protocol_b200 import abi, synth
from protocol_b200._lib import PrimeMatchError
from test_gpu_auction_warm import cfg3, engine, tables

pytestmark = pytest.mark.gpu

NONE = wc.NONE
REV = abi.PM_MODE_AUCTION | abi.PM_AUCTION_REVERSE
TUNES = [0, 2, 8, 64, 128, 0x100 | 16]


def scipy_instance(T, W, seed):
    """test_oracle_auction.py's scipy instances (the first, 60 x 200 seed 1, ends 54 % above the optimum when
    eps-scaled without reverse rounds)."""
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed, price="loguniform")
    a = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS + seed)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)
    cap = np.exp(np.log(20) + synth._unit(synth.SEED_EXT + seed, T, 3) * np.log(60)).astype(np.uint32)
    return t, cap


def run(eng, T, S, eps_start, eps_div, mode=REV):
    eng.set_auction_params(cost_scale=S, eps_start=eps_start, eps_div=eps_div)
    eng.match(mode)
    res = eng.fetch()
    got = np.full(T, NONE, dtype=np.uint32)
    for ask, members in res.groups():
        assert len(members) == 1
        got[ask] = members[0]
    price, warm, _ = eng.auction_state()
    assert not warm
    return got, price, res.stats, eng.auction_reverse_stats()


def check(t, cap, S, eps_start, eps_div, tune=0, floors=None, reputation=None):
    T = len(cap)
    eng = engine(t, cap, tune=tune, floors=floors, reputation=reputation)
    got, price, st, (phases, n_rev, bids) = run(eng, T, S, eps_start, eps_div)
    eng.close()
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap, reputation, floors)
    a, p, n_fwd, want_rev, want_bids, want_phases = rc.scaled(F, t["wb"]["ext_ask_price"], cap, S, eps_start, eps_div)
    assert np.array_equal(got, a)
    assert np.array_equal(price, p)
    assert (st["n_rounds"], n_rev, bids, phases) == (n_fwd, want_rev, want_bids, want_phases)
    return F, got, n_rev


@pytest.mark.parametrize("tune", TUNES)
def test_the_54_percent_instance_matches_the_checker_and_the_bound(tune):
    t, cap = scipy_instance(60, 200, 1)
    T = len(cap)
    ap = t["wb"]["ext_ask_price"]
    F, got, n_rev = check(t, cap, 1, 64, 4, tune=tune)
    assert n_rev > 0
    opt = rc.optimum(F, ap, cap)
    assert opt <= wc.total_cost(got, ap, cap) <= opt + T
    F, got, _ = check(t, cap, T + 1, 64, 4, tune=tune)
    assert wc.total_cost(got, ap, cap) == opt


@pytest.mark.parametrize("tune", TUNES)
def test_300_x_2500_eps_16_div_4(tune):
    t, cap = tables(300, 2500, 3)
    check(t, cap, 1, 16, 4, tune=tune)


@pytest.mark.parametrize("tune", TUNES)
@pytest.mark.parametrize("n_base,copies,n_workers,plo,phi,seed", [(12, 40, 3000, 10, 14, 5), (3, 200, 2500, 7, 9, 8)])
def test_identical_bidders_and_ties(tune, n_base, copies, n_workers, plo, phi, seed):
    t, cap = tables(n_base, n_workers, seed, dup=(copies, plo, phi))
    check(t, cap, 1, 64, 4, tune=tune)
    check(t, cap, 1, 1024, 8, tune=tune)


@pytest.mark.parametrize("tune", TUNES)
def test_reputation_floors(tune):
    t, cap = tables(120, 1500, 31)
    rng = np.random.default_rng(31)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 120).astype(np.uint32)
    check(t, cap, 1, 64, 2, tune=tune, floors=floors, reputation=rep)


@pytest.mark.parametrize("tune", TUNES)
def test_first_eps_beyond_2_to_40_takes_the_unpacked_path(tune):
    t, cap = tables(50, 700, 2)
    check(t, cap, 1, (1 << 41) + 12345, 16, tune=tune)


@pytest.mark.parametrize("tune", [0, 128])
def test_eps_start_1_equals_the_pass_without_the_bit(tune):
    t, cap = tables(300, 2500, 9)
    T = len(cap)
    eng = engine(t, cap, tune=tune)
    a0, p0, st0, rs0 = run(eng, T, 1, 1, 4, mode=abi.PM_MODE_AUCTION)
    a1, p1, st1, rs1 = run(eng, T, 1, 1, 4)
    eng.close()
    assert rs0 == (0, 0, 0) and rs1 == (1, 0, 0)
    assert np.array_equal(a0, a1) and np.array_equal(p0, p1)
    assert st0["n_rounds"] == st1["n_rounds"] and st0["evals"] == st1["evals"]


def test_2000_x_2000_within_T_of_scipy_and_exact_with_the_scale():
    t, cap = scipy_instance(2000, 2000, 4)
    T = len(cap)
    ap = t["wb"]["ext_ask_price"]
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    opt = rc.optimum(F, ap, cap)
    eng = engine(t, cap)
    got, price, st, (phases, n_rev, bids) = run(eng, T, 1, 64, 4)
    assert phases == 4 and n_rev > 0 and bids > 0
    sold = np.flatnonzero(got != NONE)
    assert len(np.unique(got[sold])) == len(sold) and F[sold, got[sold]].all()
    assert opt <= wc.total_cost(got, ap, cap) <= opt + T
    owned = np.zeros(len(ap), dtype=bool)
    owned[got[sold]] = True
    assert np.all(price[~owned] == 0)
    got, _, _, _ = run(eng, T, T + 1, 64, 4)
    assert wc.total_cost(got, ap, cap) == opt
    eng.close()


def test_warm_pass_after_a_reverse_pass_equals_the_warm_checker():
    t, cap = tables(300, 2500, 3)
    T = len(cap)
    m = wc.Market(t, cap)
    eng = engine(t, cap)
    got, price, _, _ = run(eng, T, 1, 64, 4)
    F = m.F()
    a, p, *_ = rc.scaled(F, t["wb"]["ext_ask_price"], cap, 1, 64, 4)
    assert np.array_equal(got, a) and np.array_equal(price, p)
    m.store(p, a)
    rng = np.random.default_rng(12)
    for _ in range(3):
        wc.random_step(m, rng, eng=eng)
        eng.match(abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM)
        res = eng.fetch()
        got = np.full(T, NONE, dtype=np.uint32)
        for ask, members in res.groups():
            got[ask] = members[0]
        price, warm, released = eng.auction_state()
        a, p, n, rel = m.warm(1)
        assert warm and released == len(rel)
        assert np.array_equal(got, a) and np.array_equal(price, p) and res.stats["n_rounds"] == n
        assert eng.auction_reverse_stats() == (0, 0, 0)
        m.store(p, a)
    eng.close()


def test_refusals():
    t, cap = tables(50, 700, 2)
    eng = engine(t, cap)
    with pytest.raises(PrimeMatchError) as ex:
        eng.auction_reverse_stats()
    assert ex.value.status == abi.PM_E_STATE
    for mode in (abi.PM_MODE_FIRST_FIT | abi.PM_AUCTION_REVERSE, abi.PM_MODE_PROXIMITY | abi.PM_AUCTION_REVERSE,
                 abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_AUCTION_REVERSE,
                 REV | abi.PM_AUCTION_WARM):
        with pytest.raises(PrimeMatchError) as ex:
            eng.match(mode)
        assert ex.value.status == abi.PM_E_INVALID, hex(mode)
    with pytest.raises(PrimeMatchError) as ex:
        eng.match_finish(abi.PM_MODE_FIRST_FIT | abi.PM_AUCTION_REVERSE)
    assert ex.value.status == abi.PM_E_INVALID
    eng.set_auction_params(eps_start=64)
    eng.set_ask_enabled([3], False)
    with pytest.raises(PrimeMatchError) as ex:
        eng.match(REV)
    assert ex.value.status == abi.PM_E_UNSUPPORTED
    eng.set_ask_enabled([3], True)
    eng.set_shard(0, 350)
    with pytest.raises(PrimeMatchError) as ex:
        eng.match(REV)
    assert ex.value.status == abi.PM_E_UNSUPPORTED
    eng.close()


def test_scaled_pass_at_cfg3_size():
    """100k asks x 1M workers, eps 64 / 4 with reverse rounds: injective, caps and requirements respected on a sample
    (the oracle's predicate), every unowned worker at price 0 (all of them), and eps-complementary slackness at eps = 1
    on 300 sampled asks against every worker."""
    t, cap = cfg3()
    T, W = len(cap), len(t["wa"])
    eng = engine(t, cap)
    got, price, st, (phases, n_rev, bids) = run(eng, T, 1, 64, 4)
    eng.close()
    assert phases == 4 and n_rev > 0 and bids > 0
    ap = t["wb"]["ext_ask_price"].astype(np.int64)
    sold = np.flatnonzero(got != NONE)
    assert len(np.unique(got[sold])) == len(sold) and np.all(ap[got[sold]] <= cap[sold])
    owned = np.zeros(W, dtype=bool)
    owned[got[sold]] = True
    assert np.all(price[~owned] == 0) and np.all(price >= 0)
    rng = np.random.default_rng(6)
    value = -ap - price
    for tk in rng.choice(T, 300, replace=False):
        F = wc.feasible(t["wa"], t["wb"], t["asks"][tk:tk + 1], t["opts"], t["bits"], t["words"], cap[tk:tk + 1])[0]
        pi = value[got[tk]] if got[tk] != NONE else -(int(cap[tk]) + 1)
        if got[tk] != NONE:
            assert F[got[tk]]
        if F.any():
            assert value[F].max() <= pi + 1
