"""pm_auction_certificate on the device: every field and every per-ask row term equal the exact-integer restatement
(auction_certificate.py) on instances that select each predicate variant (acceptance rows in shared or global memory,
one uniform word, the worker-major word, asks with more OR-options than the stage holds; generic and fast predicate),
at the u32 edges and at the top of the integer domain, on stored states made stale by table changes; cold, reverse,
warm and repair passes all certify within T; with cost_scale = T + 1 at 2000 x 2000 the cost is scipy's optimum; the
eps-scaled pass without reverse rounds is flagged; the call has no side effects; refusals; and one cold pass at the
100k x 1M size of BASELINE configs[2]."""
import ctypes as C
import os
import time

import numpy as np
import pytest

import auction_certificate as ac
import auction_reverse_checker as rc
import auction_warm_checker as wc
from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError
from protocol_b200.engine import Engine
from test_auction_exact_checker import U32, last_admitted_scale, ladder
from test_gpu_auction_domain import edge_market
from test_gpu_auction_reverse import scipy_instance
from test_gpu_auction_warm import cfg3, engine, tables
from test_gpu_variants import many_option_tables, wide_tables

pytestmark = pytest.mark.gpu

NONE = wc.NONE
AUC, REV = abi.PM_MODE_AUCTION, abi.PM_MODE_AUCTION | abi.PM_AUCTION_REVERSE
WARM = AUC | abi.PM_AUCTION_WARM
REPAIR = WARM | abi.PM_AUCTION_REPAIR


def stored(eng, T):
    """The last pass's assignment (from the result) and prices (pm_auction_state)."""
    res = eng.fetch()
    got = np.full(T, NONE, dtype=np.uint32)
    got[res.group_ask] = res.group_members
    return got, eng.auction_state()[0]


def check_equal(eng, F, ap, cap, S, price, assigned):
    """The device's certificate against the restatement, field by field and row by row."""
    got = eng.auction_certificate(ask_bound=True)
    want = ac.certificate(F, ap, cap, S, price, assigned)
    for k in ac.FIELDS:
        assert got[k] == want[k], (k, got[k], want[k])
    assert np.array_equal(got["ask_bound"], want["ask_bound"])
    return got


def check_sound(c, T):
    assert (c["n_bad_holds"], c["n_shared"], c["n_priced_unowned"], c["n_slack_over"]) == (0, 0, 0, 0)
    assert c["max_slack"] <= 1 and 0 <= c["gap"] <= T and c["priced_unowned_sum"] == 0


# ---------------------------------------------------------------- every predicate variant, bit for bit
def variant_case(name):
    if name == "bits1":
        return wide_tables(400, 6000, n_models=200, n_patterns=112, seed_shift=1)
    if name == "bits0":
        return wide_tables(400, 6000, n_models=3000, n_patterns=112, seed_shift=2, last_rows=True)
    if name == "models100k":
        return wide_tables(260, 20000, n_models=100_000, n_patterns=40, seed_shift=3, last_rows=True)
    if name in ("wm30", "wm31"):
        n = int(name[2:])
        return wide_tables(400, 9000, n_models=3000, n_patterns=n, seed_shift=11 + n, last_rows=True)
    if name == "uniform":
        return wide_tables(300, 5000, n_models=30, n_patterns=900, seed_shift=4, last_rows=True)
    return many_option_tables(16 if name == "options16" else 200)


@pytest.mark.parametrize("name", ["bits1", "bits0", "models100k", "wm30", "wm31", "uniform", "options16", "options200"])
def test_equals_the_restatement_on_every_predicate_variant(name):
    w, a, obits, pbits, npat, nmod, words = variant_case(name)
    T, W = len(a.asks), len(w.a)
    rng = np.random.default_rng(len(name))
    wb = w.b.copy()
    wb["ext_ask_price"] = rng.integers(10, 1000, W).astype(np.uint32)
    cap = rng.integers(50, 1500, T).astype(np.uint32)
    rep = rng.integers(0, 4, W).astype(np.uint32)
    floors = rng.integers(0, 3, T).astype(np.uint32)
    for generic in ("0", "1"):
        os.environ["PM_TUNE_GENERIC"] = generic   # read at pm_create
        try:
            eng = Engine()
        finally:
            os.environ.pop("PM_TUNE_GENERIC", None)
        eng.set_asks(a.asks, a.opts)
        eng.set_model_table(pbits, npat, nmod, words)
        eng.set_workers(w.a, wb)
        eng.set_price_caps(cap)
        eng.set_worker_reputation(rep)
        eng.set_min_reputation(floors)
        eng.match(AUC)
        assigned, price = stored(eng, T)
        F = wc.feasible(w.a, wb, a.asks, a.opts, obits, words, cap, rep, floors)
        check_sound(check_equal(eng, F, wb["ext_ask_price"], cap, 1, price, assigned), T)
        # stale: rows rewritten (health flipped, prices moved, held rows among them) and caps changed since the pass
        idx = np.unique(np.concatenate([rng.choice(W, 40, replace=False), assigned[assigned != NONE][:20]])).astype(np.uint32)
        wa2, wb2 = w.a.copy(), wb.copy()
        wa2["flags"][idx[::2]] ^= abi.PM_W_HEALTHY
        wb2["ext_ask_price"][idx[1::2]] = rng.integers(10, 1000, len(idx[1::2]))
        eng.update_workers(idx, wa2[idx], wb2[idx])
        cap2 = cap.copy()
        cap2[rng.choice(T, 20, replace=False)] //= 2
        eng.set_price_caps(cap2)
        F2 = wc.feasible(wa2, wb2, a.asks, a.opts, obits, words, cap2, rep, floors)
        c = check_equal(eng, F2, wb2["ext_ask_price"], cap2, 1, price, assigned)
        assert c["n_bad_holds"] > 0
        eng.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_equals_the_restatement_at_the_u32_edges(seed):
    """Prices and caps at 0, 2^31 - 1, 2^31, 2^32 - 2, 2^32 - 1, reputations and floors at 0 or 2^32 - 1; S = 1 and
    T + 1, and the eps-scaled pass without reverse rounds (priced unowned workers)."""
    t, cap, rep, floors = edge_market(seed)
    T = len(cap)
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap, rep, floors)
    eng = Engine()
    eng.set_asks(t["asks"], t["opts"])
    eng.set_workers(t["wa"], t["wb"])
    eng.set_price_caps(cap)
    eng.set_worker_reputation(rep)
    eng.set_min_reputation(floors)
    for S, eps, mode in ((1, 1, AUC), (T + 1, 1, AUC), (T + 1, 1 << 20, AUC), (T + 1, 1 << 40, REV)):
        eng.set_auction_params(cost_scale=S, eps_start=eps, eps_div=16)
        eng.match(mode)
        assigned, price = stored(eng, T)
        c = check_equal(eng, F, t["wb"]["ext_ask_price"], cap, S, price, assigned)
        if eps == 1 or mode == REV:
            check_sound(c, T)
    eng.close()


DOMAIN_CASES = [   # test_gpu_auction_domain.py's: (prices, caps, P)
    ([1, 2, (1 << 31) + 3], [U32, U32 - 1, U32], (1 << 31) + 3),
    ([0, 0x7FFFFFFF, 0x80000000, U32 - 1], [U32, 0x80000000, U32, U32 - 1], U32),
    ([5, 6, 1000], [1500, 1499, 1500], 2000),
]


@pytest.mark.parametrize("case", range(len(DOMAIN_CASES)))
def test_equals_the_restatement_at_the_top_of_the_domain(case):
    """The last admitted S, and the last admitted eps_start at S = T + 1; one step past the domain through a cap is
    refused (PM_E_INVALID) and changes nothing."""
    ap, caps, P = DOMAIN_CASES[case]
    t, cap, rep, floors = ladder(ap, caps, extra_price=P)
    T, K = len(caps), max(caps)
    S = last_admitted_scale(P, K)
    E = (1 << 61) - 1 - (P + K + 2) * (T + 1)
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap, rep, floors)
    eng = Engine()
    eng.set_asks(t["asks"], t["opts"])
    eng.set_workers(t["wa"], t["wb"])
    eng.set_price_caps(cap)
    eng.set_worker_reputation(rep)
    eng.set_min_reputation(floors)
    for s, e, mode in ((T + 1, E, REV), (S, 1, AUC)):
        eng.set_auction_params(cost_scale=s, eps_start=e, eps_div=1 << 20)
        eng.match(mode)
        assigned, price = stored(eng, T)
        check_sound(check_equal(eng, F, t["wb"]["ext_ask_price"], cap, s, price, assigned), T)
    if K < U32:   # a larger cap puts the tables past the domain at this S
        before = eng.auction_certificate(ask_bound=True)
        eng.set_price_caps(np.full(T, U32, dtype=np.uint32))
        with pytest.raises(PrimeMatchError) as exc:
            eng.auction_certificate()
        assert exc.value.status == abi.PM_E_INVALID
        eng.set_price_caps(cap)
        after = eng.auction_certificate(ask_bound=True)
        assert all(after[k] == before[k] for k in ac.FIELDS) and np.array_equal(after["ask_bound"], before["ask_bound"])
    eng.close()


# ---------------------------------------------------------------- every pass kind keeps the bound
@pytest.mark.parametrize("S", [1, 121])
def test_every_pass_kind_certifies_within_T(S):
    t, cap = tables(120, 1500, 31)
    rng = np.random.default_rng(31 + S)
    rep = rng.integers(0, 4, 1500).astype(np.uint32)
    floors = rng.integers(0, 3, 120).astype(np.uint32)
    T = len(cap)
    m = wc.Market(t, cap, rep, floors)
    eng = engine(t, cap, floors=floors, reputation=rep, S=S)

    def certify():
        assigned, price = stored(eng, T)
        check_sound(check_equal(eng, m.F(), m.wb["ext_ask_price"], m.cap, S, price, assigned), T)
        m.store(price, assigned)

    eng.match(AUC)
    certify()
    eng.set_auction_params(cost_scale=S, eps_start=64, eps_div=4)
    eng.match(REV)
    certify()
    for mode in (WARM, REPAIR, WARM, REPAIR, REPAIR):
        for _ in range(int(rng.integers(1, 3))):
            wc.random_step(m, rng, eng=eng)
        eng.match(mode)
        certify()
    eng.close()


def test_exact_optimum_at_2000_x_2000():
    t, cap = scipy_instance(2000, 2000, 4)
    T = len(cap)
    S = T + 1
    eng = engine(t, cap)
    eng.set_auction_params(cost_scale=S, eps_start=64, eps_div=4)
    eng.match(REV)
    c = eng.auction_certificate()
    check_sound(c, T)
    assert c["gap"] < S
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    assert c["cost"] == rc.optimum(F, t["wb"]["ext_ask_price"], cap, S)
    eng.close()


def test_the_scaled_pass_without_reverse_rounds_is_flagged():
    t, cap = scipy_instance(60, 200, 1)
    T = len(cap)
    eng = engine(t, cap)
    eng.set_auction_params(eps_start=64, eps_div=4)
    eng.match(AUC)
    assigned, price = stored(eng, T)
    F = wc.feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    c = check_equal(eng, F, t["wb"]["ext_ask_price"], cap, 1, price, assigned)
    assert c["n_priced_unowned"] > 0 and c["gap"] > T
    eng.close()


def test_a_stale_hold_is_flagged_until_the_next_warm_pass():
    t, cap = tables(50, 700, 2)
    T = len(cap)
    m = wc.Market(t, cap)
    eng = engine(t, cap)
    eng.match(AUC)
    assigned, price = stored(eng, T)
    m.store(price, assigned)
    check_sound(eng.auction_certificate(), T)
    w = int(assigned[assigned != NONE][0])
    m.set_flags([w], [m.wa["flags"][w] ^ abi.PM_W_HEALTHY], eng)
    c = check_equal(eng, m.F(), m.wb["ext_ask_price"], m.cap, 1, price, assigned)
    assert c["n_bad_holds"] >= 1
    eng.match(WARM)
    check_sound(eng.auction_certificate(), T)
    eng.close()


# ---------------------------------------------------------------- no side effects
def snapshot(eng, T):
    res = eng.fetch()
    st = {k: v for k, v in res.stats.items() if not k.startswith("ms_")}
    return (res.worker_group.copy(), res.worker_ask.copy(), res.group_ask.copy(), res.group_members.copy(),
            res.ask_best.copy(), res.ask_count.copy(), st, eng.table_version(), eng.auction_state(),
            eng.auction_reverse_stats())


def same(x, y):
    for a, b in zip(x, y):
        if isinstance(a, tuple):
            assert same(a, b)
        elif isinstance(a, np.ndarray):
            assert np.array_equal(a, b)
        else:
            assert a == b, (a, b)
    return True


@pytest.mark.parametrize("first", [AUC, REV])
def test_no_side_effects_on_a_twin_engine(first):
    t, cap = tables(300, 2500, 3)
    T = len(cap)
    twins = [engine(t, cap), engine(t, cap)]
    rng = [np.random.default_rng(9), np.random.default_rng(9)]
    markets = [wc.Market(t, cap), wc.Market(t, cap)]
    for e in twins:
        e.set_auction_params(eps_start=64 if first == REV else 1, eps_div=4)
        e.match(first)
    for mode in (WARM, REPAIR, WARM, REPAIR):
        before = snapshot(twins[0], T)
        c = twins[0].auction_certificate(ask_bound=True)
        assert c["evals"] == T * twins[0].n_workers
        assert same(snapshot(twins[0], T), before)
        assert same(snapshot(twins[1], T), before)
        for e, m, r in zip(twins, markets, rng):
            got, price = stored(e, T)
            m.store(price, got)
            wc.random_step(m, r, eng=e, kinds=("price", "flags", "spec", "caps", "floors", "toggle"))
        twins[0].auction_certificate()   # also after the changes: the warm start's marks stay as they were
        for e in twins:
            e.match(mode)
        assert same(snapshot(twins[0], T), snapshot(twins[1], T))
    for e in twins:
        e.close()


# ---------------------------------------------------------------- refusals
def test_refusals_change_nothing():
    t, cap = tables(50, 700, 2)
    eng = engine(t, cap)
    lib = eng._lib
    cert = abi.PmAuctionCert()
    assert lib.pm_auction_certificate(None, C.byref(cert), None) == abi.PM_E_INVALID
    assert lib.pm_auction_certificate(eng._h, None, None) == abi.PM_E_INVALID
    with pytest.raises(PrimeMatchError) as exc:      # no auction pass yet
        eng.auction_certificate()
    assert exc.value.status == abi.PM_E_STATE
    eng.match(abi.PM_MODE_FIRST_FIT)                 # a reference-mode pass stores no auction state
    with pytest.raises(PrimeMatchError) as exc:
        eng.auction_certificate()
    assert exc.value.status == abi.PM_E_STATE
    eng.match(AUC)
    ref = eng.auction_certificate(ask_bound=True)

    def light():
        return ({k: v for k, v in eng.stats().items() if not k.startswith("ms_")}, eng.auction_state(),
                eng.auction_reverse_stats(), eng.table_version())

    def refused(status):
        before = light()
        with pytest.raises(PrimeMatchError) as exc:
            eng.auction_certificate(ask_bound=True)
        assert exc.value.status == status
        assert same(light(), before)

    eng.set_ask_enabled([3], False)
    refused(abi.PM_E_UNSUPPORTED)
    eng.set_ask_enabled([3], True)
    W = len(t["wa"])
    eng.resize_workers(W + 5)                        # the stored pass had W rows
    refused(abi.PM_E_STATE)
    eng.resize_workers(W)
    c = eng.auction_certificate(ask_bound=True)
    assert all(c[k] == ref[k] for k in ac.FIELDS) and np.array_equal(c["ask_bound"], ref["ask_bound"])
    eng.set_auction_params(cost_scale=1 << 40)       # discards the stored state
    with pytest.raises(PrimeMatchError) as exc:
        eng.auction_certificate()
    assert exc.value.status == abi.PM_E_STATE
    eng.close()


def test_the_domain_refusal_through_a_written_row():
    """At the largest scale P = 3 admits, a row written to ask_price 2^32 - 1 puts the tables past the domain: refused;
    written back, the same certificate as before."""
    t, cap, rep, floors = ladder([1, 2, 3], [3, 3, 3])
    T = len(cap)
    eng = Engine()
    eng.set_asks(t["asks"], t["opts"])
    eng.set_workers(t["wa"], t["wb"])
    eng.set_price_caps(cap)
    eng.set_worker_reputation(rep)
    eng.set_min_reputation(floors)
    eng.set_auction_params(cost_scale=last_admitted_scale(3, 3))
    eng.match(AUC)
    ref = eng.auction_certificate(ask_bound=True)
    check_sound(ref, T)
    b = t["wb"][1:2].copy()
    b["ext_ask_price"] = U32
    eng.update_workers(np.array([1], dtype=np.uint32), t["wa"][1:2], b)
    with pytest.raises(PrimeMatchError) as exc:
        eng.auction_certificate()
    assert exc.value.status == abi.PM_E_INVALID
    eng.update_workers(np.array([1], dtype=np.uint32), t["wa"][1:2], t["wb"][1:2])
    c = eng.auction_certificate(ask_bound=True)
    assert all(c[k] == ref[k] for k in ac.FIELDS) and np.array_equal(c["ask_bound"], ref["ask_bound"])
    eng.close()


# ---------------------------------------------------------------- full size
def test_cold_pass_at_cfg3_size_certifies_within_T():
    """100k asks x 1M workers: one cold pass, then the certificate of its state — the first check of the bound at the
    size the benchmark runs.  The time is printed, not asserted."""
    t, cap = cfg3()
    T, W = len(cap), len(t["wa"])
    eng = engine(t, cap)
    eng.match(AUC)
    eng.auction_certificate()
    t0 = time.perf_counter()
    c = eng.auction_certificate(ask_bound=True)
    ms = (time.perf_counter() - t0) * 1e3
    eng.close()
    print(f"\ncertificate at 100k x 1M: {ms:.1f} ms, gap {c['gap']}, held {c['n_held']}, max slack {c['max_slack']}")
    check_sound(c, T)
    assert c["evals"] == T * W and c["n_held"] > 0
    assert c["bound"] <= c["cost"] and np.all(c["ask_bound"] >= 0)
