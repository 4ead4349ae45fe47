"""The feature predicate of pm_build_argmin_feat, restated in numpy (feature_tables.py), held against the fast
predicate's restatement and the CPU oracle pair by pair: the dictionary of distinct (clause, threshold) pairs, the
worker words F, the requirement masks R and u = R & ~F, on random tables and at the edge values of every feature kind."""
import numpy as np
import pytest

import feature_tables as ft
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from test_fast_predicate_formulation import fast_cost_matrix


def oracle_cost(t):
    return orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], 0, len(t["asks"]), 0,
                               len(t["wa"]), want_cost=True)["cost"]


def assert_three_agree(t):
    got = ft.feature_cost_matrix(t)
    assert np.array_equal(got, fast_cost_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["n_patterns"],
                                                t["n_models"], t["words"]))
    assert np.array_equal(got, oracle_cost(t))
    return got


@pytest.mark.parametrize("kind,price", [("mixed", None), ("skewed", "zipf"), ("uniform1", "loguniform")])
def test_feature_formulation_on_synthetic_tables(kind, price):
    w = synth.make_workers(1500, price=price)
    a = synth.make_asks(200, kind, group_sizes=[(1, 1), (0, 0), (2, 3)])
    bits, npat, nmod, words = synth.intern_tables(w, a)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)
    assert_three_agree(t)


@pytest.mark.parametrize("seed", range(6))
def test_feature_formulation_at_edge_values(seed):
    t = ft.edge_tables(seed, 120, 900)
    got = assert_three_agree(t)
    assert (got != ft.INF).any() and (got == ft.INF).any()


def test_every_feature_kind_alone():
    """One ask per kind of clause, and no other clause than the candidate bit: each kind decides alone."""
    base = ft.edge_tables(11, 0, 1200)
    O = abi.GPU_OPT
    rows = [  # (ask flags, cpu, ram, storage, option or None)
        (0, 0, 0, 0, None),
        (abi.PM_A_HAS_REQ | abi.PM_A_REQ_CPU | abi.PM_A_REQ_CPU_CORES, 8, 0, 0, None),
        (abi.PM_A_HAS_REQ | abi.PM_A_REQ_RAM, 0, 2, 0, None),
        (abi.PM_A_HAS_REQ | abi.PM_A_REQ_STORAGE, 0, 0, 0x7FFFFFFE, None),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_COUNT, 4, 0, 0, 0, 0, 0, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_COUNT, 0, 0, 0, 0, 0, 0, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_MODEL, 0, 0, 0, 0, 0, 0, 3)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_MEM, 0, 1, 0, 0, 0, 0, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_MEM_MAX, 0, 0, 0, 40000, 0, 0, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_MEM_MIN | abi.PM_O_MEM_MAX, 0, 0, 40000, 40000, 0, 0, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_MEM_MIN | abi.PM_O_MEM_MAX, 0, 0, 80000, 40000, 0, 0, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_TOT_MIN, 0, 0, 0, 0, 100000, 0, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_TOT_MAX, 0, 0, 0, 0, 0, 320000, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_TOT_MIN | abi.PM_O_TOT_MAX, 0, 0, 0, 0, 320000, 100000, 0)),
        (abi.PM_A_HAS_REQ, 0, 0, 0, (abi.PM_O_TOT_MIN | abi.PM_O_TOT_MAX, 0, 0, 0, 0, 1, 1, 0)),
    ]
    asks, opts = [], []
    for fl, cpu, ram, sto, o in rows:
        asks.append((fl, 0 if o is None else 1, len(opts), cpu, ram, sto, 1, 1))
        if o is not None:
            opts.append(o)
    t = dict(base, asks=np.array(asks, dtype=abi.ASK), opts=np.array(opts, dtype=O))
    got = assert_three_agree(t)
    d = ft.dictionary(ft.converted(t["asks"], t["opts"]))
    assert {k for k, _ in d} == set(range(10)), "every kind of feature is reached"
    # no two of the single-clause asks accept the same workers (ask 0 takes every candidate)
    feas = got != ft.INF
    assert len({row.tobytes() for row in feas}) >= len(rows) - 2


def test_or_options_that_miss_different_features():
    """Two options that each fail on a different feature: the ask still fails (the kernel takes the minimum over the
    options, not an AND of the masks), and one that passes makes the ask pass."""
    t = ft.edge_tables(3, 0, 1000, max_opts=0)
    O = abi.GPU_OPT
    opts = [(abi.PM_O_COUNT, 8, 0, 0, 0, 0, 0, 0), (abi.PM_O_MEM, 0, 80000, 0, 0, 0, 0, 0),
            (abi.PM_O_MODEL, 0, 0, 0, 0, 0, 0, 2), (abi.PM_O_TOT_MAX, 0, 0, 0, 0, 0, 1, 0)]
    fl = abi.PM_A_HAS_REQ | abi.PM_A_REQ_RAM | abi.PM_A_REQ_CPU | abi.PM_A_REQ_CPU_CORES
    asks = [(fl, 2, 0, 8, 64, 0, 1, 1), (fl, 4, 0, 0, 2, 0, 1, 1), (abi.PM_A_HAS_REQ, 3, 1, 0, 0, 0, 1, 1),
            (abi.PM_A_HAS_REQ | abi.PM_A_REQ_STORAGE, 2, 2, 0, 0, 0x7FFFFFFE, 1, 1)]
    t = dict(t, asks=np.array(asks, dtype=abi.ASK), opts=np.array(opts, dtype=O))
    assert_three_agree(t)


def test_disabled_asks_need_no_new_feature():
    t = ft.edge_tables(5, 80, 600)
    rng = np.random.default_rng(1)
    on = rng.random(len(t["asks"])) > .3
    conv_on = ft.converted(t["asks"], t["opts"])
    assert ft.dictionary(ft.converted(t["asks"], t["opts"], on)) == ft.dictionary(conv_on)
    got = ft.feature_cost_matrix(t, on)
    ref = oracle_cost(t)
    assert np.array_equal(got[on], ref[on])
    assert (got[~on] == ft.INF).all()


def test_64_features_fit_and_65_do_not():
    base = ft.edge_tables(7, 30, 500)
    for n in (64, 65):
        t = ft.with_features(base, n)
        d = ft.dictionary(ft.converted(t["asks"], t["opts"]))
        assert len(d) == n and ft.fits(d) == (n <= 64)
    assert_three_agree(ft.with_features(base, 64))
