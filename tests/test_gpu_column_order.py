"""pm_build_argmin_feat's sorted column order on hardware: column c of the tile holds worker w0 + perm[c], the workers
of the range sorted by __brevll(F), and pm_stripe_rank ranks each stripe by (price, worker).  ask_best, ask_count and
first_ask must be those of the int64 tile (PM_TUNE_BUILD=8, which builds in worker order) and of the CPU oracle, bit
for bit.

The cases aim at what a column/worker mix-up would get wrong: equal least prices on workers whose columns come in the
opposite order (the least worker wins, not the least column), ties across stripes, ragged stripes and tiles, shards
whose w0 is off a stripe boundary, and an incremental pass after an upsert that moves workers into other F runs."""
import numpy as np
import pytest

import feature_tables as ft
from helpers import load_engine
from protocol_b200 import abi
from protocol_b200.engine import Engine
from protocol_b200.sharded import shard_range
from test_column_order_formulation import column_order, features
from test_gpu_feature_predicate import FEAT, check, kernel_of, pass_arrays
from test_gpu_narrow_tile import MAT, oracle_eval
from test_gpu_tile_overlap import tile_bytes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed,T,W,price_max", [(1, 700, 3000, 3), (2, 513, 2049, 1), (3, 1025, 4099, 1 << 30)])
def test_price_ties_through_the_column_order(seed, T, W, price_max):
    t = ft.edge_tables(seed, T, W, price_max=price_max)
    got = check(t)
    assert (got[2] > 0).any()
    assert kernel_of(t) == {FEAT}


def test_least_worker_wins_a_tie_between_inverted_columns():
    """Every price 1000 but two workers at 5 in the same stripe that the sort puts in the opposite order."""
    t = ft.edge_tables(8, 600, 2048, price_max=1 << 20)
    F, n, fail = features(t, 0, 2048)
    perm = column_order(F, n, 2048)
    feas = fail == 0
    pairs = [(i, j) for i in range(1024) for j in range(i + 1, min(i + 64, 1024))
             if perm[i] > perm[j] and (feas[:, perm[i]] & feas[:, perm[j]]).any()]
    assert pairs
    i, j = pairs[0]
    wb = t["wb"].copy()
    wb["ext_ask_price"] = 1000
    wb["ext_ask_price"][[perm[i], perm[j]]] = 5
    t = dict(t, wb=wb)
    got = check(t)
    rows = feas[:, perm[i]] & feas[:, perm[j]]
    assert (got[1][rows] == (5 << 32) | int(perm[j])).all()


@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_ranges_with_ties(n_shards):
    t = ft.edge_tables(50 + n_shards, 800, 9001, price_max=4)
    W = len(t["wa"])
    for r in range(n_shards):
        lo, hi = shard_range(W, n_shards, r)
        check(t, tile_bytes(hi - lo, 256), shard=(lo, hi - lo))


@pytest.mark.parametrize("T,W,rows", [(1100, 5000, 256), (777, 3333, 100)])
def test_several_tiles_with_a_ragged_last_one(T, W, rows):
    check(ft.edge_tables(T + W + 7, T, W, price_max=2), tile_bytes(W, rows))


def test_incremental_pass_after_an_upsert_that_moves_workers_between_runs():
    """Full materialised pass (the sorted columns), then pm_upsert_workers over a block of rows with other workers'
    contents (their F changes), then an incremental pass (PM_INCREMENTAL runs on the lean fused path, from the stored
    evaluation the materialised pass left): its first_ask must be a full pass's on the same table, and so must the
    next materialised pass's."""
    t = ft.edge_tables(77, 900, 6000, price_max=3)
    W, T = len(t["wa"]), len(t["asks"])
    rng = np.random.default_rng(5)
    first = 1500
    src = rng.permutation(W)[:2000]
    na, nb = t["wa"][src].copy(), t["wb"][src].copy()
    t2 = dict(t, wa=t["wa"].copy(), wb=t["wb"].copy())
    t2["wa"][first:first + len(src)] = na
    t2["wb"][first:first + len(src)] = nb
    ev = oracle_eval(t2, 0, W)
    want = np.asarray(ev["col_first"]).astype(np.uint32)

    e = Engine(cost_tile_bytes=tile_bytes(W, 256))
    try:
        load_engine(e, t)
        e.match_local(MAT)
        e.sync()
        e.upsert_workers(na, nb, first)
        e.match_local(abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_INCREMENTAL)
        e.sync()
        inc = pass_arrays(e, W, T)[0].copy()
        e.match_local(MAT)
        e.sync()
        full = pass_arrays(e, W, T)
    finally:
        e.close()
    assert np.array_equal(inc, want)
    assert np.array_equal(full[0], want)
    assert np.array_equal(full[2], ev["row_count"]) and np.array_equal(full[1], ev["row_best"])
