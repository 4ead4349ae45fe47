"""Parity of the CUDA path against the CPU oracle, through the C ABI.  Bit-exact
(integer/index work).  Run with `pytest -m gpu` on an H100."""
import os

import numpy as np
import pytest

import kat_vectors as kv
from helpers import TableBuilder, assert_distance_certificate, groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200.engine import Engine

pytestmark = pytest.mark.gpu

MAT, FUSED = abi.PM_PATH_MATERIALIZED, abi.PM_PATH_FUSED


def synth_tables(n_asks, n_workers, kind="mixed", group_sizes=None, seed_shift=0, with_addresses=False, price=None):
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed_shift, with_addresses=with_addresses, price=price)
    a = synth.make_asks(n_asks, kind, seed=synth.SEED_ASKS + seed_shift, group_sizes=group_sizes)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    return w, a, dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod,
                      words=words, lat=w.lat, lon=w.lon)


def check_against_oracle(eng, t, mode, addr_rank=None, proximity=False, check_rows=True):
    eng.match(mode)
    res = eng.fetch()
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], addr_rank=addr_rank,
                             lat=t["lat"], lon=t["lon"], proximity=proximity)
    assert groups_equal(res, og), f"groups differ: engine {res.n_groups} vs oracle {len(og)}"
    # per-worker view is consistent with the group table
    wg = np.full(len(t["wa"]), abi.PM_NONE, dtype=np.uint32)
    wk = np.full(len(t["wa"]), abi.PM_NONE, dtype=np.uint32)
    for g in range(len(og.cfg)):
        m = og.members[og.off[g]:og.off[g + 1]]
        wg[m] = g
        wk[m] = og.cfg[g]
    assert np.array_equal(res.worker_group, wg) and np.array_equal(res.worker_ask, wk)
    if check_rows:
        T, W = len(t["asks"]), len(t["wa"])
        ev = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], 0, T, 0, W, threads=8)
        assert np.array_equal(res.ask_best, ev["row_best"])
        assert np.array_equal(res.ask_count, ev["row_count"])
    return res, og


def test_kat_vectors_on_device():
    """Every meets() vector of node.rs:659-1241 as one (ask, worker) pair: entry [i][i] of the
    materialised cost matrix is finite iff the reference test expects meets() == true."""
    tb = TableBuilder()
    for name, line, specs, req, expected in kv.MEETS:
        tb.add_config(req)
        tb.add_node(specs)
    t = tb.tables()
    eng = Engine()
    load_engine(eng, t)
    n = len(kv.MEETS)
    cost = eng.cost_tile(0, n)
    for i, (name, line, specs, req, expected) in enumerate(kv.MEETS):
        assert bool(cost[i, i] != abi.PM_COST_INF) is expected, name
        if expected:
            assert cost[i, i] == i
    ev = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], 0, n, 0, n, want_cost=True)
    assert np.array_equal(cost, ev["cost"])
    eng.close()


@pytest.mark.parametrize("path", [MAT, FUSED], ids=["materialized", "fused"])
def test_cfg1_uniform_1k_x_10k(path):
    """BASELINE configs[0]: 1k tasks x 10k workers, uniform single-GPU asks."""
    w, a, t = synth_tables(1000, 10000, "uniform1")
    eng = Engine()
    load_engine(eng, t)
    res, og = check_against_oracle(eng, t, abi.PM_MODE_FIRST_FIT | path)
    assert res.stats["evals"] == 1000 * 10000
    eng.close()


def test_cost_matrix_bit_exact_cfg1():
    w, a, t = synth_tables(1000, 10000, "mixed")
    eng = Engine()
    load_engine(eng, t)
    cost = eng.cost_tile(0, 1000)
    ev = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], 0, 1000, 0, 10000,
                             threads=8, want_cost=True)
    assert np.array_equal(cost, ev["cost"])
    eng.close()


@pytest.mark.parametrize("path", [MAT, FUSED], ids=["materialized", "fused"])
@pytest.mark.parametrize("nt,nw", [(1, 1), (3, 2), (129, 513), (257, 1023), (700, 4099)])
def test_ragged_shapes(path, nt, nw):
    w, a, t = synth_tables(nt, nw, "mixed", seed_shift=nt * 7 + nw)
    eng = Engine(cost_tile_bytes=64 * 1024)   # forces several row tiles
    load_engine(eng, t)
    check_against_oracle(eng, t, abi.PM_MODE_FIRST_FIT | path)
    eng.close()


@pytest.mark.parametrize("path", [MAT, FUSED], ids=["materialized", "fused"])
def test_group_sizes_with_underfilled_tails(path):
    """min/max > 1: the sweep that hands under-filled tails to later configurations."""
    sizes = [(1, 1), (2, 2), (2, 4), (3, 3), (4, 8), (1, 3), (5, 16)]
    w, a, t = synth_tables(300, 6000, "mixed", group_sizes=sizes, with_addresses=True)
    eng = Engine()
    load_engine(eng, t, addr_rank=w.addr_rank)
    res, og = check_against_oracle(eng, t, abi.PM_MODE_FIRST_FIT | path, addr_rank=w.addr_rank)
    assert res.stats["n_bumped"] > 0, "test input should exercise the tail sweep"
    eng.close()


def test_degenerate_group_sizes():
    """min_group_size == 0 yields a trailing empty group; max_group_size == 0 takes nobody
    (mod.rs:507-566,606)."""
    tb = TableBuilder()
    tb.add_config("gpu:count=8", 0, 0)
    tb.add_config("gpu:count=1", 0, 2)
    tb.add_config(None, 2, 3)
    for c in (1, 1, 1, 8, 2, 2, 2, 2, 4):
        tb.add_node(kv.specs(c, "A100", 40000, 8, 1000, 10))
    t = tb.tables()
    eng = Engine()
    load_engine(eng, t)
    check_against_oracle(eng, t, abi.PM_MODE_FIRST_FIT)
    eng.close()


def test_no_asks_no_workers_and_nobody_feasible():
    eng = Engine()
    w, a, t = synth_tables(5, 50, "mixed")
    # nobody healthy
    t2 = dict(t)
    wa = t["wa"].copy()
    wa["flags"] &= ~np.uint32(abi.PM_W_HEALTHY)
    t2["wa"] = wa
    load_engine(eng, t2)
    res, og = check_against_oracle(eng, t2, abi.PM_MODE_FIRST_FIT)
    assert res.n_groups == 0 and (res.worker_group == abi.PM_NONE).all()
    # empty ask table
    t3 = dict(t)
    t3["asks"] = t["asks"][:0]
    t3["opts"] = t["opts"][:0]
    load_engine(eng, t3)
    eng.match()
    assert eng.fetch().n_groups == 0
    eng.close()


def test_flag_deltas_and_rematch():
    """pm_set_flags: a worker going Dead / being assigned drops out on the next pass
    (status_update_impl.rs:8-39)."""
    w, a, t = synth_tables(50, 2000, "mixed")
    eng = Engine()
    load_engine(eng, t)
    eng.match()
    r0 = eng.fetch()
    taken = np.flatnonzero(r0.worker_group != abi.PM_NONE)[:100].astype(np.uint32)
    new_flags = (t["wa"]["flags"][taken] | abi.PM_W_ASSIGNED).astype(np.uint32)
    eng.set_flags(taken, new_flags)
    t2 = dict(t)
    wa = t["wa"].copy()
    wa["flags"][taken] = new_flags
    t2["wa"] = wa
    res, og = check_against_oracle(eng, t2, abi.PM_MODE_FIRST_FIT)
    assert (res.worker_group[taken] == abi.PM_NONE).all()
    eng.close()


def test_proximity_solo_groups_order():
    """ProximityOptimizationPolicy enabled with min=max=1: the seed rule orders located
    workers first (mod.rs:526-530)."""
    w, a, t = synth_tables(40, 3000, "mixed")
    eng = Engine()
    load_engine(eng, t, locations=True)
    check_against_oracle(eng, t, abi.PM_MODE_PROXIMITY, proximity=True)
    eng.close()


def test_materialized_and_fused_agree_multi_tile():
    """Zipf prices (many ties in the cost's high word): the fused pass's row minimum is the argmin's, lowest worker
    among the cheapest."""
    w, a, t = synth_tables(5000, 20000, "skewed", price="zipf")
    eng = Engine(cost_tile_bytes=32 << 20)
    load_engine(eng, t)
    eng.match(abi.PM_MODE_FIRST_FIT | MAT)
    r1 = eng.fetch()
    assert r1.stats["n_tiles"] > 1
    assert (r1.ask_best[r1.ask_count > 0] >> 32 >= 1).all()   # every row minimum carries a price
    eng.match(abi.PM_MODE_FIRST_FIT | FUSED)
    r2 = eng.fetch()
    for f in ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count"):
        assert np.array_equal(getattr(r1, f), getattr(r2, f)), f
    eng.close()


def test_cfg2_100k_x_100k_mixed_bit_exact():
    """BASELINE configs[1] at full size: assignment bit-identical to the CPU scheduler."""
    w, a, t = synth_tables(100_000, 100_000, "mixed")
    eng = Engine()
    load_engine(eng, t)
    check_against_oracle(eng, t, abi.PM_MODE_FIRST_FIT, check_rows=False)
    # row results on a sampled band of asks (full 1e10-pair check is minutes of CPU)
    res = eng.fetch()
    for t0 in (0, 50_000, 99_000):
        ev = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], t0, t0 + 1000,
                                 0, 100_000, threads=8)
        assert np.array_equal(res.ask_best[t0:t0 + 1000], ev["row_best"])
        assert np.array_equal(res.ask_count[t0:t0 + 1000], ev["row_count"])
    eng.close()


@pytest.mark.parametrize("path", [MAT, FUSED], ids=["materialized", "fused"])
def test_generic_predicate_path_forced(path, monkeypatch):
    """The fast predicate (operands < 2^31) and the generic one must agree; force the generic."""
    monkeypatch.setenv("PM_TUNE_GENERIC", "1")
    sizes = [(1, 1), (2, 2), (2, 4), (3, 3)]
    w, a, t = synth_tables(400, 5000, "mixed", group_sizes=sizes)
    eng = Engine()
    load_engine(eng, t)
    check_against_oracle(eng, t, abi.PM_MODE_FIRST_FIT | path)
    eng.close()


@pytest.mark.parametrize("path", [MAT, FUSED], ids=["materialized", "fused"])
def test_large_operands_fall_back_to_generic(path):
    """u32 operands >= 2^31, counts >= 2^16 and a wrapping count*memory product: the engine must
    notice (device-side range check) and stay bit-exact (node.rs:509 wraps in release builds)."""
    tb = TableBuilder()
    tb.add_config("ram_mb=3000000000", 1, 1)
    tb.add_config("gpu:count=70000", 1, 1)
    tb.add_config("gpu:total_memory_max=10", 1, 1)
    tb.add_config("gpu:count=2;gpu:memory_mb_min=2500000000", 1, 1)
    tb.add_config("storage_gb=5", 1, 2)
    tb.add_node(kv.specs(1, "A100", 40000, 8, 3500000000, 10))
    tb.add_node(kv.specs(70000, "A100", 10, 8, 1000, 10))
    tb.add_node(kv.specs(65536, "X", 65536, 8, 1000, 10))          # product wraps to 0
    tb.add_node(kv.specs(2, "A100", 3000000000, 8, 1000, 10))
    tb.add_node(kv.specs(2, "A100", 40000, 8, 1000, 10))
    tb.add_node(kv.specs(4, "H100", 80000, 8, 2999999999, 4000000000))
    t = tb.tables()
    eng = Engine()
    load_engine(eng, t)
    res, og = check_against_oracle(eng, t, abi.PM_MODE_FIRST_FIT | path)
    assert res.n_groups >= 4
    eng.close()


def test_fast_and_generic_cost_matrices_identical(monkeypatch):
    w, a, t = synth_tables(600, 3000, "skewed")
    eng = Engine()
    load_engine(eng, t)
    fast = eng.cost_tile(0, 600)
    eng.close()
    monkeypatch.setenv("PM_TUNE_GENERIC", "1")
    eng = Engine()
    load_engine(eng, t)
    generic = eng.cost_tile(0, 600)
    eng.close()
    assert np.array_equal(fast, generic)


@pytest.mark.parametrize("sizes", [[(2, 2)], [(1, 1), (2, 2), (2, 4), (3, 3), (4, 8), (1, 3)]], ids=["pairs", "mixed"])
def test_proximity_groups_general(sizes):
    """ProximityOptimizationPolicy enabled with max_group_size > 1: seed = first located remaining
    node, members = the max-1 nearest by haversine, stable ties (mod.rs:524-552, 218-255)."""
    w, a, t = synth_tables(120, 4000, "mixed", group_sizes=sizes, with_addresses=True, seed_shift=5)
    has_loc = (w.a["flags"] & abi.PM_W_HAS_LOC) != 0
    assert_distance_certificate(w.lat, w.lon, has_loc)        # parity hazard H (SURVEY 8a): no near-ties in this input
    eng = Engine()
    load_engine(eng, t, addr_rank=w.addr_rank, locations=True)
    res, og = check_against_oracle(eng, t, abi.PM_MODE_PROXIMITY, addr_rank=w.addr_rank, proximity=True)
    assert res.n_groups > 50
    eng.close()


def test_proximity_groups_at_100k_workers():
    """The default policy at a production-like size (2000 configurations x 100k workers, mixed group sizes,
    10 815 groups): groups, creation order and members equal the checker's.  The checker runs its latitude-pruned
    mode here (far faster than the literal loop), which tests/test_oracle_groups.py proves equal to the literal loop."""
    sizes = [(1, 1), (2, 2), (2, 4), (3, 3), (4, 8), (1, 3)]
    w, a, t = synth_tables(2000, 100_000, "mixed", group_sizes=sizes)
    eng = Engine()
    load_engine(eng, t, locations=True)
    eng.match(abi.PM_MODE_PROXIMITY)
    res = eng.fetch()
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], lat=t["lat"], lon=t["lon"],
                             proximity="banded")
    assert groups_equal(res, og), f"groups differ: engine {res.n_groups} vs checker {len(og)}"
    assert res.n_groups == 10815
    eng.close()


def test_proximity_montreal_dallas_on_device():
    """The coordinates of node_groups/tests.rs:2861-3064: interleaved arrivals still pair by city."""
    tb = TableBuilder()
    tb.add_config(None, 2, 2)
    A6000 = kv.specs(1, "nvidia rtx a6000", 49140)
    MONTREAL, DALLAS = (45.5186, -73.5545), (32.7942, -96.7475)
    for loc in (MONTREAL, DALLAS, MONTREAL, DALLAS):
        tb.add_node(A6000, location=loc)
    t = tb.tables()
    eng = Engine()
    load_engine(eng, t, locations=True)
    eng.match(abi.PM_MODE_PROXIMITY)
    res = eng.fetch()
    assert sorted(sorted(m) for _, m in res.groups()) == [[0, 2], [1, 3]]
    eng.close()


def test_asks_sharing_option_rows():
    """Several asks may point at the same option rows (identical requirements written once): the device
    table gets one private range per ask, which can be longer than the caller's table."""
    w, a, t = synth_tables(30, 4000, "mixed", group_sizes=[(1, 1), (1, 2), (2, 4)])
    rng = np.random.default_rng(11)
    idx = rng.permutation(np.repeat(np.arange(30), 25))
    t["asks"] = np.ascontiguousarray(t["asks"][idx])
    assert int(t["asks"]["n_opts"].sum()) > len(t["opts"])
    for mode in (abi.PM_MODE_FIRST_FIT | MAT, abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED):
        eng = Engine(cost_tile_bytes=8 << 20)
        load_engine(eng, t)
        check_against_oracle(eng, t, mode)
        eng.close()


# ------------------------------------------------------------------------------------------------
# NORTH-STAR EXTENSION (no reference counterpart): parity is against the builder's own sequential
# auction — "self-oracle, parity unpinned by the reference" (SURVEY 0, 8c).
def _auction_tables(n_asks, n_workers, seed):
    w, a, t = synth_tables(n_asks, n_workers, "mixed", seed_shift=seed)
    rng = np.random.default_rng(seed)
    wb = t["wb"].copy()
    wb["ext_ask_price"] = rng.integers(10, 1000, n_workers).astype(np.uint32)
    t["wb"] = wb
    cap = rng.integers(50, 1500, n_asks).astype(np.uint32)
    return t, cap


@pytest.mark.parametrize("n_asks,n_workers,seed", [(1, 5, 1), (50, 700, 2), (300, 2500, 3), (64, 1025, 4)])
def test_extension_auction_matches_self_oracle(n_asks, n_workers, seed):
    t, cap = _auction_tables(n_asks, n_workers, seed)
    eng = Engine()
    load_engine(eng, t)
    eng.set_price_caps(cap)
    eng.match(abi.PM_MODE_AUCTION)
    res = eng.fetch()
    want, price, rounds = orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    got = np.full(n_asks, abi.PM_NONE, dtype=np.uint32)
    for g, (ask, members) in enumerate(res.groups()):
        assert len(members) == 1
        got[ask] = members[0]
    assert np.array_equal(got, want)
    assert res.stats["n_rounds"] == rounds
    # every assignment respects feasibility and the cap; no worker is used twice
    used = got[got != abi.PM_NONE]
    assert len(set(used.tolist())) == len(used)
    for tk in np.flatnonzero(got != abi.PM_NONE):
        wk = got[tk]
        assert t["wb"]["ext_ask_price"][wk] <= cap[tk]
        assert orc.soa_compatible(t["wa"][wk], t["wb"][wk], t["asks"][tk], t["opts"], t["bits"], t["words"])
    eng.close()


def _tuned_engine(tune):
    """PM_TUNE_AUCTION is read at pm_create (see DESIGN.md 4)."""
    if tune:
        os.environ["PM_TUNE_AUCTION"] = str(tune)
    try:
        return Engine()
    finally:
        os.environ.pop("PM_TUNE_AUCTION", None)


def _check_auction(t, cap, tunes=(0,), **params):
    want, price, rounds = orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap, **params)
    for tune in tunes:
        eng = _tuned_engine(tune)
        load_engine(eng, t)
        eng.set_price_caps(cap)
        if params:
            eng.set_auction_params(**params)
        eng.match(abi.PM_MODE_AUCTION)
        res = eng.fetch()
        got = np.full(len(cap), abi.PM_NONE, dtype=np.uint32)
        for g, (ask, members) in enumerate(res.groups()):
            assert len(members) == 1
            got[ask] = members[0]
        assert np.array_equal(got, want), tune
        assert res.stats["n_rounds"] == rounds, tune
        stats = res.stats
        eng.close()
    return got, stats


@pytest.mark.parametrize("n_base,copies,n_workers,plo,phi,seed", [
    (12, 40, 3000, 10, 14, 5),      # few classes, many identical bidders, almost every value tied
    (40, 20, 5000, 10, 40, 6),
    (25, 30, 20000, 5, 300, 7),     # 20 stripes: the price-sorted scan stops early
    (3, 200, 2500, 7, 9, 8),        # caps straddle the whole price range: ties exactly at the outside option
])
def test_extension_auction_identical_bidders_and_ties(n_base, copies, n_workers, plo, phi, seed):
    """Ask classes share one cache; the cap only enters through the outside option.  Duplicated asks with
    different caps over a narrow integer price range hit every tie rule (equal values -> lowest worker,
    equal bids -> lowest ask, value == outside) — assignments and round count must still equal the
    sequential checker's, which scans every worker for every unassigned ask every round."""
    w, a, t = synth_tables(n_base, n_workers, "mixed", seed_shift=seed)
    rng = np.random.default_rng(seed)
    idx = rng.permutation(np.repeat(np.arange(n_base), copies))
    t["asks"] = np.ascontiguousarray(t["asks"][idx])     # duplicates share their option rows
    wb = t["wb"].copy()
    wb["ext_ask_price"] = rng.integers(plo, phi + 1, n_workers).astype(np.uint32)
    t["wb"] = wb
    cap = rng.integers(max(plo - 2, 0), phi + 3, len(idx)).astype(np.uint32)
    got, stats = _check_auction(t, cap)
    # classes were scanned, not asks: at least one walk per distinct requirement row, far fewer than one per bid
    n_classes = len({(int(r["flags"]), int(r["cpu_cores"]), int(r["ram_mb"]), int(r["storage_gb"]),
                      t["opts"][r["opt_off"]:r["opt_off"] + r["n_opts"]].tobytes()) for r in t["asks"]})
    assert n_classes <= stats["n_tiles"] <= n_classes * max(stats["n_rounds"], 1)


@pytest.mark.parametrize("tune", [1, 2, 8, 16, 32, 64, 128, 8 | 32, 64 | 32, 1 | 64, 128 | 32, 0x200, 0x100 | 16])
def test_extension_auction_every_shortcut_can_be_switched_off(tune):
    """PM_TUNE_AUCTION bits: 1 walks never stop early, 2 every ask scans for itself (the checker's algorithm on the device),
    8 no class pool, 16 pool re-ranked but never trusted, 32 walks never split, 64 walks start at the top of the table
    (no skip to the class's cost level), 128 selections sort (value, worker) pairs instead of packed 64-bit keys,
    bits 8+ batches between re-sorts of the worker copy.  Every setting must give the checker's assignment and round count."""
    w, a, t = synth_tables(25, 20000, "mixed", seed_shift=7)
    rng = np.random.default_rng(70)
    idx = rng.permutation(np.repeat(np.arange(25), 20))
    t["asks"] = np.ascontiguousarray(t["asks"][idx])
    wb = t["wb"].copy()
    wb["ext_ask_price"] = rng.integers(5, 120, 20000).astype(np.uint32)
    t["wb"] = wb
    cap = rng.integers(3, 140, len(idx)).astype(np.uint32)
    _check_auction(t, cap, tunes=(tune,))


def test_extension_auction_scarce_and_broad_classes_side_by_side():
    """60k workers: classes with a handful, a few thousand and tens of thousands of compatible workers in one market
    (59 stripes: pooled classes, early exits, split walks); more asks than scarce workers, so the scarce classes fight
    to their caps."""
    w, a, t = synth_tables(60, 60000, "mixed", seed_shift=17)
    rng = np.random.default_rng(170)
    idx = rng.permutation(np.repeat(np.arange(60), 30))
    t["asks"] = np.ascontiguousarray(t["asks"][idx])
    wb = t["wb"].copy()
    wb["ext_ask_price"] = rng.integers(10, 60, 60000).astype(np.uint32)
    t["wb"] = wb
    cap = rng.integers(8, 70, len(idx)).astype(np.uint32)
    ev = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], 0, len(idx), 0, 60000, want_cols=False)
    counts = ev["row_count"]
    assert (counts <= 8192).any() and (counts > 8192).any() and ((counts > 32) & (counts <= 8192)).any()
    _check_auction(t, cap)


@pytest.mark.parametrize("params", [dict(cost_scale=3), dict(cost_scale=4, eps_start=16, eps_div=4),
                                    # a first eps beyond 2^40: bids can exceed what a packed sort key holds, the selections
                                    # sort (value, worker) pairs (decided on the device, pm_auction_decide_packed)
                                    dict(cost_scale=1, eps_start=1 << 41, eps_div=1 << 20)])
def test_extension_auction_scaled_costs_and_eps_phases(params):
    t, cap = _auction_tables(300, 2500, 9)
    _check_auction(t, cap, **params)


def test_extension_auction_cfg3_100k_x_1m_properties():
    """BASELINE configs[2] names a price-capped auction at 100k asks x 1M workers.  The sequential checker cannot run at
    this size (it scans every worker for every unassigned ask every round), so the full-size run is held to what can be
    checked from the assignment alone: nobody is sold twice, every sale respects the cap and the requirements
    (sampled against the oracle predicate), and the run terminates with far fewer table walks than bids."""
    T, W = 100_000, 1_000_000
    w, a, t = synth_tables(T, W, "mixed")
    wb = t["wb"].copy()
    wb["ext_ask_price"] = np.exp(np.log(10) + synth._unit(synth.SEED_EXT, W, 1) * np.log(200)).astype(np.uint32)
    t["wb"] = wb
    cap = np.exp(np.log(20) + synth._unit(synth.SEED_EXT, T, 2) * np.log(150)).astype(np.uint32)
    eng = Engine()
    load_engine(eng, t)
    eng.set_price_caps(cap)
    eng.match(abi.PM_MODE_AUCTION)
    res = eng.fetch()
    st = res.stats
    ask_of_group = res.group_ask
    sold = res.group_members
    assert len(sold) == res.n_groups == len(ask_of_group) and res.n_groups > T // 2
    assert len(np.unique(sold)) == len(sold) and len(np.unique(ask_of_group)) == len(ask_of_group)
    assert np.all(wb["ext_ask_price"][sold] <= cap[ask_of_group])
    rng = np.random.default_rng(3)
    for g in rng.choice(res.n_groups, 300, replace=False):
        tk, wk = int(ask_of_group[g]), int(sold[g])
        assert orc.soa_compatible(t["wa"][wk], t["wb"][wk], t["asks"][tk], t["opts"], t["bits"], t["words"])
    assert st["n_rounds"] > 0 and st["n_tiles"] < 100 * st["n_rounds"]     # ~30 table walks per round, 12.4k classes
    eng.close()


def _check_auction_rep(t, cap, reputation, floors, tunes=(0,), **params):
    want, price, rounds = orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap,
                                          reputation=reputation, min_reputation=floors, **params)
    for tune in tunes:
        eng = _tuned_engine(tune)
        load_engine(eng, t)
        eng.set_price_caps(cap)
        if reputation is not None:
            eng.set_worker_reputation(reputation)
        if floors is not None:
            eng.set_min_reputation(floors)
        if params:
            eng.set_auction_params(**params)
        eng.match(abi.PM_MODE_AUCTION)
        res = eng.fetch()
        got = np.full(len(cap), abi.PM_NONE, dtype=np.uint32)
        for ask, members in res.groups():
            assert len(members) == 1
            got[ask] = members[0]
        assert np.array_equal(got, want), tune
        assert res.stats["n_rounds"] == rounds, tune
        eng.close()
    return got


@pytest.mark.parametrize("n_asks,n_workers,seed", [(50, 700, 12), (300, 2500, 13), (64, 1025, 14), (400, 20000, 15)])
def test_extension_auction_reputation_floor_matches_self_oracle(n_asks, n_workers, seed):
    """north_star worker column `reputation`: a pair is feasible only when reputation[w] >= the ask's floor.  The floor
    is part of the ask's class (two asks with the same requirement row and different floors do not share a cache)."""
    t, cap = _auction_tables(n_asks, n_workers, seed)
    rng = np.random.default_rng(seed)
    reputation = rng.integers(0, 1000, n_workers).astype(np.uint32)
    floors = np.where(rng.random(n_asks) < 0.5, 0, rng.integers(1, 1100, n_asks)).astype(np.uint32)
    got = _check_auction_rep(t, cap, reputation, floors)
    sold = got != abi.PM_NONE
    assert np.all(reputation[got[sold]] >= floors[sold])
    assert not np.any(sold & (floors > reputation.max()))          # a floor nobody reaches: the ask withdraws
    # the clause bites: without it the same market sells differently
    want0, _, _ = orc.soa_auction(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], cap)
    assert not np.array_equal(got, want0)


def test_extension_auction_reputation_duplicated_asks_and_ties():
    """Duplicated requirement rows that differ ONLY in the floor, narrow price range (every tie rule), few reputation levels."""
    w, a, t = synth_tables(10, 3000, "mixed", seed_shift=21)
    rng = np.random.default_rng(21)
    idx = rng.permutation(np.repeat(np.arange(10), 40))
    t["asks"] = np.ascontiguousarray(t["asks"][idx])
    wb = t["wb"].copy()
    wb["ext_ask_price"] = rng.integers(10, 15, 3000).astype(np.uint32)
    t["wb"] = wb
    cap = rng.integers(8, 18, len(idx)).astype(np.uint32)
    reputation = rng.integers(0, 4, 3000).astype(np.uint32)
    floors = rng.integers(0, 5, len(idx)).astype(np.uint32)
    _check_auction_rep(t, cap, reputation, floors)
    _check_auction_rep(t, cap, reputation, floors, cost_scale=3)


def test_extension_auction_reputation_defaults_are_inert():
    """No floor -> the worker column is never read; a floor without a worker column is a column of zeros."""
    t, cap = _auction_tables(120, 1500, 31)
    rng = np.random.default_rng(31)
    reputation = rng.integers(0, 100, 1500).astype(np.uint32)
    base = _check_auction_rep(t, cap, None, None)
    assert np.array_equal(_check_auction_rep(t, cap, reputation, None), base)
    assert np.array_equal(_check_auction_rep(t, cap, reputation, np.zeros(120, dtype=np.uint32)), base)
    floors = np.zeros(120, dtype=np.uint32)
    floors[::3] = 1
    got = _check_auction_rep(t, cap, None, floors)
    assert np.all(got[::3] == abi.PM_NONE)
    # reference modes ignore both columns
    eng = Engine()
    load_engine(eng, t)
    eng.match()
    r0 = eng.fetch()
    eng.set_worker_reputation(reputation)
    eng.set_min_reputation(floors)
    eng.match()
    r1 = eng.fetch()
    for f in ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_count"):
        assert np.array_equal(getattr(r0, f), getattr(r1, f)), f
    eng.close()


def test_extension_columns_are_neutral_in_reference_modes():
    """ext_ask_price only occupies the high word of the packed cost; groups do not depend on it."""
    w, a, t = synth_tables(200, 3000, "mixed")
    eng = Engine()
    load_engine(eng, t)
    eng.match()
    r0 = eng.fetch()
    t2 = dict(t)
    wb = t["wb"].copy()
    wb["ext_ask_price"] = 7
    t2["wb"] = wb
    load_engine(eng, t2)
    eng.match()
    r1 = eng.fetch()
    for f in ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_count"):
        assert np.array_equal(getattr(r0, f), getattr(r1, f)), f
    eng.close()


def test_cfg3_100k_x_1m_properties():
    """BASELINE configs[2] shape at full size (10^11 pairs: too many for an exhaustive CPU check) through
    size-independent properties: materialised == fused bit for bit; every assignment is a compatible,
    candidate pair (sampled against the oracle predicate); nobody is assigned twice; a worker's ask is the
    FIRST compatible ask (sampled); the pass is idempotent once its groups are marked assigned."""
    T, W = 100_000, 1_000_000
    w, a, t = synth_tables(T, W, "mixed")
    eng = Engine()
    load_engine(eng, t)
    eng.match(abi.PM_MODE_FIRST_FIT | MAT)
    r1 = eng.fetch()
    assert r1.stats["evals"] == T * W and r1.stats["n_tiles"] > 50
    eng.match(abi.PM_MODE_FIRST_FIT | FUSED)
    r2 = eng.fetch()
    for f in ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count"):
        assert np.array_equal(getattr(r1, f), getattr(r2, f)), f
    assigned = np.flatnonzero(r1.worker_ask != abi.PM_NONE)
    assert len(np.unique(r1.group_members)) == len(r1.group_members) == len(assigned)
    cand = (t["wa"]["flags"] & (abi.PM_W_HEALTHY | abi.PM_W_P2P | abi.PM_W_ASSIGNED)) == (abi.PM_W_HEALTHY | abi.PM_W_P2P)
    assert cand[assigned].all()
    rng = np.random.default_rng(0)
    for wk in rng.choice(assigned, 300, replace=False):
        tk = int(r1.worker_ask[wk])
        assert orc.soa_compatible(t["wa"][wk], t["wb"][wk], t["asks"][tk], t["opts"], t["bits"], t["words"])
        for earlier in rng.integers(0, max(tk, 1), 5):            # no earlier ask accepts the worker
            if earlier < tk:
                assert not orc.soa_compatible(t["wa"][wk], t["wb"][wk], t["asks"][int(earlier)], t["opts"], t["bits"], t["words"])
    unassigned_cand = np.flatnonzero(cand & (r1.worker_ask == abi.PM_NONE))
    for wk in rng.choice(unassigned_cand, 20, replace=False):     # left over => no ask at all accepts it
        for tk in rng.integers(0, T, 50):
            assert not orc.soa_compatible(t["wa"][wk], t["wb"][wk], t["asks"][int(tk)], t["opts"], t["bits"], t["words"])
    # per-ask counts add up: every candidate-compatible pair is counted once
    band = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], 500, 520, 0, W, threads=8)
    assert np.array_equal(r1.ask_count[500:520], band["row_count"]) and np.array_equal(r1.ask_best[500:520], band["row_best"])
    # idempotence: mark the formed groups' members assigned -> the next pass forms nothing
    idx = assigned.astype(np.uint32)
    eng.set_flags(idx, (t["wa"]["flags"][idx] | abi.PM_W_ASSIGNED).astype(np.uint32))
    eng.match(abi.PM_MODE_FIRST_FIT | MAT)
    assert eng.fetch().n_groups == 0
    eng.close()


def test_fused_lean_gives_the_same_groups():
    """PM_NO_ASK_STATS: same assignment, per-ask statistics skipped."""
    sizes = [(1, 1), (2, 2), (2, 4)]
    w, a, t = synth_tables(500, 8000, "mixed", group_sizes=sizes)
    eng = Engine()
    load_engine(eng, t)
    eng.match(abi.PM_MODE_FIRST_FIT)
    r1 = eng.fetch()
    eng.match(abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS)
    r2 = eng.fetch()
    for f in ("worker_group", "worker_ask", "group_ask", "group_off", "group_members"):
        assert np.array_equal(getattr(r1, f), getattr(r2, f)), f
    assert (r2.ask_count == 0).all() and (r2.ask_best == abi.PM_COST_INF).all()
    eng.close()


def skewed_tables(T, W, seed_shift=0):
    """BASELINE configs[3]/[4] columns (SURVEY 8d): mixed asks with 10 % made infeasible (gpu:count = 3), worker
    ask prices Zipf(1.1) over 1024 levels in the extension column (the high word of the packed cost)."""
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + seed_shift, price="zipf")
    a = synth.make_asks(T, "skewed", seed=synth.SEED_ASKS + seed_shift)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    return w, a, dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod,
                      words=words, lat=w.lat, lon=w.lon)


def test_one_million_asks_full_groups_at_20k_workers():
    """T = 1M (BASELINE configs[3]/[4] ask count), Zipf prices, 10 % infeasible asks, against the oracle's
    per-configuration loop (orc_soa_form_groups) — complete group table, both evaluation paths."""
    T, W = 1_000_000, 20_000
    w, a, t = skewed_tables(T, W, seed_shift=41)
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"])
    eng = Engine(cost_tile_bytes=1 << 30)
    load_engine(eng, t)
    for path in (MAT, FUSED, FUSED | abi.PM_NO_ASK_STATS):
        eng.match(abi.PM_MODE_FIRST_FIT | path)
        res = eng.fetch()
        assert groups_equal(res, og)
    eng.close()


def test_cfg4_shape_one_million_asks_x_250k_workers():
    """The per-GPU shape of BASELINE configs[3] (1M asks x 1M workers over 4 GPUs): every worker's configuration
    against the oracle's first-feasible search (with solo configurations that IS try_form_new_groups' allocation,
    mod.rs:505-609), sampled rows of the per-ask (min cost, argmin) and counts with prices in the cost's high word,
    every infeasible ask empty, group table consistent with the per-worker view."""
    import os
    T, W = 1_000_000, 250_000
    w, a, t = skewed_tables(T, W)
    eng = Engine()
    load_engine(eng, t)
    eng.match(abi.PM_MODE_FIRST_FIT | MAT)
    r1 = eng.fetch()
    assert r1.stats["evals"] == T * W
    threads = max(1, len(os.sched_getaffinity(0)))
    first = orc.soa_first_feasible(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], threads=threads)
    assert np.array_equal(r1.worker_ask, first)
    # groups: one per assigned worker, creation order = (configuration, canonical worker order)
    assigned = np.flatnonzero(first != abi.PM_NONE)
    order = assigned[np.argsort(first[assigned], kind="stable")]
    assert r1.n_groups == len(order) and np.array_equal(r1.group_members, order.astype(np.uint32))
    assert np.array_equal(r1.group_ask, first[order]) and np.array_equal(r1.group_off, np.arange(len(order) + 1, dtype=np.uint32))
    assert np.array_equal(r1.worker_group[order], np.arange(len(order), dtype=np.uint32))
    # infeasible asks (gpu:count = 3 on every option) see nobody
    infeasible = np.flatnonzero(np.minimum.reduceat((a.opts["count"] == 3).astype(np.uint8), a.asks["opt_off"].astype(np.int64)) == 1)
    assert 0.08 * T < len(infeasible) < 0.12 * T
    assert (r1.ask_count[infeasible] == 0).all() and (r1.ask_best[infeasible] == abi.PM_COST_INF).all()
    # sampled rows, prices included: argmin is the cheapest compatible candidate, lowest index on ties
    rng = np.random.default_rng(4)
    for t0 in rng.integers(0, T - 16, 12):
        band = orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], int(t0), int(t0) + 16, 0, W, threads=threads)
        assert np.array_equal(r1.ask_count[t0:t0 + 16], band["row_count"]) and np.array_equal(r1.ask_best[t0:t0 + 16], band["row_best"])
    feasible_best = r1.ask_best[r1.ask_best != abi.PM_COST_INF]
    assert ((feasible_best >> 32) >= 1).all() and ((feasible_best >> 32) <= 1024).all()
    # the other paths agree bit for bit
    eng.match(abi.PM_MODE_FIRST_FIT | FUSED)
    r2 = eng.fetch()
    for f in ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count"):
        assert np.array_equal(getattr(r1, f), getattr(r2, f)), f
    eng.close()


def test_extension_auction_against_scipy_at_2k_x_2k():
    """An anchor that is not this repo's code (VERDICT r1): at 2000 asks x 2000 workers the engine's auction (default
    parameters: cost_scale 1, eps 1) must land within T * eps of scipy.optimize.linear_sum_assignment's optimum on the
    feasibility-masked, cap-filtered cost matrix (unassigned asks pay their outside option cap + 1)."""
    from scipy.optimize import linear_sum_assignment

    T = W = 2000
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + 31, price="loguniform")
    a = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS + 31)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)
    cap = np.exp(np.log(20) + synth._unit(synth.SEED_EXT + 31, T, 3) * np.log(60)).astype(np.uint32)
    eng = Engine()
    load_engine(eng, t)
    eng.set_price_caps(cap)
    eng.match(abi.PM_MODE_AUCTION)
    res = eng.fetch()
    eng.close()
    got = np.full(T, abi.PM_NONE, dtype=np.uint32)
    for ask, members in res.groups():
        got[ask] = members[0]
    price = w.b["ext_ask_price"].astype(np.int64)
    feasible = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, bits, words, 0, T, 0, W, threads=8, want_cost=True)["cost"] != abi.PM_COST_INF
    ok = feasible & (price[None, :] <= cap[:, None])
    BIG = 1 << 40
    C = np.full((T, W + T), BIG, dtype=np.int64)
    C[:, :W][ok] = np.broadcast_to(price[None, :], (T, W))[ok]
    C[np.arange(T), W + np.arange(T)] = cap.astype(np.int64) + 1
    r, c = linear_sum_assignment(C)
    opt = int(C[r, c].sum())
    sold = np.flatnonzero(got != abi.PM_NONE)
    assert ok[sold, got[sold]].all() and len(np.unique(got[sold])) == len(sold)
    total = int(price[got[sold]].sum() + (cap.astype(np.int64) + 1)[got == abi.PM_NONE].sum())
    assert opt <= total <= opt + T, (opt, total)
