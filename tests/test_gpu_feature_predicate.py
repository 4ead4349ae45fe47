"""pm_build_argmin_feat, the materialised pass's build + argmin on the feature predicate, on hardware: against the
int64 tile (PM_TUNE_BUILD=8: separate build and argmin launches on the fast predicate) and the CPU oracle, every result
array whole.  Tables at exactly 64 features run it and at 65 run the FastRow pm_build_argmin; ask deltas move a
resident engine across that budget both ways; the kernel that ran is read from the kernel names torch.profiler
records."""
import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import feature_tables as ft
from helpers import load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi
from protocol_b200.engine import Engine
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_gpu_narrow_tile import MAT, RESULT_FIELDS, assert_same, make_engine
from test_gpu_tile_overlap import tile_bytes
from test_gpu_tile_pipeline import assert_oracle, table_dict
from test_gpu_variants import wide_tables

pytestmark = pytest.mark.gpu

FEAT, FASTROW = "feature", "fastrow"


def build_kernels(names):
    """Which build + argmin kernels ran, from the kernel names of a trace."""
    out = set()
    for n in names:
        if "pm_build_argmin_feat" in n:
            out.add(FEAT)
        elif "pm_build_argmin<" in n:
            out.add(FASTROW)
    return out


def profiled_match(e):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.match_local(MAT)
        e.sync()
    return build_kernels(ev.name for ev in prof.events())


def pass_arrays(e, W, T):
    fa, best, cnt = (x.cpu().numpy().copy() for x in wrap_device_buffers(e, W, T))
    return fa.view(np.uint32), best, cnt.view(np.uint32)


def check(t, cost_tile_bytes=1 << 20, shard=None):
    got = assert_same(t, cost_tile_bytes, shard)
    if shard is None:
        assert_oracle(t, got)
    else:
        assert_oracle(t, got, shard[0], shard[0] + shard[1])
    return got


def kernel_of(t, cost_tile_bytes=1 << 20):
    e = Engine(cost_tile_bytes=cost_tile_bytes)
    try:
        load_engine(e, t)
        e.match_local(MAT)   # warm: modules loaded, tables converted
        e.sync()
        return profiled_match(e)
    finally:
        e.close()


@pytest.mark.parametrize("n", [64, 65])
def test_tables_at_the_feature_budget(n):
    t = ft.with_features(ft.edge_tables(21, 700, 5000), n)
    check(t)
    assert kernel_of(t) == ({FEAT} if n <= 64 else {FASTROW})


@pytest.mark.parametrize("seed,T,W", [(0, 1, 1), (1, 513, 1023), (2, 1025, 1025), (3, 700, 4099), (4, 2000, 3000)])
def test_edge_values(seed, T, W):
    """Thresholds 0, 1 and 0x7FFFFFFE, lo == hi, empty intervals, workers without count or memory, OR-options next
    to scalar clauses, asks without options, max_group_size == 0; ragged CTA stripes and row bands."""
    t = ft.edge_tables(seed, T, W)
    assert ft.n_features(t) <= 64
    got = check(t)
    assert (got[2] > 0).any() or W == 1


@pytest.mark.parametrize("T,W,rows", [(1100, 4099, 256), (2500, 2000, 1024), (613, 6007, 21)])
def test_several_tiles_with_a_ragged_last_one(T, W, rows):
    check(ft.edge_tables(T + W, T, W), tile_bytes(W, rows))


@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_ranges(n_shards):
    t = ft.edge_tables(40 + n_shards, 900, 10007)
    W = len(t["wa"])
    for r in range(n_shards):
        lo, hi = shard_range(W, n_shards, r)
        check(t, tile_bytes(hi - lo, 256), shard=(lo, hi - lo))


@pytest.mark.parametrize("n_models,n_patterns", [(30, 20), (200, 30), (3000, 30), (100000, 12)],
                         ids=["bits2", "bits1", "worker_major", "wide_catalogue"])
def test_acceptance_forms(n_models, n_patterns):
    """Model features from a one-word table, a shared-memory one, the worker-major word and a wide catalogue."""
    w, a, obits, pbits, npat, nmod, words = wide_tables(600, 6000, n_models=n_models, n_patterns=n_patterns,
                                                        seed_shift=90 + n_patterns, last_rows=True)
    t = table_dict(w, a, pbits, npat, nmod, words)
    assert ft.n_features(t) <= 64
    check(t)
    assert kernel_of(t) == {FEAT}


def test_asks_with_hundreds_of_options():
    """Asks with 300 and 700 OR-options over the dictionary's few thresholds, between ordinary asks."""
    t = ft.edge_tables(77, 400, 5000, max_opts=2)
    rng = np.random.default_rng(3)
    asks, opts = t["asks"].copy(), [t["opts"]]
    n = len(t["opts"])
    for i, k in ((37, 300), (211, 700)):
        o = np.zeros(k, dtype=abi.GPU_OPT)
        o["present"] = abi.PM_O_COUNT | abi.PM_O_MODEL | abi.PM_O_MEM_MIN
        o["count"] = rng.choice([1, 2, 4, 8], k)
        o["memory_mb_min"] = rng.choice([24000, 40000, 80000], k)
        o["pattern_id"] = rng.integers(0, t["n_patterns"], k)
        asks[i]["flags"] = abi.PM_A_HAS_REQ | abi.PM_A_REQ_RAM
        asks[i]["n_opts"], asks[i]["opt_off"], asks[i]["max_group_size"], asks[i]["min_group_size"] = k, n, 1, 1
        opts.append(o)
        n += k
    t = dict(t, asks=asks, opts=np.concatenate(opts))
    assert ft.n_features(t) <= 64
    got = check(t)
    assert got[2][37] > 0 and got[2][211] > 0


def history_step(engines, t, enabled=None):
    """One pass on each engine (default, int64 tile): every array equal, and to the oracle when every ask is enabled;
    returns the build kernels the default engine ran."""
    W, T = len(t["wa"]), len(t["asks"])
    ran = profiled_match(engines[0])
    engines[1].match_local(MAT)
    engines[1].sync()
    got, ref = (pass_arrays(e, W, T) for e in engines)
    for x, y in zip(got, ref):
        assert np.array_equal(x, y)
    if enabled is None:
        assert_oracle(t, got)
    res = []
    for e in engines:
        e.match_finish(MAT)
        res.append(e.fetch())
    for f in RESULT_FIELDS:
        assert np.array_equal(getattr(res[0], f), getattr(res[1], f)), f
    return ran


def test_deltas_across_the_budget_and_model_table_changes():
    base = ft.edge_tables(55, 800, 6000)
    big = ft.with_features(base, 65)
    fit = ft.with_features(base, 64)
    added = big["asks"][len(base["asks"]):]
    engines = [make_engine(wide, cost_tile_bytes=1 << 20) for wide in (False, True)]
    try:
        for e in engines:
            load_engine(e, fit)
        assert history_step(engines, fit) == {FEAT}
        for e in engines:   # past the budget: the FastRow kernel
            e.resize_asks(len(base["asks"]))
            e.resize_asks(len(big["asks"]), added)
        assert history_step(engines, big) == {FASTROW}
        for e in engines:   # and back
            e.resize_asks(len(fit["asks"]))
        assert history_step(engines, fit) == {FEAT}
        # a replaced row whose thresholds are new, within the budget
        row = fit["asks"][-1:].copy()
        row["cpu_cores"] = 7_777_777
        fit2 = dict(fit, asks=np.concatenate([fit["asks"][:-1], row]))
        for e in engines:
            e.update_asks(np.array([len(fit["asks"]) - 1], dtype=np.uint32), row)
        assert history_step(engines, fit2) == {FEAT}
        # toggles set the never bit, a feature every dictionary holds
        on = np.random.default_rng(8).random(len(fit2["asks"])) > .25
        for e in engines:
            e.set_ask_enabled(np.flatnonzero(~on).astype(np.uint32), False)
        assert history_step(engines, fit2, on) == {FEAT}
        for e in engines:
            e.set_ask_enabled(np.flatnonzero(~on).astype(np.uint32), True)
        # a new acceptance table between passes: the model features follow it
        rng = np.random.default_rng(9)
        bits = rng.integers(0, 1 << 32, size=fit2["bits"].shape, dtype=np.uint64).astype(np.uint32)
        if fit2["n_models"] % 32:
            bits.reshape(fit2["n_patterns"], -1)[:, -1] &= np.uint32((1 << (fit2["n_models"] % 32)) - 1)
        fit3 = dict(fit2, bits=bits)
        for e in engines:
            e.set_model_table(bits, fit3["n_patterns"], fit3["n_models"], fit3["words"])
        assert history_step(engines, fit3) == {FEAT}
    finally:
        for e in engines:
            e.close()


def test_groups_equal_the_oracle_on_the_feature_path():
    t = ft.edge_tables(99, 1500, 8000)
    e = Engine(cost_tile_bytes=1 << 22)
    try:
        load_engine(e, t)
        e.match(MAT)
        res = e.fetch()
    finally:
        e.close()
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"])
    assert np.array_equal(res.group_ask, og.cfg)
    assert np.array_equal(res.group_off, og.off) and np.array_equal(res.group_members, og.members)
