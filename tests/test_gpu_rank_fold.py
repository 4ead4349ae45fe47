"""pm_build_argmin's register fold on hardware: the per-stripe price rank (pm_stripe_rank) and the per-row fold of
(least rank, feasible count), against the int64 tile (PM_TUNE_BUILD=8) and the CPU oracle.

The rank table is computed from the prices at every pass.  The cases aim at what a stale or misread table would get
wrong: prices changed by pm_update_workers between two passes with no host synchronisation in between, the worker
table resized (ld changes), equal least prices only in the last warp / last lane of a stripe, worker counts one either
side of a 1024-column stripe (padding columns rank last) and a shard whose first worker w0 is not a stripe multiple."""
import numpy as np
import pytest

from helpers import load_engine
from protocol_b200 import abi
from protocol_b200.engine import _ptr
from protocol_b200.sharded import wrap_device_buffers
from test_gpu_narrow_tile import MAT, assert_same, make_engine, oracle_eval, tables
from test_gpu_tile_overlap import tile_bytes
from test_gpu_tile_pipeline import assert_oracle

pytestmark = pytest.mark.gpu


def passes_across_an_update(t, idx, a, b, wide, resize=None):
    """Pass 1, pm_update_workers (and pm_resize_workers first when `resize`) and pass 2, enqueued with no host
    synchronisation between them; returns pass 2's (first_ask, ask_best, ask_count, stats)."""
    W = resize if resize is not None else len(t["wa"])
    T = len(t["asks"])
    e = make_engine(wide, cost_tile_bytes=tile_bytes(W, 256))
    try:
        load_engine(e, t)
        e.match_local(MAT)
        if resize is not None:
            e.resize_workers(resize)
        # the raw entry point: Engine.update_workers would synchronise the stream
        assert e._lib.pm_update_workers(e._h, _ptr(idx), _ptr(a), _ptr(b), None, None, len(idx)) == abi.PM_OK
        e.match_local(MAT)
        e.sync()
        fa, best, cnt = (x.cpu().numpy().copy() for x in wrap_device_buffers(e, W, T))
        st = e.stats()
    finally:
        e.close()
    return fa.view(np.uint32), best, cnt.view(np.uint32), st


def check_update(t, t2, idx, a, b, resize=None):
    ref = passes_across_an_update(t, idx, a, b, True, resize)
    got = passes_across_an_update(t, idx, a, b, False, resize)
    for x, y in zip(got[:3], ref[:3]):
        assert np.array_equal(x, y)
    assert got[3]["cost_bytes_written"] == got[3]["cost_bytes_read"] == 4 * len(t2["asks"]) * len(t2["wa"])
    assert ref[3]["cost_bytes_written"] == ref[3]["cost_bytes_read"] == 8 * len(t2["asks"]) * len(t2["wa"])
    ev = assert_oracle(t2, got)
    assert (ev["row_count"] > 0).any()


@pytest.mark.parametrize("kind", ["cheapest", "dearest"])
def test_prices_changed_between_passes(kind):
    """Pass 2's least worker changes: the changed rows become the cheapest of the table, or the former cheapest
    become the dearest.  A rank table left from pass 1 would pick pass 1's worker."""
    W, T = 5000, 600
    t = tables(T, W, seed_shift=31)
    price = t["wb"]["ext_ask_price"]
    rng = np.random.default_rng(7)
    if kind == "cheapest":
        idx = np.sort(rng.choice(W, 400, replace=False)).astype(np.uint32)
        new = np.zeros(len(idx), dtype=np.uint32) + rng.integers(0, 2, len(idx)).astype(np.uint32)
    else:
        idx = np.sort(np.argsort(price, kind="stable")[:400]).astype(np.uint32)
        new = np.full(len(idx), 0x7FFFFFF0, dtype=np.uint32) - rng.integers(0, 3, len(idx)).astype(np.uint32)
    a, b = t["wa"][idx].copy(), t["wb"][idx].copy()
    b["ext_ask_price"] = new
    t2 = dict(t, wb=t["wb"].copy())
    t2["wb"][idx] = b
    ev1, ev2 = oracle_eval(t), oracle_eval(t2)
    assert (ev1["row_best"] != ev2["row_best"]).any(), "the update must move some row minimum"
    check_update(t, t2, idx, a, b)


@pytest.mark.parametrize("W0,W1", [(3000, 4099), (4099, 2000)])
def test_resized_worker_table(W0, W1):
    """pm_resize_workers between the passes changes ld (3 -> 5 and 5 -> 2 stripes); the new rows are written by
    pm_update_workers, cheaper than every old row."""
    T = 500
    big = tables(T, max(W0, W1), seed_shift=W0 + W1)
    t = dict(big, wa=big["wa"][:W0].copy(), wb=big["wb"][:W0].copy())
    t2 = dict(big, wa=big["wa"][:W1].copy(), wb=big["wb"][:W1].copy())
    if W1 > W0:
        idx = np.arange(W0, W1, dtype=np.uint32)
        t2["wb"]["ext_ask_price"][W0:] = np.arange(W1 - W0, dtype=np.uint32) % 5
    else:
        idx = np.arange(0, W1, 7, dtype=np.uint32)
        t2["wb"]["ext_ask_price"][idx] = 1
    a, b = t2["wa"][idx].copy(), t2["wb"][idx].copy()
    check_update(t, t2, idx, a, b, resize=W1)


@pytest.mark.parametrize("where", ["last_lane", "last_warp"])
def test_equal_least_prices_at_the_end_of_a_stripe(where):
    """The least price only at columns 1021..1023 of each stripe (the last lane of warp 7), or at 900, 1000 and
    1023 (three lanes of warp 7): the least of the tied columns must win, and a later stripe's tie must lose."""
    W, T = 5000, 700
    t = tables(T, W, seed_shift=41)
    col = np.arange(W) % 1024
    low = col >= 1021 if where == "last_lane" else np.isin(col, [900, 1000, 1023])
    t["wb"] = t["wb"].copy()
    t["wb"]["ext_ask_price"] = np.where(low, 3, 777).astype(np.uint32)
    got = assert_same(t, tile_bytes(W, 256))
    ev = assert_oracle(t, got)
    hit = ev["row_count"] > 0
    assert low[ev["row_best"][hit] & 0xFFFFFFFF].any(), "no row reaches a tied least price"


@pytest.mark.parametrize("W", [1023, 1025, 2047, 2049])
@pytest.mark.parametrize("price", ["loguniform", "constant"])
def test_worker_counts_around_a_stripe(W, price):
    """Padding columns rank last in the last stripe and never count, with distinct prices and all prices equal."""
    t = tables(600, W, seed_shift=W)
    if price == "constant":
        t["wb"] = t["wb"].copy()
        t["wb"]["ext_ask_price"] = 5
    got = assert_same(t, tile_bytes(W, 256))
    assert_oracle(t, got)


@pytest.mark.parametrize("lo,n", [(3001, 4000), (5000, 5007), (1024, 1023)])
def test_shard_with_offset(lo, n):
    """pm_set_shard with w0 > 0: best_of_rank carries w0 + column, and the rank table covers the shard's own ld."""
    t = tables(700, 10007, seed_shift=lo + n)
    got = assert_same(t, tile_bytes(n, 256), shard=(lo, n))
    assert_oracle(t, got, lo, lo + n)
