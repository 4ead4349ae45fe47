"""The materialised pass over several 32-bit cost tiles on hardware (pm_build_argmin, one launch per tile), against the
CPU oracle.

The per-worker first feasible ask, the per-ask (best, count) and the groups must equal the oracle's, the 32-bit tile
must have run, and the build and argmin timers must have recorded.  The cases aim at the ordering of the tiles: the
tile buffer reused by 1, 2, an odd number and five tiles, the shard offset, a second pass enqueued behind a table
update with no host synchronisation in between, the end-to-end pattern on a caller's stream, and the tile in plain
rather than compressible memory."""
import os

import numpy as np
import pytest
import torch

from helpers import groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi
from protocol_b200.engine import Engine, _ptr
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_gpu_narrow_tile import MAT, RESULT_FIELDS, oracle_eval, tables

pytestmark = pytest.mark.gpu


def one_pass(t, cost_tile_bytes=0, shard=None):
    """(first_ask, ask_best, ask_count, stats, result or None) of one materialised pass."""
    W, T = len(t["wa"]), len(t["asks"])
    e = Engine(cost_tile_bytes=cost_tile_bytes, timing=True)
    load_engine(e, t)
    if shard is not None:
        e.set_shard(*shard)
    e.match_local(MAT)
    e.sync()
    fa, best, cnt = (x.cpu().numpy().copy() for x in wrap_device_buffers(e, W, T))
    res = None
    if shard is None:
        e.match_finish(MAT)   # also resolves the kernel timers
        res = e.fetch()
    st = e.stats()
    e.close()
    return fa.view(np.uint32), best, cnt.view(np.uint32), st, res


def assert_results_equal(a, b):
    for f in RESULT_FIELDS:
        assert np.array_equal(getattr(a, f), getattr(b, f)), f"{f} differs"


def narrow_pass(t, cost_tile_bytes, shard=None):
    """one_pass, checked to have run the 32-bit tile (and, unsharded, to have timed its launches)"""
    T = len(t["asks"])
    nw = shard[1] if shard is not None else len(t["wa"])
    o = one_pass(t, cost_tile_bytes, shard)
    st = o[3]
    assert st["cost_bytes_written"] == st["cost_bytes_read"] == 4 * T * nw, "the 32-bit tile did not run"
    assert shard is not None or (st["ms_build"] > 0 and st["ms_argmin"] > 0)
    return o


def tile_bytes(W, rows):
    """pm_cfg.cost_tile_bytes that gives `rows` rows per tile (rows are sized at 8 B per element of the padded row)."""
    ld = -(-W // 1024) * 1024
    return rows * ld * 8


@pytest.mark.parametrize("T,W,rows,n_tiles", [(200, 4099, 256, 1), (500, 4099, 256, 2), (700, 4099, 256, 3),
                                              (1100, 1025, 256, 5), (5000, 20000, 1024, 5)])
def test_overlap_equals_sequential(T, W, rows, n_tiles):
    t = tables(T, W, seed_shift=3 * T + W)
    got = narrow_pass(t, tile_bytes(W, rows))
    assert got[3]["n_tiles"] == n_tiles
    ev = oracle_eval(t)
    assert np.array_equal(got[1], ev["row_best"]) and np.array_equal(got[2], ev["row_count"])
    assert np.array_equal(got[0], np.asarray(ev["col_first"]).astype(np.uint32))
    assert groups_equal(got[4], orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"]))


@pytest.mark.parametrize("n_shards", [2, 3])
def test_overlap_equals_sequential_sharded(n_shards):
    """pm_set_shard with w0 > 0 and three tiles per pass."""
    t = tables(700, 10007, seed_shift=78)
    W = len(t["wa"])
    for r in range(1, n_shards):
        lo, hi = shard_range(W, n_shards, r)
        got = narrow_pass(t, tile_bytes(hi - lo, 256), shard=(lo, hi - lo))
        assert got[3]["n_tiles"] == 3
        ev = oracle_eval(t, lo, hi)
        assert np.array_equal(got[2], ev["row_count"])
        feas = got[2] > 0
        assert np.array_equal(got[1][feas], ev["row_best"][feas])
        assert np.array_equal(got[0][lo:hi], np.asarray(ev["col_first"]).astype(np.uint32))
        assert (got[0][:lo] == 0xFFFFFFFF).all() and (got[0][hi:] == 0xFFFFFFFF).all()


def changed_rows(t, seed):
    """A few hundred workers get new prices and half of them lose their candidate flags."""
    rng = np.random.default_rng(seed)
    idx = np.sort(rng.choice(len(t["wa"]), 300, replace=False)).astype(np.uint32)
    a, b = t["wa"][idx].copy(), t["wb"][idx].copy()
    b["ext_ask_price"] = rng.integers(0, 1000, len(idx)).astype(np.uint32)
    a["flags"][::2] &= ~np.uint32(abi.PM_W_HEALTHY)
    return idx, a, b


@pytest.mark.parametrize("n_tiles,T", [(2, 500), (3, 700)])
def test_back_to_back_passes_across_a_table_update(n_tiles, T):
    """Pass 1, pm_update_workers and pass 2 are enqueued with no host synchronisation between them: pass 2's first
    build reuses the tile pass 1's last launch wrote, and its table update lands behind pass 1."""
    W = 4099
    t = tables(T, W, seed_shift=5 + T)
    idx, a, b = changed_rows(t, T)
    t2 = dict(t, wa=t["wa"].copy(), wb=t["wb"].copy())
    t2["wa"][idx], t2["wb"][idx] = a, b
    e = Engine(cost_tile_bytes=tile_bytes(W, 256))
    load_engine(e, t)
    e.match_local(MAT)
    # the raw entry point: Engine.update_workers would synchronise the stream
    rc = e._lib.pm_update_workers(e._h, _ptr(idx), _ptr(a), _ptr(b), None, None, len(idx))
    assert rc == abi.PM_OK
    e.match(MAT)
    assert e.stats()["n_tiles"] == n_tiles
    res = e.fetch()
    e.close()
    ev = oracle_eval(t2)
    assert np.array_equal(res.ask_best, ev["row_best"]) and np.array_equal(res.ask_count, ev["row_count"])
    assert groups_equal(res, orc.soa_form_groups(t2["wa"], t2["wb"], t2["asks"], t2["opts"], t2["bits"], t2["words"]))


def test_e2e_pattern_on_a_caller_stream():
    """set_asks + upsert_workers(sync=False) + match + fetch on a caller-provided stream, twice with different tables
    on one engine: every upload, launch and read-back is ordered on the caller's stream."""
    W = 4099
    t = tables(700, W, seed_shift=201)
    idx, a, b = changed_rows(t, 201)
    t2 = dict(t, asks=t["asks"][:500], wa=t["wa"].copy(), wb=t["wb"].copy())   # same model table, fewer asks
    t2["wa"][idx], t2["wb"][idx] = a, b
    passes = [t, t2]
    got = []
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        e = Engine(cost_tile_bytes=tile_bytes(W, 256), stream=stream.cuda_stream)
        load_engine(e, passes[0])
        for t in passes:
            e.set_asks(t["asks"], t["opts"])
            e.upsert_workers(t["wa"], t["wb"], sync=False)
            e.match(MAT)
            r = e.fetch(copy=False)
            got.append({f: np.array(getattr(r, f), copy=True) for f in RESULT_FIELDS})
        e.close()
    stream.synchronize()
    for t, o in zip(passes, got):
        ev = oracle_eval(t)
        assert np.array_equal(o["ask_best"], ev["row_best"]) and np.array_equal(o["ask_count"], ev["row_count"])
        og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"])
        assert np.array_equal(o["group_ask"], og.cfg) and np.array_equal(o["group_members"], og.members)


def test_plain_tile_memory_equals_compressible():
    """The cost tile in compressible memory (the default where the device offers it) and in plain cudaMalloc memory
    (PM_TUNE_COMPRESS=0) give the same outputs."""
    t = tables(700, 4099, seed_shift=303)
    os.environ["PM_TUNE_COMPRESS"] = "0"
    try:
        plain = one_pass(t, tile_bytes(4099, 256))
    finally:
        os.environ.pop("PM_TUNE_COMPRESS", None)
    got = one_pass(t, tile_bytes(4099, 256))
    for a, b in zip(got[:3], plain[:3]):
        assert np.array_equal(a, b)
    assert_results_equal(got[4], plain[4])
