"""The 32-bit cost tile on hardware: the materialised first-fit pass with the narrow tile (the default on the FastRow
path when every price is below 0x7FFFFFFF) against the int64 tile (PM_TUNE_BUILD=8) and the CPU oracle.

Every pm_result array, the per-worker first feasible ask and the per-ask (best, count) must be equal between the two
widths.  The byte counters show which tile ran: 4 B per evaluation for the narrow tile, 8 B for the int64 one."""
import os

import numpy as np
import pytest

from helpers import groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200.engine import Engine
from protocol_b200.sharded import shard_range, wrap_device_buffers
from test_gpu_variants import wide_tables

pytestmark = pytest.mark.gpu

MAT = abi.PM_MODE_FIRST_FIT | abi.PM_PATH_MATERIALIZED
RESULT_FIELDS = ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count")


def make_engine(wide, **kw):
    """wide: the int64 tile on the FastRow path (PM_TUNE_BUILD=8), the 32-bit tile's reference"""
    if wide:
        os.environ["PM_TUNE_BUILD"] = "8"   # read at pm_create
    try:
        return Engine(**kw)
    finally:
        os.environ.pop("PM_TUNE_BUILD", None)


def tables(n_asks, n_workers, seed_shift, price="loguniform"):
    w = synth.make_workers(n_workers, seed=synth.SEED_WORKERS + seed_shift, price=price)
    a = synth.make_asks(n_asks, "mixed", seed=synth.SEED_ASKS + seed_shift)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    return dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=bits, n_patterns=npat, n_models=nmod, words=words)


def one_pass(t, wide, cost_tile_bytes=0, shard=None):
    """(first_ask, ask_best, ask_count, stats, result or None) of one materialised pass."""
    W, T = len(t["wa"]), len(t["asks"])
    e = make_engine(wide, cost_tile_bytes=cost_tile_bytes, timing=True)
    try:
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
    finally:
        e.close()
    return fa.view(np.uint32), best, cnt.view(np.uint32), st, res


def assert_same(t, cost_tile_bytes=0, shard=None):
    """The 32-bit tile's pass against the int64 tile's; returns the 32-bit tile's."""
    T = len(t["asks"])
    nw = shard[1] if shard is not None else len(t["wa"])
    n = one_pass(t, False, cost_tile_bytes, shard)
    w = one_pass(t, True, cost_tile_bytes, shard)
    assert n[3]["cost_bytes_written"] == n[3]["cost_bytes_read"] == 4 * T * nw, "the narrow tile did not run"
    assert w[3]["cost_bytes_written"] == w[3]["cost_bytes_read"] == 8 * T * nw, "the int64 tile did not run"
    for st in (n[3], w[3]):
        assert shard is not None or (st["ms_build"] > 0 and st["ms_argmin"] > 0)
    for k in ("n_tiles", "n_build_launches", "n_argmin_launches"):
        assert n[3][k] == w[3][k], k
    assert n[3]["n_argmin_launches"] == n[3]["n_build_launches"] == n[3]["n_tiles"]
    assert np.array_equal(n[0], w[0]), "first_ask differs"
    assert np.array_equal(n[1], w[1]), "ask_best differs"
    assert np.array_equal(n[2], w[2]), "ask_count differs"
    if shard is None:
        for f in RESULT_FIELDS:
            assert np.array_equal(getattr(n[4], f), getattr(w[4], f)), f"{f} differs"
    return n


def oracle_eval(t, w0=0, w1=None):
    w1 = len(t["wa"]) if w1 is None else w1
    return orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], 0, len(t["asks"]),
                               w0, w1, threads=8)


def assert_oracle(t, got, w0=0, w1=None):
    ev = oracle_eval(t, w0, w1)
    w1 = len(t["wa"]) if w1 is None else w1
    assert np.array_equal(got[1], ev["row_best"]) and np.array_equal(got[2], ev["row_count"])
    assert np.array_equal(got[0][w0:w1], np.asarray(ev["col_first"]).astype(np.uint32))


@pytest.mark.parametrize("T,W,tile", [(700, 1, 0), (700, 1023, 0), (700, 1025, 1 << 20), (1300, 4099, 1 << 20),
                                      (2500, 4099, 0), (1031, 20000, 4 << 20)])
@pytest.mark.parametrize("price", ["loguniform", None], ids=["cfg3_prices", "no_prices"])
def test_narrow_equals_wide_ragged(T, W, tile, price):
    t = tables(T, W, seed_shift=T + W, price=price)
    got = assert_same(t, cost_tile_bytes=tile)
    assert_oracle(t, got)
    assert got[3]["n_tiles"] > 1 or tile == 0


@pytest.mark.parametrize("n_models,n_patterns,bits", [(30, 900, 2), (200, 112, 1), (3000, 112, 0), (3000, 30, 0)],
                         ids=["bits2", "bits1", "bits0", "worker_major"])
def test_narrow_equals_wide_acceptance_forms(n_models, n_patterns, bits):
    """BITS 2 / 1 / 0 and the worker-major table, with several OR-options per ask ("mixed" asks) and random prices."""
    w, a, obits, pbits, npat, nmod, words = wide_tables(600, 6000, n_models=n_models, n_patterns=n_patterns,
                                                        seed_shift=40 + n_patterns, last_rows=True)
    assert (a.asks["n_opts"] > 1).any()
    rng = np.random.default_rng(n_models)
    w.b["ext_ask_price"] = rng.integers(0, 3000, len(w.b)).astype(np.uint32)
    t = dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=pbits, n_patterns=npat, n_models=nmod, words=words)
    got = assert_same(t, cost_tile_bytes=1 << 20)
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, obits, words, 0, len(a.asks), 0, len(w.a), threads=8)
    assert np.array_equal(got[1], ev["row_best"]) and np.array_equal(got[2], ev["row_count"])


@pytest.mark.parametrize("n_shards", [2, 3])
def test_narrow_equals_wide_sharded(n_shards):
    """pm_set_shard with w0 > 0: the argmin adds the shard offset back to the column."""
    t = tables(900, 10007, seed_shift=77)
    W = len(t["wa"])
    for r in range(1, n_shards):
        lo, hi = shard_range(W, n_shards, r)
        got = assert_same(t, cost_tile_bytes=1 << 20, shard=(lo, hi - lo))
        ev = oracle_eval(t, lo, hi)
        assert np.array_equal(got[2], ev["row_count"])
        feas = got[2] > 0
        assert np.array_equal(got[1][feas], ev["row_best"][feas])
        assert np.array_equal(got[0][lo:hi], np.asarray(ev["col_first"]).astype(np.uint32))
        assert (got[0][:lo] == 0xFFFFFFFF).all() and (got[0][hi:] == 0xFFFFFFFF).all()


@pytest.mark.parametrize("edge", [0x7FFFFFFE, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF])
def test_price_edges_select_the_width_and_match_the_oracle(edge):
    """One feasible worker priced at the edge: 0x7FFFFFFE still runs narrow, the others keep the int64 tile; after
    pm_update_workers replaces the price the next pass runs narrow again."""
    t = tables(600, 5000, seed_shift=91)
    T, W = len(t["asks"]), len(t["wa"])
    ev = oracle_eval(t)
    first = np.asarray(ev["col_first"]).astype(np.uint32)
    i = int(np.nonzero(first != 0xFFFFFFFF)[0][len(np.nonzero(first != 0xFFFFFFFF)[0]) // 2])   # feasible for some asks
    t["wb"] = t["wb"].copy()
    t["wb"]["ext_ask_price"][i] = edge
    e = Engine()
    load_engine(e, t)
    e.match(MAT)
    res = e.fetch()
    want = 4 if edge < 0x7FFFFFFF else 8
    assert e.stats()["cost_bytes_written"] == want * T * W
    ev = oracle_eval(t)
    assert np.array_equal(res.ask_best, ev["row_best"]) and np.array_equal(res.ask_count, ev["row_count"])
    assert groups_equal(res, orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"]))
    if edge >= 0x80000000:
        assert (res.ask_best >> 32 == np.int64(np.int32(np.uint32(edge)))).any(), "the edge worker is nobody's best"
    b = t["wb"][i:i + 1].copy()
    b["ext_ask_price"] = 17
    e.update_workers(np.array([i], dtype=np.uint32), t["wa"][i:i + 1], b)
    t["wb"]["ext_ask_price"][i] = 17
    e.match(MAT)
    res = e.fetch()
    assert e.stats()["cost_bytes_written"] == 4 * T * W
    ev = oracle_eval(t)
    assert np.array_equal(res.ask_best, ev["row_best"]) and np.array_equal(res.ask_count, ev["row_count"])
    e.close()
