"""The one-launch build + argmin of the 32-bit cost tile (pm_build_argmin, the default wherever that tile runs) on
hardware, against the int64 tile's separate build and argmin launches (PM_TUNE_BUILD=8) and the CPU oracle.

pm_build_argmin folds each row in registers as it writes it, two rows per loop iteration, 512 rows per CTA.  The cases
aim at the row edges (ask counts around the row pairs and the CTA's 512 rows), the padding columns past the last
worker, short last tiles that leave stale rows of the previous tile in the buffer, the shard offset, every
acceptance-table form, asks with more OR-options than the stage holds, row minima that tie across CTAs, the largest
price the tile holds, and two passes around a table update with no host synchronisation between them.  Every pm_result
array, the per-worker first feasible ask and the per-ask (best, count) must be equal (test_gpu_narrow_tile.assert_same)."""
import numpy as np
import pytest

from helpers import groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi
from protocol_b200.engine import _ptr
from protocol_b200.sharded import shard_range
from test_gpu_narrow_tile import MAT, RESULT_FIELDS, assert_same, make_engine, oracle_eval, tables
from test_gpu_tile_overlap import changed_rows, tile_bytes
from test_gpu_variants import many_option_tables, wide_tables

pytestmark = pytest.mark.gpu


def assert_oracle(t, got, w0=0, w1=None):
    ev = oracle_eval(t, w0, w1)
    w1 = len(t["wa"]) if w1 is None else w1
    assert np.array_equal(got[2], ev["row_count"])
    assert np.array_equal(got[1], ev["row_best"])
    assert np.array_equal(got[0][w0:w1], np.asarray(ev["col_first"]).astype(np.uint32))
    assert (got[0][:w0] == 0xFFFFFFFF).all() and (got[0][w1:] == 0xFFFFFFFF).all()
    return ev


def table_dict(w, a, pbits, npat, nmod, words):
    return dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=pbits, n_patterns=npat, n_models=nmod, words=words)


def test_ask_counts_around_the_band_and_the_cta():
    """T around 8, 16, 32 and 64 rows, and 511, 512, 513, 1025: odd and even row counts, and a short last CTA.  Tiles
    of 1024 rows or more are cut to whole 512-row bands, so 1025 asks take a second tile of one row."""
    W = 4099
    base = tables(1025, W, seed_shift=8)
    for T in sorted({1, 511, 512, 513, 1025} | {r + d for r in (8, 16, 32, 64) for d in (-1, 0, 1)}):
        t = dict(base, asks=base["asks"][:T])
        got = assert_same(t)
        assert got[3]["n_tiles"] == (2 if T == 1025 else 1)
        assert_oracle(t, got)
        assert groups_equal(got[4], orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"]))


@pytest.mark.parametrize("W", [1, 1023, 1024, 1025, 4099])
def test_worker_counts_around_the_cta_stripe(W):
    """Padding columns past the last worker hold the infeasible word and count nowhere."""
    t = tables(1025, W, seed_shift=7 + W)
    got = assert_same(t)
    assert_oracle(t, got)


@pytest.mark.parametrize("T,W,rows,n_tiles", [(1100, 4099, 256, 5), (2500, 2000, 1024, 3), (613, 6007, 21, 30)])
def test_short_last_tile_over_stale_rows(T, W, rows, n_tiles):
    """The last tile is short: the rows past it in the buffer still hold the previous tile's words."""
    t = tables(T, W, seed_shift=T + 3 * W)
    got = assert_same(t, tile_bytes(W, rows))
    assert got[3]["n_tiles"] == n_tiles
    assert_oracle(t, got)


@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_offsets(n_shards):
    """pm_set_shard with w0 > 0: the packed minimum and the first-ask column carry w0 + column."""
    t = tables(700, 10007, seed_shift=78)
    W = len(t["wa"])
    for r in range(1, n_shards):
        lo, hi = shard_range(W, n_shards, r)
        got = assert_same(t, tile_bytes(hi - lo, 256), shard=(lo, hi - lo))
        assert got[3]["n_tiles"] == 3
        assert_oracle(t, got, lo, hi)


@pytest.mark.parametrize("n_models,n_patterns", [(30, 900), (200, 112), (3000, 112), (3000, 30)],
                         ids=["bits2", "bits1", "bits0", "worker_major"])
def test_acceptance_forms(n_models, n_patterns):
    """BITS 2 / 1 / 0 and the worker-major table, with several OR-options per ask and random prices."""
    w, a, obits, pbits, npat, nmod, words = wide_tables(600, 6000, n_models=n_models, n_patterns=n_patterns,
                                                        seed_shift=60 + n_patterns, last_rows=True)
    rng = np.random.default_rng(n_patterns)
    w.b["ext_ask_price"] = rng.integers(0, 3000, len(w.b)).astype(np.uint32)
    got = assert_same(table_dict(w, a, pbits, npat, nmod, words), 1 << 20)
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, obits, words, 0, len(a.asks), 0, len(w.a), threads=8)
    assert np.array_equal(got[1], ev["row_best"]) and np.array_equal(got[2], ev["row_count"])
    assert np.array_equal(got[0], np.asarray(ev["col_first"]).astype(np.uint32))


@pytest.mark.parametrize("n_models", [16, 200])
def test_asks_with_hundreds_of_options(n_models):
    """Asks with 384 to 1200 OR-options: their further options are read from global memory in the build phase."""
    w, a, obits, pbits, npat, nmod, words = many_option_tables(n_models)
    got = assert_same(table_dict(w, a, pbits, npat, nmod, words), 1 << 20)
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, obits, words, 0, len(a.asks), 0, len(w.a), threads=8)
    assert np.array_equal(got[1], ev["row_best"]) and np.array_equal(got[2], ev["row_count"])
    assert np.array_equal(got[0], np.asarray(ev["col_first"]).astype(np.uint32))


def test_all_infeasible():
    t = tables(600, 5000, seed_shift=17)
    t["wa"] = t["wa"].copy()
    t["wa"]["flags"] &= ~np.uint32(abi.PM_W_HEALTHY)   # nobody is a candidate
    got = assert_same(t, 1 << 20)
    assert (got[2] == 0).all() and (got[0] == 0xFFFFFFFF).all()
    assert_oracle(t, got)


def test_all_feasible():
    """Asks without requirements over candidate workers: every evaluation is feasible."""
    t = tables(600, 5000, seed_shift=18)
    t["wa"] = t["wa"].copy()
    t["wa"]["flags"] = (t["wa"]["flags"] | np.uint32(abi.PM_W_HEALTHY | abi.PM_W_P2P)) & ~np.uint32(abi.PM_W_ASSIGNED)
    asks = t["asks"].copy()
    asks["flags"] = 0
    asks["n_opts"] = 0
    asks["opt_off"] = 0
    asks["min_group_size"] = asks["max_group_size"] = 1
    t["asks"] = asks
    got = assert_same(t, 1 << 20)
    assert (got[2] == 5000).all() and (got[0] == 0).all()
    assert_oracle(t, got)


@pytest.mark.parametrize("prices", ["constant", "mod3", "top"])
def test_price_ties_across_stripes(prices):
    """Every row minimum ties across lanes, warps and CTAs: the lowest worker must win.  "top" prices every worker at
    0x7FFFFFFE, the largest price the 32-bit tile holds, one below its infeasible word."""
    W = 9000
    t = tables(700, W, seed_shift=19)
    t["wb"] = t["wb"].copy()
    t["wb"]["ext_ask_price"] = {"constant": np.full(W, 4242), "mod3": np.arange(W) % 3 + 5,
                                "top": np.full(W, 0x7FFFFFFE)}[prices].astype(np.uint32)
    got = assert_same(t, tile_bytes(W, 256))
    ev = assert_oracle(t, got)
    assert (ev["row_count"] > 1).any()


def test_back_to_back_passes_across_a_table_update():
    """Pass 1, pm_update_workers and pass 2 are enqueued with no host synchronisation between them."""
    W, T = 4099, 700
    t = tables(T, W, seed_shift=5 + T)
    idx, a, b = changed_rows(t, T)
    t2 = dict(t, wa=t["wa"].copy(), wb=t["wb"].copy())
    t2["wa"][idx], t2["wb"][idx] = a, b
    out = []
    for wide in (True, False):   # the int64 tile, then the default 32-bit one
        e = make_engine(wide, cost_tile_bytes=tile_bytes(W, 256))
        try:
            load_engine(e, t)
            e.match_local(MAT)
            # the raw entry point: Engine.update_workers would synchronise the stream
            rc = e._lib.pm_update_workers(e._h, _ptr(idx), _ptr(a), _ptr(b), None, None, len(idx))
            assert rc == abi.PM_OK
            e.match(MAT)
            assert e.stats()["n_tiles"] == 3
            out.append(e.fetch())
        finally:
            e.close()
    for o in out[1:]:
        for f in RESULT_FIELDS:
            assert np.array_equal(getattr(o, f), getattr(out[0], f)), f"{f} differs"
    ev = oracle_eval(t2)
    assert np.array_equal(out[0].ask_best, ev["row_best"]) and np.array_equal(out[0].ask_count, ev["row_count"])
    assert groups_equal(out[0], orc.soa_form_groups(t2["wa"], t2["wb"], t2["asks"], t2["opts"], t2["bits"], t2["words"]))
