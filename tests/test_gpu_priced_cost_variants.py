"""Every selectable cost-kernel variant of the first-fit pass, with priced workers, against the CPU oracle.

ask_best is each ask's signed int64 least (price << 32) | worker over the workers that meet it (PM_COST_INF when none
does) on every path: the 32-bit tile, the int64 tile on the FastRow path (PM_TUNE_BUILD=8), the generic predicate,
plain tile memory, and the fused pass.  Prices
are where a row minimum goes wrong quietly: ties must go to the lowest worker, and prices of 2^31 and above make the
packed cost negative.  Each case runs one engine and compares with the oracle (soa_eval_matrix, soa_form_groups):
  * the per-worker first feasible ask and the per-ask (best, count), read from the engine's device buffers;
  * the groups and the fetched ask_best / ask_count;
  * on the materialised path, the tile width that ran (4 or 8 B per evaluation, cost_bytes_written).
Further: the exported int64 cost rows (pm_build_cost_tile), sharded passes (w0 > 0) on one GPU, and pm_multi."""
import contextlib
import functools
import os

import numpy as np
import pytest

from helpers import groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200.engine import Engine, MultiEngine
from protocol_b200.sharded import wrap_device_buffers
from test_gpu_narrow_tile import tables as synth_tables
from test_gpu_sharded import sharded_pass_on_one_gpu
from test_gpu_variants import many_option_tables, wide_tables

pytestmark = pytest.mark.gpu

FF = abi.PM_MODE_FIRST_FIT
MAT, FUSED, LEAN = FF | abi.PM_PATH_MATERIALIZED, FF | abi.PM_PATH_FUSED, FF | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS
NONE = 0xFFFFFFFF
TILE = 1 << 20

# name -> (PM_TUNE_* environment read at pm_create, mode)
VARIANTS = {
    "default": ({}, MAT),                                             # FastRow build, 32-bit tile when prices allow
    "build8": ({"PM_TUNE_BUILD": "8"}, MAT),                          # the int64 tile on the FastRow path
    "generic": ({"PM_TUNE_GENERIC": "1"}, MAT),
    "plain_memory": ({"PM_TUNE_COMPRESS": "0"}, MAT),
    "fused": ({}, FUSED),
    "fused_generic": ({"PM_TUNE_GENERIC": "1"}, FUSED),
    "fused_lean": ({}, LEAN),                                         # first_ask and groups only
}
PRICES = ["none", "loguniform", "zipf", "constant", "top", "sign"]
EDGES = {"top": [0x7FFFFFFE] * 3,                                     # the 32-bit tile's largest price
         "sign": [0x7FFFFFFE, 0x7FFFFFFE, 0x80000000, 0x80000000, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF]}


@contextlib.contextmanager
def tuned(env):
    os.environ.update(env)
    try:
        yield
    finally:
        for k in env:
            os.environ.pop(k, None)


def with_prices(t, kind):
    """A copy of the tables with the price column set.  "top" and "sign" put edge prices on workers that meet some ask,
    spread over the table, on top of Zipf prices."""
    t = dict(t)
    n = len(t["wb"])
    wb = t["wb"].copy()
    if kind == "none":
        p = np.zeros(n, dtype=np.uint32)
    elif kind == "constant":
        p = np.full(n, 4242, dtype=np.uint32)              # every row minimum is a tie
    else:
        p = synth.make_workers(n, price="zipf" if kind in EDGES else kind).b["ext_ask_price"].copy()
    if kind in EDGES:
        first = np.asarray(oracle(t)["col_first"]).astype(np.uint32)
        feas = np.flatnonzero(first != NONE)
        pick = feas[np.linspace(0, len(feas) - 1, len(EDGES[kind]) + 2).astype(np.int64)[1:-1]]
        p[pick] = EDGES[kind]
    wb["ext_ask_price"] = p
    t["wb"] = wb
    return t


def oracle(t, t0=0, t1=None, w0=0, w1=None, want_cost=False):
    t1 = len(t["asks"]) if t1 is None else t1
    w1 = len(t["wa"]) if w1 is None else w1
    return orc.soa_eval_matrix(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"], t0, t1, w0, w1,
                               threads=8, want_cost=want_cost)


@functools.lru_cache(maxsize=None)
def base_tables(form):
    if form == "ragged":            # 613 x 6007: 29 tiles of 21 rows at 1 MB, "mixed" asks with several OR-options
        return synth_tables(613, 6007, seed_shift=5, price=None)
    if form.startswith("many_options"):
        w, a, obits, pbits, npat, nmod, words = many_option_tables(16 if form.endswith("16") else 200)
    else:
        n_models, n_patterns = {"bits2": (30, 900), "bits1": (200, 112), "bits0": (3000, 112),
                                "worker_major": (3000, 30)}[form]
        w, a, obits, pbits, npat, nmod, words = wide_tables(600, 6000, n_models=n_models, n_patterns=n_patterns,
                                                            seed_shift=50 + n_patterns, last_rows=True)
    assert (a.asks["n_opts"] > 1).any()
    return dict(asks=a.asks, opts=a.opts, wa=w.a, wb=w.b, bits=pbits, n_patterns=npat, n_models=nmod, words=words)


@functools.lru_cache(maxsize=None)
def case(form, price):
    """(tables, oracle evaluation, oracle groups) of one form with one price kind."""
    t = with_prices(base_tables(form), price)
    ev = oracle(t)
    og = orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"])
    hi = ev["row_best"][ev["row_count"] > 0] >> 32
    if price == "sign":             # the edge prices below zero are some asks' best
        assert (hi == np.int32(np.uint32(0x80000000))).any() and (hi == -1).any()
    elif price != "none":
        assert (hi != 0).all()
    return t, ev, og


def narrow_expected(env, t):
    """The engine's width selection: the FastRow build with every price below 0x7FFFFFFF takes the 32-bit tile."""
    return (env.get("PM_TUNE_GENERIC") != "1" and env.get("PM_TUNE_BUILD") != "8"
            and int(t["wb"]["ext_ask_price"].max()) < 0x7FFFFFFF)


def run_variant(t, ev, og, variant):
    env, mode = VARIANTS[variant]
    T, W = len(t["asks"]), len(t["wa"])
    with tuned(env):
        e = Engine(cost_tile_bytes=TILE)
    try:
        load_engine(e, t)
        e.match_local(mode)
        e.sync()
        fa, best, cnt = (x.cpu().numpy().copy() for x in wrap_device_buffers(e, W, T))
        st = e.stats()
        e.match_finish(mode)
        res = e.fetch()
    finally:
        e.close()
    assert np.array_equal(fa.view(np.uint32), np.asarray(ev["col_first"]).astype(np.uint32)), "first_ask differs"
    assert groups_equal(res, og), "groups differ"
    if mode != LEAN:
        assert np.array_equal(cnt.view(np.uint32), ev["row_count"]), "ask_count differs"
        assert np.array_equal(best, ev["row_best"]), "ask_best differs"
        assert np.array_equal(res.ask_best, ev["row_best"]) and np.array_equal(res.ask_count, ev["row_count"])
    if mode == MAT:
        width = 4 if narrow_expected(env, t) else 8
        assert st["cost_bytes_written"] == st["cost_bytes_read"] == width * T * W, "unexpected tile width"
        assert st["n_tiles"] > 1


@pytest.mark.parametrize("price", PRICES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_variant_ragged_multi_tile(variant, price):
    """613 asks x 6007 workers in 29 tiles, one-word acceptance rows (BITS 2)."""
    run_variant(*case("ragged", price), variant)


COMMON = ["default", "build8", "generic", "fused", "fused_generic", "fused_lean"]
FORM_VARIANTS = [(f, v) for f in ("bits2", "bits1", "bits0", "worker_major") for v in COMMON]


@pytest.mark.parametrize("price", ["zipf", "sign"])
@pytest.mark.parametrize("form,variant", FORM_VARIANTS)
def test_variant_acceptance_forms(form, variant, price):
    """Wide catalogues: acceptance rows of one word (BITS 2), per worker in shared memory (1), in global memory (0),
    and the worker-major table."""
    run_variant(*case(form, price), variant)


@pytest.mark.parametrize("price", ["zipf", "sign"])
@pytest.mark.parametrize("variant", ["default", "build8", "generic", "fused", "fused_generic"])
@pytest.mark.parametrize("n_models", [16, 200])
def test_variant_more_options_than_the_stage_holds(n_models, variant, price):
    """Asks with 384, 385, 400, 500 and 1200 OR-options: the staged kernels evaluate those beyond 384 with
    eval_row_global."""
    run_variant(*case(f"many_options_{n_models}", price), variant)


@pytest.mark.parametrize("price", ["zipf", "sign"])
@pytest.mark.parametrize("variant", ["default", "generic"])
@pytest.mark.parametrize("form", ["ragged", "worker_major"])
def test_exported_cost_rows(form, variant, price):
    """pm_build_cost_tile: the int64 rows, bit-equal to the oracle's packed costs, negative ones included."""
    t, ev, _ = case(form, price)
    T = len(t["asks"])
    env = VARIANTS[variant][0]
    with tuned(env):
        e = Engine(cost_tile_bytes=TILE)
    try:
        load_engine(e, t)
        got = e.cost_tile(0, T)
    finally:
        e.close()
    want = oracle(t, want_cost=True)["cost"]
    assert np.array_equal(got, want)
    assert (want < 0).any() == (price == "sign")


@functools.lru_cache(maxsize=None)
def sharded_case(price):
    t = with_prices(synth_tables(700, 10007, seed_shift=77, price=None), price)
    return t, oracle(t), orc.soa_form_groups(t["wa"], t["wb"], t["asks"], t["opts"], t["bits"], t["words"])


@pytest.mark.parametrize("price", ["loguniform", "sign"])
@pytest.mark.parametrize("mode", [MAT, FUSED], ids=["materialized", "fused"])
@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_priced(n_shards, mode, price):
    """Shards with w0 > 0, merged as the collective merges them: the per-shard minima carry the global worker index."""
    t, ev, og = sharded_case(price)
    for res in sharded_pass_on_one_gpu(t, n_shards, mode):
        assert np.array_equal(res.ask_best, ev["row_best"]) and np.array_equal(res.ask_count, ev["row_count"])
        assert groups_equal(res, og)


@pytest.mark.parametrize("price", ["loguniform", "sign"])
@pytest.mark.parametrize("mode", [MAT, FUSED], ids=["materialized", "fused"])
def test_multi_gpu_priced(mode, price):
    import torch

    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    t, ev, og = sharded_case(price)
    m = MultiEngine(list(range(n)), cost_tile_bytes=4 << 20)
    try:
        m.set_asks(t["asks"], t["opts"])
        m.set_model_table(t["bits"], t["n_patterns"], t["n_models"], t["words"])
        m.set_workers(t["wa"], t["wb"])
        m.match(mode)
        res = m.fetch()
    finally:
        m.close()
    assert groups_equal(res, og)
    assert np.array_equal(res.ask_best, ev["row_best"]) and np.array_equal(res.ask_count, ev["row_count"])
