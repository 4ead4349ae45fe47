"""The benchmark's own workloads on the GPU, every array compared in full against the collapsed reference.

The tables come from bench.make_tables, so what is checked is what bench.py measures.  The reference
(tests/collapsed_oracle.py) evaluates the oracle's predicate once per (distinct ask row, worker profile) and expands the
result exactly; tests/test_collapsed_oracle.py pins it to the dense oracle.  Nothing here is sampled: every array of
every result taken is compared whole.

PM_TEST_BIG=1 adds the 1M asks x 1M workers per-GPU shape of cfg5 on every path and a rank's share of cfg5's 8M-worker
table; without it the file runs in a few minutes.
"""
import functools
import os

import numpy as np
import pytest

import collapsed_oracle as co
from oracle import pm_oracle as orc
from protocol_b200 import abi, synth
from protocol_b200.engine import Engine, pinned_empty
from protocol_b200.sharded import wrap_device_buffers
from test_collapsed_oracle import bench_module, tile_rows

pytestmark = pytest.mark.gpu

BIG = os.environ.get("PM_TEST_BIG") == "1"
big = pytest.mark.skipif(not BIG, reason="cfg5's per-GPU shape and 8M-worker table: run with PM_TEST_BIG=1")
BENCH = bench_module()
FF = abi.PM_MODE_FIRST_FIT
LEAN = abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS
PATHS = {"materialized": abi.PM_PATH_MATERIALIZED, "fused": abi.PM_PATH_FUSED, "fused-lean": LEAN}
TILE = 8 << 30   # bench.py's default --tile-gib


@functools.lru_cache(maxsize=2)
def workload(name, n_gpus=1, models=0):
    """(workers, asks, model table, reference) of bench.make_tables(name, n_gpus, models)."""
    w, a, tbl, _ = BENCH.make_tables(name, n_gpus, models)
    return w, a, tbl, co.Reference(w.a, w.b, a.asks, a.opts, *tbl)


@functools.lru_cache(maxsize=4)
def expected(name, n_gpus=1, models=0, ask_stats=True):
    return workload(name, n_gpus, models)[3].result(ask_stats)


def load(eng, w, a, tbl):
    eng.set_asks(a.asks, a.opts)
    eng.set_model_table(*tbl)
    eng.set_workers(w.a, w.b)


def assert_result(res, want, what=""):
    for f in co.FIELDS:
        assert np.array_equal(getattr(res, f), want[f]), f"{what}: {f} differs from the reference"


# ------------------------------------------------------------------ every workload on one GPU, every path
ONE_GPU = [(wl, p) for wl in ("cfg1", "cfg2", "cfg3", "cfg4") for p in PATHS] + \
          [pytest.param("cfg5", p, marks=big) for p in PATHS]


@pytest.mark.parametrize("wl,path", ONE_GPU)
def test_workload_on_one_gpu(wl, path):
    """cfg1-3 at their one-GPU shape, cfg4 and cfg5 at their per-GPU shape, as bench.py runs them."""
    w, a, tbl, ref = workload(wl)
    eng = Engine(timing=True, cost_tile_bytes=TILE)
    load(eng, w, a, tbl)
    eng.match(FF | PATHS[path])
    res = eng.fetch()
    assert res.stats["evals"] == len(a.asks) * len(w.a)
    assert_result(res, expected(wl, ask_stats=path != "fused-lean"), f"{wl} {path}")
    if path == "materialized" and len(a.asks) * len(w.a) >= 10 ** 11:
        assert res.stats["n_tiles"] == -(-len(a.asks) // tile_rows(len(a.asks), len(w.a)))
    eng.close()


@pytest.mark.parametrize("env", [{"PM_TUNE_BUILD": "8"}, {"PM_TUNE_GENERIC": "1"}, {"PM_TUNE_COMPRESS": "0"}],
                         ids=["build8_int64_tile", "generic", "compress0"])
def test_cfg3_kernel_settings(env, monkeypatch):
    """The other build / argmin forms at the headline shape: the int64 tile (separate build and argmin), the generic
    predicate, the uncompressed tile (the knobs are read when the engine is created)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w, a, tbl, ref = workload("cfg3")
    eng = Engine(timing=True, cost_tile_bytes=TILE)
    load(eng, w, a, tbl)
    eng.match(FF | abi.PM_PATH_MATERIALIZED)
    assert_result(eng.fetch(), expected("cfg3"), str(env))
    eng.close()


def test_cfg3_as_the_benchmark_drives_it():
    """bench.run_ours: a caller stream, timing on, 8 GiB tiles, warm-up and timed steps back to back, then end-to-end
    steps that re-upload the asks and workers from pinned memory without a synchronise.  Every result taken is whole."""
    import torch

    w, a, tbl, ref = workload("cfg3")
    want = expected("cfg3")
    mode = FF | abi.PM_PATH_MATERIALIZED
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng = Engine(timing=True, cost_tile_bytes=TILE, stream=stream.cuda_stream)
        load(eng, w, a, tbl)
        for _ in range(6):
            eng.match(mode)
            eng.stats()
        assert_result(eng.fetch(), want, "timed steps")
        pa, pb = pinned_empty(len(w.a), abi.WORKER_A), pinned_empty(len(w.b), abi.WORKER_B)
        p_asks, p_opts = pinned_empty(len(a.asks), abi.ASK), pinned_empty(len(a.opts), abi.GPU_OPT)
        pa[:], pb[:], p_asks[:], p_opts[:] = w.a, w.b, a.asks, a.opts
        for step in range(2):
            eng.set_asks(p_asks, p_opts)
            eng.upsert_workers(pa, pb, first=0, sync=False)
            eng.match(mode)
            assert_result(eng.fetch(copy=False), want, f"e2e step {step}")
        eng.close()
    torch.cuda.synchronize()


@pytest.mark.parametrize("models", [200, 3000, 100_000])
def test_cfg3_wide_catalogues(models):
    """bench.py --models N: the per-worker acceptance word in shared memory, the table in global memory, the
    worker-major word.  The interned table is the oracle's own model clause, and every path gives the reference."""
    w, a, tbl, ref = workload("cfg3", 1, models)
    bits, npat, nmod, words = tbl
    assert nmod == models
    assert np.array_equal(bits, orc.model_table(w.model_strings, a.pattern_strings, threads=co.threads())[0])
    eng = Engine(timing=True, cost_tile_bytes=TILE)
    load(eng, w, a, tbl)
    for path, bit in PATHS.items():
        eng.match(FF | bit)
        assert_result(eng.fetch(), expected("cfg3", 1, models, path != "fused-lean"), f"{models} models, {path}")
    eng.close()


def test_cfg3_first_asks_past_the_first_tile():
    """With the first tile's asks disabled, every worker's first ask lies in a later tile, and the per-ask statistics
    of the disabled rows are empty."""
    w, a, tbl, _ = workload("cfg3")
    T, W = len(a.asks), len(w.a)
    rows = tile_rows(T, W)
    enabled = np.ones(T, dtype=bool)
    enabled[:rows + 7] = False
    want = co.Reference(w.a, w.b, a.asks, a.opts, *tbl, enabled=enabled).result()
    assert want["worker_ask"][want["worker_ask"] != co.NONE].min() >= rows
    eng = Engine(timing=True, cost_tile_bytes=TILE)
    load(eng, w, a, tbl)
    eng.set_ask_enabled(np.flatnonzero(~enabled), False)
    for path, bit in PATHS.items():
        eng.match(FF | bit)
        ref = want if path != "fused-lean" else dict(want, ask_best=np.full(T, co.INF, np.int64), ask_count=np.zeros(T, np.uint32))
        assert_result(eng.fetch(), ref, path)
    eng.close()


# ------------------------------------------------------------------ a rank's share
def local_arrays(eng, W, T):
    fa, best, cnt = wrap_device_buffers(eng, W, T)
    return fa.cpu().numpy().view(np.uint32).copy(), best.cpu().numpy().copy(), cnt.cpu().numpy().view(np.uint32).copy()


def assert_local(got, want, what):
    for name, g in zip(("first_ask", "ask_best", "ask_count"), got):
        assert np.array_equal(g, want[name]), f"{what}: {name} differs from the range reference"


def test_cfg4_four_ranks_on_one_gpu():
    """bench.py --gpus 4 --workload cfg4: 1M asks x 1M workers, each rank evaluating its 250k workers.  Every rank's
    local arrays equal the range reference; merged as the exchange merges them, pm_match_finish gives the full one."""
    import torch

    n = 4
    w, a, tbl, ref = workload("cfg4", n)
    T, W = len(a.asks), len(w.a)
    Wg = W // n
    first = np.full(W, co.NONE, dtype=np.uint32)
    bests, cnts = [], []
    for r in range(n):
        eng = Engine(timing=True, cost_tile_bytes=TILE)
        load(eng, w, a, tbl)
        eng.set_shard(r * Wg, Wg)
        eng.match_local(FF | abi.PM_PATH_MATERIALIZED)
        eng.sync()
        got = local_arrays(eng, W, T)
        assert_local(got, ref.local(r * Wg, Wg), f"rank {r}")
        first[r * Wg:(r + 1) * Wg] = got[0][r * Wg:(r + 1) * Wg]
        bests.append(got[1])
        cnts.append(got[2])
        if r < n - 1:
            eng.close()
    fa, best, cnt = wrap_device_buffers(eng, W, T)
    fa.copy_(torch.from_numpy(first.view(np.int32)))
    best.copy_(torch.from_numpy(np.min(bests, axis=0)))
    cnt.copy_(torch.from_numpy(np.sum(cnts, axis=0, dtype=np.uint32).view(np.int32)))
    torch.cuda.synchronize()
    eng.match_finish(FF | abi.PM_PATH_MATERIALIZED)
    assert_result(eng.fetch(), expected("cfg4", n), "merged")
    eng.close()


@big
def test_cfg5_last_of_eight_ranks():
    """bench.py --gpus 8: the last rank of cfg5's 1M asks x 8M workers evaluates workers [7M, 8M)."""
    n = 8
    w, a, tbl, ref = workload("cfg5", n)
    T, W = len(a.asks), len(w.a)
    Wg = W // n
    for path in ("materialized", "fused"):
        eng = Engine(timing=True, cost_tile_bytes=TILE)
        load(eng, w, a, tbl)
        eng.set_shard((n - 1) * Wg, Wg)
        eng.match_local(FF | PATHS[path])
        eng.sync()
        assert_local(local_arrays(eng, W, T), ref.local((n - 1) * Wg, Wg), path)
        eng.close()


# ------------------------------------------------------------------ incremental passes at cfg3
def test_cfg3_incremental_passes():
    """PM_INCREMENTAL lean passes after 1 000 and 100 000 rewritten worker rows (other specs, health and prices), then
    after 100 disabled asks, each against the reference rebuilt from the new tables."""
    w, a, tbl, _ = workload("cfg3")
    T, W = len(a.asks), len(w.a)
    wa, wb = w.a.copy(), w.b.copy()
    pool = synth.make_workers(100_000, seed=synth.SEED_WORKERS + 77, price="zipf")
    rng = np.random.default_rng(77)
    mode = FF | LEAN | abi.PM_INCREMENTAL
    eng = Engine(timing=True, cost_tile_bytes=TILE)
    load(eng, w, a, tbl)
    eng.match(mode)
    for n in (1000, 100_000):
        idx = np.sort(rng.choice(W, n, replace=False)).astype(np.uint32)
        sel = rng.integers(0, len(pool), n)
        ra, rb = pool.a[sel].copy(), pool.b[sel].copy()
        ra["flags"][rng.random(n) < 0.2] ^= abi.PM_W_HEALTHY
        eng.update_workers(idx, ra, rb)
        wa[idx], wb[idx] = ra, rb
        eng.match(mode)
        res = eng.fetch()
        if n == 1000:                                  # only the written rows were evaluated again
            assert res.stats["n_tiles"] == n and 0 < res.stats["evals"] <= T * n, res.stats
        assert_result(res, co.Reference(wa, wb, a.asks, a.opts, *tbl).result(ask_stats=False), f"{n} rows")
    enabled = np.ones(T, dtype=bool)
    off = np.concatenate([np.arange(5), rng.choice(np.arange(5, T), 95, replace=False)])   # the first asks own most workers
    enabled[off] = False
    eng.set_ask_enabled(off, False)
    eng.match(mode)
    assert_result(eng.fetch(), co.Reference(wa, wb, a.asks, a.opts, *tbl, enabled=enabled).result(ask_stats=False),
                  "100 asks disabled")
    eng.close()


# ------------------------------------------------------------------ the auction at cfg3
def assert_certificate(eng, wa, wb, a, tbl, caps, what):
    cert = eng.auction_certificate(ask_bound=True)
    price, _, _ = eng.auction_state()
    want = co.certificate(wa, wb, a.asks, a.opts, *tbl, caps, 1, price, eng.auction_assignment())
    for f in co.CERT_FIELDS:
        assert cert[f] == want[f], f"{what}: {f} {cert[f]} != {want[f]}"
    assert np.array_equal(cert["ask_bound"], want["ask_bound"]), what
    assert 0 <= cert["gap"] <= len(a.asks) and cert["n_bad_holds"] == cert["n_shared"] == 0, what


def test_cfg3_auction_certificate():
    """bench.auction_record's market: the device's certificate equals the collapsed restatement field by field and row
    by row, and the gap is at most T; again after a warm pass that follows 1 000 rewritten worker rows."""
    w, a, tbl, _ = workload("cfg3")
    T, W = len(a.asks), len(w.a)
    caps = np.exp(np.log(20) + synth._unit(synth.SEED_EXT, T, 3) * np.log(100)).astype(np.uint32)
    wa, wb = w.a.copy(), w.b.copy()
    eng = Engine(timing=True, cost_tile_bytes=TILE)
    load(eng, w, a, tbl)
    eng.set_price_caps(caps)
    eng.match(abi.PM_MODE_AUCTION)
    assert eng.fetch().n_groups > T // 2
    assert_certificate(eng, wa, wb, a, tbl, caps, "cold")
    rng = np.random.default_rng(78)
    pool = synth.make_workers(1000, seed=synth.SEED_WORKERS + 78, price="loguniform")
    idx = np.sort(rng.choice(W, 1000, replace=False)).astype(np.uint32)
    eng.update_workers(idx, pool.a, pool.b)
    wa[idx], wb[idx] = pool.a, pool.b
    eng.match(abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM)
    assert eng.auction_state(prices=False)[1]          # the pass started warm
    assert_certificate(eng, wa, wb, a, tbl, caps, "warm")
    eng.close()
