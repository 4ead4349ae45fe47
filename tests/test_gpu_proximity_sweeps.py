"""Proximity group formation past one CTA: pm_proximity_grid (the cooperative all-SM sweep) and pm_proximity_sweep (the
single-CTA fallback, PM_TUNE_PROX=2) on thousands of configurations, runs of configurations nobody reaches, hand-downs
of 127 / 128 / 129 / 2000, a 2200-link cascade, seed-parallel batches on 1, 2 and 118 CTAs, and groups selected in
several chunks of 16 across CTA chunks.

Inputs and the guards proving that each reaches its path live in tests/test_proximity_sweep_inputs.py, which runs
them on the CPU.  Here the engine's groups, worker_group and worker_ask are compared with the checker's
(orc.soa_form_groups under proximity); the engine's count of hand-downs (stats["n_bumped"]) must equal the number the
checker's groups imply, and a second pass on the same engine must give the same result.  On the grid kernel the
diagnostics must agree with the groups: n_rounds (groups formed in seed-parallel batches) + n_build_launches (groups
formed one at a time) = the non-empty groups of configurations with max >= 2, no batch on one CTA, and a batch
wherever the guard says one must open.
"""
import os

import numpy as np
import pytest

from helpers import load_engine
from protocol_b200 import abi
from protocol_b200.engine import Engine
from test_gpu_sharded import sharded_pass_on_one_gpu
from test_proximity_sweep_inputs import CASES, NONE, Case, Evidence, enabled_tables, guard, n_ctas

pytestmark = pytest.mark.gpu

KERNELS = {"grid": "0", "single_cta": "2"}
INCR = abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS | abi.PM_INCREMENTAL


def new_engine(kernel):
    os.environ["PM_TUNE_PROX"] = KERNELS[kernel]   # read at pm_create
    try:
        return Engine()
    finally:
        os.environ.pop("PM_TUNE_PROX", None)


def load(eng, case):
    load_engine(eng, case.t, addr_rank=case.rank, locations=True)
    off = np.flatnonzero(~case.on)
    if len(off):
        eng.set_ask_enabled(off, False)


def per_worker(ev):
    wg = np.full(ev.W, NONE, dtype=np.uint32)
    wk = np.full(ev.W, NONE, dtype=np.uint32)
    for g in range(len(ev.cfg)):
        m = ev.members(g)
        wg[m], wk[m] = g, ev.cfg[g]
    return wg, wk


def check(res, ev, cfg=None):
    """Engine result == the checker's groups (full-table ask indices unless `cfg` gives others)."""
    cfg = ev.cfg if cfg is None else cfg
    assert len(res.group_ask) == len(cfg), f"engine {len(res.group_ask)} groups vs checker {len(cfg)}"
    assert np.array_equal(res.group_ask, cfg), f"first differing group {np.flatnonzero(res.group_ask != cfg)[:1]}"
    assert np.array_equal(res.group_off, ev.og.off) and np.array_equal(res.group_members, ev.og.members)
    wg, wk = per_worker(ev)
    if cfg is not ev.cfg:
        wk = np.where(wg == NONE, NONE, cfg[np.where(wg == NONE, 0, wg)]).astype(np.uint32)
    assert np.array_equal(res.worker_group, wg) and np.array_equal(res.worker_ask, wk)
    assert res.stats["n_bumped"] == ev.n_bumped


def check_diagnostics(res, ev, name):
    s = res.stats
    must = ev.batches_must_run()
    if ev.W > 50_000:
        print(f"\n[proximity grid] {name}: W = {ev.W}, {n_ctas(ev.W)} CTAs, {len(ev.cfg)} groups, batches = {s['n_tiles']}, "
              f"groups formed in batches = {s['n_rounds']}, one at a time = {s['n_build_launches']}")
    assert s["n_rounds"] + s["n_build_launches"] == ev.grouped_non_solo()
    if n_ctas(ev.W) == 1:
        assert s["n_tiles"] == 0 and s["n_rounds"] == 0
    assert s["n_tiles"] >= len(must) and s["n_rounds"] >= len(must)      # every such configuration opens a batch


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("name", sorted(CASES))
def test_proximity_sweep_past_the_first_chunk(name, kernel):
    """Every input on every kernel; a second pass on the same engine reuses every buffer."""
    ev = guard(name)
    eng = new_engine(kernel)
    load(eng, ev.case)
    for _ in range(2):
        eng.match(abi.PM_MODE_PROXIMITY)
        res = eng.fetch()
        check(res, ev)
        if kernel == "grid":
            check_diagnostics(res, ev, name)
    eng.close()


@pytest.mark.parametrize("n_shards", [2, 3])
@pytest.mark.parametrize("name", ["cascade", "handdown_sizes"])
def test_sharded_proximity_sweep(name, n_shards):
    """The grid kernel after the exchange (several engines on one GPU, merged here as the collective merges them), on
    the enabled asks alone (a sharded pass sees the table its caller compacted)."""
    ev = guard(name)
    t = enabled_tables(ev.case)
    for res in sharded_pass_on_one_gpu(t, n_shards, abi.PM_MODE_PROXIMITY, addr_rank=ev.case.rank, locations=True):
        check(res, ev, cfg=ev.og.cfg)


def test_incremental_pass_after_a_long_cascade():
    """The sweep rewrites each handed-down worker's current ask (the `cur` array) all along the cascade; an incremental
    pass after a few written rows must start from the stored evaluation, not from what the sweep left there.  Rows
    written: five chain workers become count-6 (they now reach the (0, 3) asks), three move city, four synth workers
    go unhealthy."""
    ev = guard("cascade")
    case = ev.case
    eng = new_engine("grid")
    load(eng, case)
    eng.match(abi.PM_MODE_PROXIMITY | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS)
    check(eng.fetch(), ev)
    t2 = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in case.t.items()}
    fives = case.fives
    idx = np.concatenate([fives[[3, 17, 40, 77, 120]], fives[[5, 60, 99]], [10, 5000, 15000, 19000]]).astype(np.uint32)
    t2["wa"]["gpu_count"][fives[[3, 17, 40, 77, 120]]] = 6
    t2["lat"][fives[[5, 60, 99]]], t2["lon"][fives[[5, 60, 99]]] = t2["lat"][fives[0]], t2["lon"][fives[0]]
    t2["wa"]["flags"][[10, 5000, 15000, 19000]] &= ~np.uint32(abi.PM_W_HEALTHY)
    eng.update_workers(idx, t2["wa"][idx], t2["wb"][idx], t2["lat"][idx], t2["lon"][idx])
    ev2 = Evidence(Case(t2, case.on, case.rank))
    assert ev2.n_bumped != ev.n_bumped or not np.array_equal(ev2.og.members, ev.og.members)
    for _ in range(2):
        eng.match(abi.PM_MODE_PROXIMITY | INCR)
        check(eng.fetch(), ev2)
    eng.close()
