"""The resolution kernels past their first stride: pm_sweep (first-fit under-filled tails handed to later
configurations) and pm_merge_sweep (try_merge_solo_groups under the proximity policy), single CTAs of 1024 threads.

Inputs and the guards proving that each reaches its path live in tests/test_resolution_sweep_inputs.py, which runs
them on the CPU.  Here the engine's groups are compared with the oracle: first-fit with orc.soa_form_groups (the
per-configuration loop, not the hand-down formulation), merging through the plugin with orc.merge_solo_groups.  The
engine's own count of hand-downs (stats["n_bumped"]) must equal the number the oracle's groups imply.
"""
import os

import numpy as np
import pytest

from helpers import assert_distance_certificate, groups_equal, load_engine
from oracle import pm_oracle as orc
from protocol_b200 import abi
from protocol_b200.engine import Engine
from protocol_b200.plugin import ComputeSpecs, GpuSpecs, NodeGroupConfiguration, NodeGroupsPlugin, OrchestratorNode, Task
from test_gpu_sharded import sharded_pass_on_one_gpu
from test_resolution_sweep_inputs import (MERGE_CASES, NONE, first_fit_case, guard_first_fit, guard_merge, guard_wide,
                                          merge_oracle_setup, oracle_groups, sweep_trace, wide)

pytestmark = pytest.mark.gpu

MAT, FUSED, LEAN = abi.PM_PATH_MATERIALIZED, abi.PM_PATH_FUSED, abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS
PATHS = pytest.mark.parametrize("path", [MAT, FUSED, LEAN], ids=["materialized", "fused", "fused_lean"])


def per_worker(og, W):
    wg = np.full(W, NONE, dtype=np.uint32)
    wk = np.full(W, NONE, dtype=np.uint32)
    for g in range(len(og.cfg)):
        m = og.members[og.off[g]:og.off[g + 1]]
        wg[m], wk[m] = g, og.cfg[g]
    return wg, wk


def check(res, og, W, n_bumped):
    assert groups_equal(res, og), f"groups differ: engine {res.n_groups} vs oracle {len(og)}"
    wg, wk = per_worker(og, W)
    assert np.array_equal(res.worker_group, wg) and np.array_equal(res.worker_ask, wk)
    assert res.stats["n_bumped"] == n_bumped


def _engine(generic=False, **kw):
    if generic:
        os.environ["PM_TUNE_GENERIC"] = "1"        # read at pm_create
    try:
        return Engine(**kw)
    finally:
        os.environ.pop("PM_TUNE_GENERIC", None)


# ------------------------------------------------------------------------------------------------ pm_sweep
@PATHS
@pytest.mark.parametrize("name", ["many_configs", "late_tails", "cascade", "big_pops"])
def test_sweep_past_the_first_chunk(name, path):
    """Cases 1-5 and 7: bad tails at 1023 / 1024 / 2047 / 2048 and throughout 5000 configurations; a 2200-link cascade
    whose links hold only handed-down workers, with max_group_size 0 and min_group_size 0 asks among them; pops of
    1100 and of 50; pops alternating between the base segment and the handed-down list; a group of 3000 members in
    address-rank order."""
    t, rank, og, tr = first_fit_case(name)
    n_bumped = guard_first_fit(name, t, og, tr)
    eng = Engine(cost_tile_bytes=64 << 20)
    load_engine(eng, t, addr_rank=rank)
    eng.match(abi.PM_MODE_FIRST_FIT | path)
    check(eng.fetch(), og, len(t["wa"]), n_bumped)
    eng.close()


@pytest.mark.parametrize("generic", [False, True], ids=["range_checked", "generic_forced"])
@PATHS
def test_sweep_hands_down_on_wide_operands(path, generic):
    """Case 6: operands >= 2^31 and a count x memory product that wraps decide where handed-down workers go."""
    t, rank, og, tr = first_fit_case("large_operands")
    n_bumped = guard_first_fit("large_operands", t, og, tr)
    eng = _engine(generic)
    load_engine(eng, t)
    eng.match(abi.PM_MODE_FIRST_FIT | path)
    check(eng.fetch(), og, len(t["wa"]), n_bumped)
    eng.close()


@pytest.mark.parametrize("n_models,n_patterns", [(200, 112), (3000, 112), (3000, 30)],
                         ids=["bits1", "bits0", "worker_major"])
@PATHS
def test_sweep_hands_down_past_acceptance_word_zero(n_models, n_patterns, path):
    """Case 6: the evaluation kernels decide first_ask with the BITS = 1 / 0 tables or the worker-major acceptance
    word; the sweep decides each hand-down with ask_meets on the 31-models-per-word table.  Targets depend on models
    past the first word."""
    t, pbits = wide(n_models, n_patterns)
    og = oracle_groups(t)
    tr = sweep_trace(t, og)
    n_bumped = guard_wide(t, og, tr)
    eng = Engine(cost_tile_bytes=1 << 20)
    load_engine(eng, dict(t, bits=pbits))
    eng.match(abi.PM_MODE_FIRST_FIT | path)
    check(eng.fetch(), og, len(t["wa"]), n_bumped)
    eng.close()


def test_second_pass_reuses_sweep_buffers():
    """Case 8: the sweep's base_len / xhead / xcount / xnext are sized by the first pass (5000 configurations) and
    reused by a second one with 3000 configurations and some workers assigned or gone unhealthy."""
    t, rank, og, tr = first_fit_case("many_configs")
    eng = Engine()
    load_engine(eng, t, addr_rank=rank)
    eng.match(abi.PM_MODE_FIRST_FIT)
    check(eng.fetch(), og, len(t["wa"]), int(tr["pop"].sum()))
    t2 = dict(t)
    t2["asks"] = t["asks"][:3000].copy()
    n_opts = int(t2["asks"]["opt_off"][-1] + t2["asks"]["n_opts"][-1])
    t2["opts"] = t["opts"][:n_opts]
    rng = np.random.default_rng(8)
    idx = np.sort(rng.choice(60_000, 6000, replace=False)).astype(np.uint32)    # the planted count-3 chain stays
    flags = t["wa"]["flags"][idx].copy()
    flags[::2] |= abi.PM_W_ASSIGNED
    flags[1::2] &= ~np.uint32(abi.PM_W_HEALTHY)
    wa = t["wa"].copy()
    wa["flags"][idx] = flags
    t2["wa"] = wa
    og2 = oracle_groups(t2, rank)
    tr2 = sweep_trace(t2, og2)
    assert tr2["bad"][[1023, 1024, 2047, 2048]].all() and tr2["bad"][2049:].any() and tr2["pop"].sum() > 500
    eng.set_asks(t2["asks"], t2["opts"])
    eng.set_flags(idx, flags)
    for path in (MAT, LEAN):
        eng.match(abi.PM_MODE_FIRST_FIT | path)
        check(eng.fetch(), og2, len(wa), int(tr2["pop"].sum()))
    eng.close()


@pytest.mark.parametrize("n_shards", [2, 3])
def test_sharded_sweep_past_the_first_chunk(n_shards):
    """Case 9: the sweep after the exchange (several engines on one GPU, merged here as the collective merges them),
    over the 2200-link cascade."""
    t, rank, og, tr = first_fit_case("cascade")
    for res in sharded_pass_on_one_gpu(t, n_shards, abi.PM_MODE_FIRST_FIT):
        check(res, og, len(t["wa"]), int(tr["pop"].sum()))


# ------------------------------------------------------------------------------------------------ pm_merge_sweep
def merge_through_plugin(case, proximity=True):
    """Every node forms a solo group, then the merge configurations are enabled and the plugin merges; returns
    (plugin's merged groups, oracle's merged groups) as sorted (configuration, addresses) pairs."""
    w, onodes, avail, _ = merge_oracle_setup(case)
    spec = MERGE_CASES[case]
    located = (w.a["flags"] & abi.PM_W_HAS_LOC) != 0
    if located.any():
        assert_distance_certificate(w.lat, w.lon, located)
    cfgs = [NodeGroupConfiguration(name, mn, mx, req) for name, mn, mx, req in spec["cfgs"]]
    eng = Engine()
    plugin = NodeGroupsPlugin(cfgs, engine=eng, proximity_enabled=proximity)
    plugin.add_task(Task(allowed_topologies=["solo"]))
    for i in range(len(w)):
        f = int(w.a["flags"][i])
        spec_i = None
        if f & abi.PM_W_HAS_SPECS:
            spec_i = ComputeSpecs(gpu=GpuSpecs(count=int(w.a["gpu_count"][i]), model=w.model_strings[int(w.a["model_id"][i])],
                                               memory_mb=int(w.a["gpu_mem_mb"][i]) if f & abi.PM_W_HAS_GPU_MEM else None),
                                  cpu_cores=int(w.b["cpu_cores"][i]), ram_mb=int(w.b["ram_mb"][i]),
                                  storage_gb=int(w.b["storage_gb"][i]))
        loc = (float(w.lat[i]), float(w.lon[i])) if f & abi.PM_W_HAS_LOC else None
        plugin.add_node(OrchestratorNode(w.addresses[i], compute_specs=spec_i, location=loc))
    assert plugin.try_form_new_groups() == len(w)
    addr_to_idx = {nd.address.decode(): i for i, nd in enumerate(onodes)}
    solos = [(g["id"], addr_to_idx[g["nodes"][0]], False) for g in plugin.get_all_groups()]
    for c in cfgs:
        if c.name != "solo":
            plugin.enable_configuration(c.name)
    want = orc.merge_solo_groups(onodes, solos, avail, proximity=proximity)
    n_merged = plugin.try_merge_solo_groups()
    got = sorted((g["configuration_name"], tuple(g["nodes"])) for g in plugin.get_all_groups() if len(g["nodes"]) > 1)
    plugin.close()
    eng.close()
    # the oracle's groups in solo-list order, so the guard sees the list the kernel walks
    exp = sorted((avail[c][0], tuple(onodes[m].address.decode() for m in ms)) for c, ms in want.as_list())
    guard_merge(case, w, onodes, avail, want)
    assert n_merged == len(want)
    return got, exp


@pytest.mark.parametrize("case", sorted(MERGE_CASES))
def test_merge_sweep_past_the_first_stride(case):
    """Cases 1-5: more than 1024 nodes handed on by a configuration whose min exceeds its compatible count (bitonic
    stages with P > 1024, a 4000-entry list whose seeds and nearest members lie past the first stride); nobody located
    and batches of 1500 filled in list order; every distance tied within two points of 1700 and 1300 nodes; 1100
    configurations before the ones that merge."""
    got, exp = merge_through_plugin(case)
    assert got == exp


def test_first_fit_merge_hands_down_past_the_first_stride():
    """The other policy: first-fit batches cut like formation chunks (pm_sweep on the merge table) on the hand-down
    input."""
    got, exp = merge_through_plugin("handdown", proximity=False)
    assert got == exp
