"""The plugin over pm_multi (pm_plugin_create_multi): the management pass runs on several GPUs, each device evaluating
its share of the resident worker table incrementally, and publishes exactly what a plugin over one engine publishes.
Every test runs on pm_multi over device 0 alone, and over devices 0 and 1 and over every visible GPU (both skipped with
fewer than two).  Covered: a random history of node arrivals, status changes, deaths, task events (which toggle
configurations) and merge passes against a plugin over a plain Engine, both policies; per-device incremental stats; a
table call made directly on one device's engine forcing a full upload; the merge pass with solo groups of unstored
nodes; and a refused pass (proximity with an enabled max_group_size == 0 configuration) followed by recovery."""
import numpy as np
import pytest

from protocol_b200 import abi
from protocol_b200._lib import PrimeMatchError, load
from protocol_b200.engine import Engine, MultiEngine
from protocol_b200.plugin import NodeGroupConfiguration, NodeGroupsPlugin, NodeStatus, OrchestratorNode, Scheduler, Task
from protocol_b200.sharded import shard_range
from test_gpu_plugin_resident import addr, node

pytestmark = pytest.mark.gpu

DEVICE_SETS = ["multi_0", "multi_0_1", "multi_all"]


def devices_of(which):
    import torch

    n = torch.cuda.device_count()
    if which == "multi_0":
        return [0]
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    return [0, 1] if which == "multi_0_1" else list(range(n))


def configs(rng, n=24):
    return [NodeGroupConfiguration(f"cfg-{c}", mn, mn + int(rng.integers(0, 3)),
                                   f"gpu:count={[1, 2, 4, 8][c % 4]}" if c % 5 else None)
            for c, mn in enumerate(rng.integers(1, 4, n).tolist())]


def add_nodes(plugins, lo, hi):
    for i in range(lo, hi):
        nd = node(i, np.random.default_rng(i))
        for p in plugins:
            p.add_node(nd)


def settle(p):
    """Passes until one forms nothing: the members of new groups are rows the next pass uploads, so afterwards no row
    is waiting to be written."""
    while p.try_form_new_groups():
        pass


def assert_incremental(m, W, T, touched, what):
    """Each device walked exactly the touched rows in its share (no configuration was toggled) and evaluated fewer
    than T x its share's pairs."""
    touched = np.asarray(sorted(touched))
    for r in range(m.n):
        lo, hi = shard_range(W, m.n, r)
        st = m.stats(r)
        want = int(((touched >= lo) & (touched < hi)).sum())
        assert st["n_tiles"] == want, (what, r, st["n_tiles"], want)
        assert st["evals"] < T * (hi - lo), (what, r, st["evals"])


def assert_full(m, W, T, what):
    """A full-upload pass: every device evaluated every pair of its share."""
    for r in range(m.n):
        lo, hi = shard_range(W, m.n, r)
        assert m.stats(r)["evals"] == T * (hi - lo), (what, r, m.stats(r))


def close(*objs):
    for o in objs:   # plugins before the engines they use
        o.close()


# ------------------------------------------------------------------ 1. random history against the engine plugin
@pytest.mark.parametrize("proximity", [False, True], ids=["first_fit", "proximity"])
@pytest.mark.parametrize("which", DEVICE_SETS)
def test_random_history_equals_engine_plugin(which, proximity):
    devices = devices_of(which)
    rng = np.random.default_rng(41 + 2 * len(devices) + proximity)
    cfgs = [NodeGroupConfiguration("h100-trio", 3, 3, "gpu:count=8;gpu:model=H100"),
            NodeGroupConfiguration("pair", 2, 2, "gpu:count=8"), NodeGroupConfiguration("flex", 1, 4),
            NodeGroupConfiguration("solo", 1, 1, "gpu:count=1"), NodeGroupConfiguration("quad", 4, 4)]
    m, e = MultiEngine(devices), Engine()
    a = NodeGroupsPlugin(cfgs, engine=m, proximity_enabled=proximity)
    b = NodeGroupsPlugin(cfgs, engine=e, proximity_enabled=proximity)
    sa, sb = Scheduler(a), Scheduler(b)
    tasks = []
    n = 0
    for step in range(40):
        ops = [("add", i, int(rng.integers(0, 1 << 30))) for i in range(n, n + (600 if step == 0 else int(rng.integers(0, 30))))]
        n += len(ops)
        ops += [("status", int(rng.integers(0, n)),
                 int(rng.choice([NodeStatus.Healthy, NodeStatus.Dead, NodeStatus.Unhealthy, NodeStatus.Healthy])))
                for _ in range(int(rng.integers(0, 12)))]
        if rng.random() < 0.5 or not tasks:
            ops.append(("task+", Task(allowed_topologies=[c.name for c in cfgs if rng.random() < 0.4], created_at=step)))
        if tasks and rng.random() < 0.35:
            ops.append(("task-", tasks[int(rng.integers(0, len(tasks)))].id))
        for op in ops:
            for p in (a, b):
                if op[0] == "add":
                    p.add_node(node(op[1], np.random.default_rng(op[2])))
                elif op[0] == "status":
                    p.update_node_status(addr(op[1]), op[2])
                elif op[0] == "task+":
                    p.add_task(op[1])
                else:
                    p.delete_task(op[1])
            if op[0] == "task+":
                tasks.append(op[1])
            elif op[0] == "task-":
                tasks = [t for t in tasks if t.id != op[1]]
        fa, fb = a.try_form_new_groups(), b.try_form_new_groups()
        assert fa == fb, f"step {step}: {fa} vs {fb} groups formed"
        if step % 3 == 2:
            ma, mb = a.try_merge_solo_groups(), b.try_merge_solo_groups()
            assert ma == mb, f"step {step}: {ma} vs {mb} merged"
        assert a.get_all_groups() == b.get_all_groups(), f"step {step}: published groups differ"
        for i in rng.choice(n, min(n, 25), replace=False).tolist():
            assert sa.get_task_for_node(addr(i)) == sb.get_task_for_node(addr(i)), f"step {step}: node {i}"
    assert len(a.get_all_groups()) > 20
    close(a, b, m, e)


# ------------------------------------------------------------------ 2. the pass is incremental on every device
@pytest.mark.parametrize("which", DEVICE_SETS)
def test_tick_is_incremental_on_every_device(which):
    devices = devices_of(which)
    rng = np.random.default_rng(5)
    cfgs = configs(rng)
    T, W = len(cfgs), 6000
    m = MultiEngine(devices)
    p = NodeGroupsPlugin(cfgs, engine=m, proximity_enabled=False)
    p.add_task(Task(allowed_topologies=[c.name for c in cfgs]))
    add_nodes([p], 0, W)
    assert p.try_form_new_groups() > 0
    assert_full(m, W, T, "first pass")
    settle(p)
    for tick in range(6):
        touched = set(rng.integers(0, W, int(rng.integers(1, 60))).tolist())
        for i in touched:
            p.update_node_status(addr(i), int(rng.choice([NodeStatus.Healthy, NodeStatus.Unhealthy])))
        p.try_form_new_groups()
        assert_incremental(m, W, T, touched, f"tick {tick}")
        settle(p)
    close(p, m)


# ------------------------------------------------------------------ 3. a table call from outside is detected
@pytest.mark.parametrize("which", DEVICE_SETS)
def test_outside_table_call_forces_a_full_upload(which):
    devices = devices_of(which)
    rng = np.random.default_rng(9)
    cfgs = configs(rng)
    T, W = len(cfgs), 4000
    m, e = MultiEngine(devices), Engine()
    a = NodeGroupsPlugin(cfgs, engine=m, proximity_enabled=False)
    b = NodeGroupsPlugin(cfgs, engine=e, proximity_enabled=False)
    task = Task(allowed_topologies=[c.name for c in cfgs])
    for p in (a, b):
        p.add_task(task)
    add_nodes([a, b], 0, W)
    assert a.try_form_new_groups() == b.try_form_new_groups()
    lib = load()
    for i in range(m.n):
        touched = set(rng.integers(0, W, 30).tolist())
        for j in touched:
            for p in (a, b):
                p.update_node_status(addr(j), NodeStatus.Unhealthy)
        v = m.table_version()
        assert lib.pm_resize_workers(lib.pm_multi_engine(m._h, i), 0) == abi.PM_OK
        assert m.table_version() != v, f"device {i}: a table call on its engine left the version"
        assert a.try_form_new_groups() == b.try_form_new_groups()
        assert a.get_all_groups() == b.get_all_groups(), f"device {i}: published groups differ"
        assert_full(m, W, T, f"outside call on device {i}")
    settle(a)
    settle(b)
    touched = set(rng.integers(0, W, 30).tolist())
    for j in touched:
        for p in (a, b):
            p.update_node_status(addr(j), NodeStatus.Healthy)
    assert a.try_form_new_groups() == b.try_form_new_groups()
    assert a.get_all_groups() == b.get_all_groups()
    assert_incremental(m, W, T, touched, "after the outside calls")
    close(a, b, m, e)


# ------------------------------------------------------------------ 4. merge pass: solo groups of unstored nodes
@pytest.mark.parametrize("which", DEVICE_SETS)
def test_merge_pass_skips_solo_groups_of_unstored_nodes(which):
    """A restored solo group may name a node that is not in the node table yet; find_compatible_solo_groups treats it
    as compatible with nothing (mod.rs:733-741).  On a multi plugin the merge pass runs on device 0's sibling engine."""
    m = MultiEngine(devices_of(which))
    p = NodeGroupsPlugin([NodeGroupConfiguration("merge-config", 1, 3)], engine=m, proximity_enabled=False)
    p.add_task(Task(allowed_topologies=["merge-config"]))
    for i in range(3):
        p.add_node(OrchestratorNode(addr(i), p2p_id=f"p{i}"))
    p.restore_group("a1", "merge-config", [addr(0)])
    p.restore_group("a2", "merge-config", [addr(1)])
    p.restore_group("a3", "merge-config", [addr(77)])       # node 77 was never stored
    assert p.try_merge_solo_groups() == 1
    groups = {g["id"]: g for g in p.get_all_groups()}
    assert "a3" in groups and groups["a3"]["nodes"] == [addr(77)]
    merged = [g for g in groups.values() if len(g["nodes"]) == 2]
    assert len(merged) == 1 and sorted(merged[0]["nodes"]) == sorted([addr(0), addr(1)])
    close(p, m)


# ------------------------------------------------------------------ 5. a refused pass, then the next tick works
@pytest.mark.parametrize("which", DEVICE_SETS)
def test_refused_pass_is_retried_next_tick(which):
    """Proximity mode refuses an enabled max_group_size == 0 configuration on every device before the exchange.  With
    several devices that pass aborts the communicators; once the task that enabled it is deleted, the next pass
    re-creates them, runs in full and equals the engine plugin, and the passes after it are incremental again."""
    devices = devices_of(which)
    rng = np.random.default_rng(12)
    cfgs = configs(rng, 12) + [NodeGroupConfiguration("zero", 0, 0)]
    T, W = len(cfgs), 3000
    m, e = MultiEngine(devices), Engine()
    a = NodeGroupsPlugin(cfgs, engine=m, proximity_enabled=True)
    b = NodeGroupsPlugin(cfgs, engine=e, proximity_enabled=True)
    base = Task(allowed_topologies=[c.name for c in cfgs[:-1]], created_at=1)
    bad = Task(allowed_topologies=["zero"], created_at=2)
    for p in (a, b):
        p.add_task(base)
    add_nodes([a, b], 0, W)
    assert a.try_form_new_groups() == b.try_form_new_groups()
    for p in (a, b):
        p.add_task(bad)
        with pytest.raises(PrimeMatchError) as ei:
            p.try_form_new_groups()
        assert ei.value.status == abi.PM_E_UNSUPPORTED, str(ei.value)
        p.delete_task(bad.id)
    assert a.try_form_new_groups() == b.try_form_new_groups()
    assert a.get_all_groups() == b.get_all_groups()
    assert_full(m, W, T, "the pass after the refusal")
    settle(a)
    settle(b)
    assert a.get_all_groups() == b.get_all_groups()
    for tick in range(3):
        touched = set(rng.integers(0, W, 40).tolist())
        for j in touched:
            st = int(rng.choice([NodeStatus.Healthy, NodeStatus.Unhealthy]))
            for p in (a, b):
                p.update_node_status(addr(j), st)
        assert a.try_form_new_groups() == b.try_form_new_groups()
        assert a.get_all_groups() == b.get_all_groups(), f"tick {tick}"
        assert_incremental(m, W, T, touched, f"tick {tick}")
        settle(a)
        settle(b)
    close(a, b, m, e)
