#!/usr/bin/env python
"""A resident management tick of the plugin mirror (try_form_new_groups + try_merge_solo_groups), on a plugin over one
engine and on a plugin over pm_multi.

    python tools/plugin_tick_bench.py [--nodes 200000] [--configs 36] [--k 100] [--ticks 20] [--warmup 3]
                                      [--devices 0[,1,...]] [--first-fit] [--out DIR]

Workload: `--nodes` synthetic nodes (the shapes of tests/test_gpu_plugin_resident.py: 1 or 8 GPUs of three models,
a tenth without specs, four locations), `--configs` configurations with group sizes 1-5 and GPU-count requirements.
One task enables all but the last six configurations.  Between ticks: `--k` random status changes (Healthy, Unhealthy
or Dead; a death dissolves the node's group) and one task event, alternately creating a task that enables one of the
last six configurations and deleting it again.  The two plugins receive the same events and their ticks alternate,
the order swapped every tick; after every tick both must publish the same groups.

Per tick and plugin: `tick_ms` (wall time of both passes), `form_ms` and `merge_ms`, `device_ms` (pm_stats.ms_total of
the formation pass per device, CUDA events on the engine stream), `host_ms` (form_ms minus the slowest device's
ms_total: the plugin's host work of the formation pass — collecting the written rows, the upload calls, reading the
result back and publishing the groups), `writeback_ms` (pm_plugin_redis_writeback, the tick's groups in the
reference's Redis key formats) and `evals` per device.  Prints one JSON line with the card (name, power limit, SM clock
of every device used, from the same run) and the median of each field; `--out DIR` also writes every tick."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from protocol_b200.engine import Engine, MultiEngine  # noqa: E402
from protocol_b200.plugin import (ComputeSpecs, GpuSpecs, NodeGroupConfiguration, NodeGroupsPlugin,  # noqa: E402
                                  NodeStatus, OrchestratorNode, Task)

MODELS = ["NVIDIA H100", "NVIDIA A100 80GB", "RTX 4090"]
CITIES = [(45.5186, -73.5545), (32.7942, -96.7475), (48.85, 2.35), None]
BUF = 1 << 28   # the JSON answers of 200k nodes outgrow the wrappers' default buffers


def addr(i):
    return "0x" + f"{(i * 2654435761) & 0xFFFFFFFF:08x}".upper() + f"{i:032x}"


def node(i, rng):
    spec = ComputeSpecs(gpu=GpuSpecs(count=int(rng.choice([1, 8])), model=MODELS[int(rng.integers(0, 3))], memory_mb=80000),
                        ram_mb=64000, storage_gb=1000) if rng.random() > 0.1 else None
    return OrchestratorNode(addr(i), status=NodeStatus.Healthy if rng.random() > 0.15 else NodeStatus.Discovered,
                            p2p_id=f"p2p-{i}" if rng.random() > 0.05 else None, compute_specs=spec,
                            location=CITIES[int(rng.integers(0, 4))])


def json_call(p, fn, buf):
    p._check(fn(p._h, buf, len(buf)))
    return buf.value


def cards(devices):
    q = "index,name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--id={','.join(map(str, devices))}", f"--query-gpu={q}",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        rows = []
        for line in out.strip().splitlines():
            i, name, pl, sm, smax = [x.strip() for x in line.split(",")]
            rows.append({"index": int(i), "name": name, "power_limit_w": float(pl), "sm_mhz": int(sm), "sm_max_mhz": int(smax)})
        return rows
    except Exception as ex:  # the numbers below still stand; the card is then unknown
        return [{"name": None, "error": str(ex)}]


def tick(p, stats, buf):
    t0 = time.perf_counter()
    formed = p.try_form_new_groups()
    t1 = time.perf_counter()
    merged = p.try_merge_solo_groups()
    t2 = time.perf_counter()
    st = stats()
    json_call(p, p._lib.pm_plugin_redis_writeback, buf)
    t3 = time.perf_counter()
    form_ms = (t1 - t0) * 1e3
    dev_ms = [s["ms_total"] for s in st]
    return {"tick_ms": (t2 - t0) * 1e3, "form_ms": form_ms, "merge_ms": (t2 - t1) * 1e3, "device_ms": dev_ms,
            "host_ms": form_ms - max(dev_ms), "writeback_ms": (t3 - t2) * 1e3, "evals": [s["evals"] for s in st],
            "formed": formed, "merged": merged}


def median(rows, key):
    v = np.array([r[key] for r in rows], dtype=float)
    return np.median(v, axis=0).round(3).tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=200_000)
    ap.add_argument("--configs", type=int, default=36)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--ticks", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--devices", default="0")
    ap.add_argument("--first-fit", action="store_true", help="ProximityOptimizationPolicy off (default: on)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    devices = [int(d) for d in args.devices.split(",")]
    card = cards(sorted(set(devices) | {0}))

    rng = np.random.default_rng(7)
    cfgs = [NodeGroupConfiguration(f"cfg-{c}", mn, mn + int(rng.integers(0, 3)),
                                   f"gpu:count={[1, 8][c % 2]}" if c % 5 else None)
            for c, mn in enumerate(rng.integers(1, 4, args.configs).tolist())]
    toggled = [c.name for c in cfgs[-6:]]
    eng, multi = Engine(timing=True), MultiEngine(devices, timing=True)
    prox = not args.first_fit
    plugins = {"engine": NodeGroupsPlugin(cfgs, engine=eng, proximity_enabled=prox),
               "multi": NodeGroupsPlugin(cfgs, engine=multi, proximity_enabled=prox)}
    stats = {"engine": lambda: [eng.stats()], "multi": lambda: [multi.stats(i) for i in range(multi.n)]}
    base = Task(allowed_topologies=[c.name for c in cfgs[:-6]], created_at=0)
    t_load = time.perf_counter()
    for p in plugins.values():
        p.add_task(base)
    for i in range(args.nodes):
        nd = node(i, np.random.default_rng(i))
        for p in plugins.values():
            p.add_node(nd)
    load_s = time.perf_counter() - t_load
    buf = C.create_string_buffer(BUF)

    def groups(name):
        p = plugins[name]
        return json_call(p, p._lib.pm_plugin_get_all_groups, buf)

    first = {}
    for name, p in plugins.items():   # the first tick uploads everything
        first[name] = tick(p, stats[name], buf)
    assert groups("engine") == groups("multi")

    rows = {"engine": [], "multi": []}
    extra = None
    for t in range(args.warmup + args.ticks):
        for i in rng.integers(0, args.nodes, args.k).tolist():
            st = int(rng.choice([NodeStatus.Healthy, NodeStatus.Unhealthy, NodeStatus.Dead]))
            for p in plugins.values():
                p.update_node_status(addr(i), st)
        if extra is None:
            extra = Task(allowed_topologies=[toggled[t % len(toggled)]], created_at=t + 1)
            for p in plugins.values():
                p.add_task(extra)
        else:
            for p in plugins.values():
                p.delete_task(extra.id)
            extra = None
        order = ["engine", "multi"] if t % 2 == 0 else ["multi", "engine"]
        for name in order:
            r = tick(plugins[name], stats[name], buf)
            if t >= args.warmup:
                rows[name].append(r)
        assert groups("engine") == groups("multi"), f"tick {t}: the two plugins publish different groups"

    summary = {
        "workload": {"nodes": args.nodes, "configs": args.configs, "k": args.k, "ticks": args.ticks,
                     "proximity": prox, "devices": devices, "load_s": round(load_s, 1)},
        "card": card,
        "first_tick": {n: {k: v for k, v in r.items() if k in ("tick_ms", "device_ms", "evals")} for n, r in first.items()},
        "same_groups": True,
        "groups": len(json.loads(groups("engine"))),
    }
    for name in rows:
        summary[name] = {k: median(rows[name], k) for k in ("tick_ms", "form_ms", "merge_ms", "device_ms", "host_ms",
                                                             "writeback_ms", "evals")}
    print(json.dumps(summary))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"plugin_tick_{'_'.join(map(str, devices))}.json"), "w") as f:
            json.dump(dict(summary, ticks=rows), f, indent=1)
    for p in plugins.values():
        p.close()
    eng.close()
    multi.close()


if __name__ == "__main__":
    main()
