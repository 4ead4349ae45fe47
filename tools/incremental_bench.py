#!/usr/bin/env python
"""Incremental management passes (PM_INCREMENTAL) against the full fused lean pass, on resident tables.

    python tools/incremental_bench.py [--workers 1000000] [--asks 100000] [--rounds 3] [--out DIR]

Workload: synth.make_workers(1M) x synth.make_asks(100k, "mixed"), BASELINE configs[2]'s shape, tables resident on
one engine.  Per round, alternated: one full `fused_lean` pass (PM_PATH_FUSED | PM_NO_ASK_STATS), then incremental
passes after k changed rows for every k in K (random flag flips through set_flags, spec changes through
update_workers).  The incremental engine is created with PM_TUNE_INCR above every k, so it never falls back to a full
evaluation and the crossover shows.  For every k, a sibling engine that received the same calls runs the full pass
and every pm_fetch_result array is compared.  Device time is pm_stats.ms_total (CUDA events on the engine stream);
host time is the wall time around match() ending in a stream sync.  The card, its power limit and SM clock come from
the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from protocol_b200 import abi, synth  # noqa: E402
from protocol_b200.engine import Engine  # noqa: E402

LEAN = abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED | abi.PM_NO_ASK_STATS
INCR = LEAN | abi.PM_INCREMENTAL
K = (0, 10, 100, 1_000, 10_000, 100_000, 300_000)
FIELDS = ("worker_group", "worker_ask", "group_ask", "group_off", "group_members", "ask_best", "ask_count")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_mhz": int(sm), "sm_max_mhz": int(smax)}
    except Exception as ex:  # the numbers below still stand; the card is then unknown
        return {"name": None, "error": str(ex)}


def timed(eng, mode):
    t = time.perf_counter()
    eng.match(mode)
    eng.sync()
    wall = (time.perf_counter() - t) * 1e3
    st = eng.stats()
    return {"ms_device": st["ms_total"], "ms_host": wall, "evals": st["evals"], "n_tiles": st["n_tiles"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workers", type=int, default=1_000_000)
    ap.add_argument("--asks", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    w = synth.make_workers(args.workers)
    pool = synth.make_workers(200_000, seed=synth.SEED_WORKERS + 101)
    a = synth.make_asks(args.asks, "mixed")
    bits, npat, nmod, words = synth.intern_tables(w, a)
    os.environ["PM_TUNE_INCR"] = str(1 << 31)   # read at pm_create: never fall back, so the crossover shows
    inc = Engine(timing=True)
    del os.environ["PM_TUNE_INCR"]
    ref = Engine(timing=True)
    engines = (inc, ref)
    for e in engines:
        e.set_asks(a.asks, a.opts)
        e.set_model_table(bits, npat, nmod, words)
        e.set_workers(w.a, w.b)
        e.match(LEAN)   # warm-up: allocations, first launches
    W, T = len(w), len(a)
    wa = w.a.copy()
    rng = np.random.default_rng(2024)
    rows = {"full": []}
    rows.update({k: [] for k in K})
    checked = set()
    env = card()
    for rnd in range(args.rounds):
        rows["full"].append(timed(inc, LEAN))   # the full pass also refreshes the stored evaluation
        for k in K:
            if k:
                idx = rng.choice(W, k, replace=False).astype(np.uint32)
                half = k // 2
                fl, up = idx[:half], idx[half:]
                if len(fl):   # flag flips: assigned on / off, a heartbeat that turns a node (un)healthy
                    f = wa["flags"][fl] ^ np.where(rng.random(len(fl)) < 0.7, abi.PM_W_ASSIGNED, abi.PM_W_HEALTHY).astype(np.uint32)
                    wa["flags"][fl] = f
                    for e in engines:
                        e.set_flags(fl, f)
                src = rng.integers(0, len(pool), len(up))
                na, nb = pool.a[src].copy(), pool.b[src].copy()
                wa[up] = na
                for e in engines:   # spec changes: another node's row
                    e.update_workers(up, na, nb)
            rows[k].append(timed(inc, INCR))
            if k not in checked:   # the sibling's full pass on the same tables: every array equal
                r = inc.fetch()
                ref.match(LEAN)
                q = ref.fetch()
                same = all(np.array_equal(getattr(r, f), getattr(q, f)) for f in FIELDS)
                if not same:
                    raise SystemExit(f"k={k}: the incremental result differs from the full pass")
                checked.add(k)
    summary = []
    for key, rs in rows.items():
        summary.append({"k": key, "ms_device_median": float(np.median([r["ms_device"] for r in rs])),
                        "ms_host_median": float(np.median([r["ms_host"] for r in rs])),
                        "evals": int(rs[-1]["evals"]), "n_tiles": int(rs[-1]["n_tiles"]), "runs": len(rs)})
    out = {"workload": f"{T} asks x {W} workers (synth mixed), first fit, fused lean", "card": env,
           "checked_equal_to_full_pass": sorted(checked), "rows": summary}
    print(f"{env.get('name')}  power limit {env.get('power_limit_w')} W  SM {env.get('sm_mhz')}/{env.get('sm_max_mhz')} MHz")
    print(f"{'k':>8} {'device ms':>10} {'host ms':>9} {'evals':>16} {'n_tiles':>9}")
    for s in summary:
        print(f"{s['k']:>8} {s['ms_device_median']:>10.3f} {s['ms_host_median']:>9.3f} {s['evals']:>16} {s['n_tiles']:>9}")
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "incremental_bench.json"), "w") as f:
            json.dump(out, f, indent=1)
    for e in engines:
        e.close()


if __name__ == "__main__":
    main()
