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
the same run.

    python tools/incremental_bench.py --toggle [...]

The toggle series: configurations enabled and disabled between passes (pm_set_ask_enabled), no worker row written.
25 000 random asks start disabled, so there are asks to enable.  Per round and for every j in J, alternated with the
full fused lean pass: ceil(j/2) asks are disabled — half of them the asks that own the most workers, half asks that
own none — and j//2 disabled ones are enabled, then one incremental pass runs.  Same sibling check as above.

    python tools/incremental_bench.py --shards N [--toggle] [...]
    python tools/incremental_bench.py --multi [--toggle] [...]

The same two series on sharded engines, reported per rank.  --shards N: N shard engines on device 0 (pm_set_shard,
equal shares of the table), each pass pm_match_local on every shard, the merge of the three arrays (concatenate / min /
sum, as the collective does) and pm_match_finish.  Per rank: `ms_local_host` (wall time of pm_match_local ending in a
stream sync), `ms_fused` (device time of its evaluation kernels), `ms_total` (device, pm_match_local to the end of
pm_match_finish, so it includes the wait for the host merge).  --multi: pm_multi over every visible GPU,
pm_multi_match; per rank `ms_total`, `ms_exchange` and `exchange_bytes` as well.  Every step is checked against an
unsharded engine's full pass (pm_fetch_result of rank 0).

    python tools/incremental_bench.py --splice [...]

Asks removed and inserted anywhere in the table (pm_remove_asks / pm_insert_asks) between passes.  Per round and for
every s in S, after a full fused lean pass that refreshes the stored evaluation: s asks that hold a group are removed
at scattered positions, one PM_INCREMENTAL lean pass runs; then s rows (copies of the table's rows, with only their own
option rows) are inserted at random priorities and one more runs.  Each call is timed on the host clock around the call
and a synchronise.  For comparison a sibling engine takes the way without the splices, pm_set_asks of the current rows
and a full lean pass (timed together, `route`), and its result is checked equal to the incremental one.

    python tools/incremental_bench.py --worker-splice [...]

Worker rows removed and inserted anywhere in the table (pm_remove_workers / pm_insert_workers) between passes.  Per
round and for every s in S, after a full fused lean pass that refreshes the stored evaluation: s rows are removed at
scattered positions and one PM_INCREMENTAL lean pass runs; then s rows (copies of other nodes' rows) are inserted at
random positions and one more runs.  Each call is timed on the host clock around the call and a synchronise.  For
comparison a sibling engine takes the way without the splices, pm_set_worker_count + pm_upsert_workers of the current
rows and a full lean pass (timed together, `route`), and its result is checked equal to the incremental one."""
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
from protocol_b200.engine import Engine, MultiEngine  # noqa: E402
from protocol_b200.sharded import shard_range, wrap_device_buffers  # noqa: E402

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


J = (1, 10, 100, 1_000, 10_000, 50_000)


def same_as_full(inc, ref):
    r = inc.fetch()
    ref.match(LEAN)
    q = ref.fetch()
    return r, all(np.array_equal(getattr(r, f), getattr(q, f)) for f in FIELDS)


def toggle_series(args, w, a, bits, npat, nmod, words, env):
    os.environ["PM_TUNE_INCR"] = str(1 << 31)   # never fall back, so the crossover shows
    inc = Engine(timing=True)
    del os.environ["PM_TUNE_INCR"]
    ref = Engine(timing=True)
    engines = (inc, ref)
    W, T = len(w), len(a)
    rng = np.random.default_rng(2025)
    on = np.ones(T, bool)
    on[rng.choice(T, 25_000, replace=False)] = False
    for e in engines:
        e.set_asks(a.asks, a.opts)
        e.set_model_table(bits, npat, nmod, words)
        e.set_workers(w.a, w.b)
        e.set_ask_enabled(np.nonzero(~on)[0], False)
        e.match(LEAN)   # warm-up: allocations, first launches
    rows = {"full": []}
    rows.update({j: [] for j in J})
    checked = set()
    for rnd in range(args.rounds):
        for j in J:
            rows["full"].append(timed(inc, LEAN))   # refreshes the stored evaluation
            wk = inc.fetch().worker_ask
            owners = np.bincount(wk[wk != abi.PM_NONE], minlength=T)
            n_off, n_on = (j + 1) // 2, j // 2
            enabled = np.nonzero(on)[0]
            top = enabled[np.argsort(owners[enabled])[::-1][:(n_off + 1) // 2]]
            idle = enabled[owners[enabled] == 0]
            off = np.concatenate([top, rng.choice(idle, min(len(idle), n_off - len(top)), replace=False)])
            disabled = np.nonzero(~on)[0]
            en = rng.choice(disabled, min(n_on, len(disabled)), replace=False)
            for e in engines:
                e.set_ask_enabled(off, False)
                e.set_ask_enabled(en, True)
            on[off], on[en] = False, True
            rows[j].append(dict(timed(inc, INCR), n_off=len(off), n_on=len(en)))
            if j not in checked:
                _, same = same_as_full(inc, ref)
                if not same:
                    raise SystemExit(f"j={j}: the incremental result differs from the full pass")
                checked.add(j)
    for e in engines:
        e.close()
    return rows, checked, f"{T} asks x {W} workers (synth mixed, 25 000 asks disabled at the start), first fit, fused lean"


class Ranks:
    """Sharded engines with the interface the series need: `apply` a table call to every rank and to the unsharded
    sibling, `timed` one PM_INCREMENTAL (or full) pass returning per-rank rows, `same_as_full` against the sibling."""

    def __init__(self, n_shards, multi, n_workers):
        import torch

        os.environ["PM_TUNE_INCR"] = str(1 << 31)   # read at pm_create: never fall back, so the crossover shows
        if multi:
            self.devices = list(range(torch.cuda.device_count()))
            self.m = MultiEngine(self.devices, timing=True)
            self.engines = []
        else:
            self.m = None
            self.engines = [Engine(timing=True) for _ in range(n_shards)]
        del os.environ["PM_TUNE_INCR"]
        self.ref = Engine(timing=True)
        self.n_shards = len(self.devices) if multi else n_shards

    def apply(self, name, *args):
        for e in ([self.m] if self.m else self.engines) + [self.ref]:
            getattr(e, name)(*args)

    def set_ranges(self, W):
        for r, e in enumerate(self.engines):
            lo, hi = shard_range(W, self.n_shards, r)
            e.set_shard(lo, hi - lo)

    def timed(self, mode):
        import torch

        if self.m:
            t = time.perf_counter()
            self.m.match(mode)
            self.m._check(self.m._lib.pm_multi_sync(self.m._h))
            wall = (time.perf_counter() - t) * 1e3
            sts = [self.m.stats(i) for i in range(self.n_shards)]
            return {"ms_host": wall, "ranks": [{k: s[k] for k in ("ms_total", "ms_exchange", "exchange_bytes", "evals",
                                                                  "n_tiles")} for s in sts]}
        W, T = self.ref.n_workers, self.ref.n_asks
        local = []
        t = time.perf_counter()
        for e in self.engines:
            t0 = time.perf_counter()
            e.match_local(mode)
            e.sync()
            local.append((time.perf_counter() - t0) * 1e3)
        bufs = [wrap_device_buffers(e, W, T) for e in self.engines]
        first = torch.cat([bufs[r][0][slice(*shard_range(W, self.n_shards, r))] for r in range(self.n_shards)])
        best = torch.stack([b[1] for b in bufs]).min(dim=0).values
        cnt = torch.stack([b[2] for b in bufs]).sum(dim=0).to(torch.int32)
        for b in bufs:
            b[0].copy_(first)
            b[1].copy_(best)
            b[2].copy_(cnt)
        torch.cuda.synchronize()
        for e in self.engines:
            e.match_finish(mode)
            e.sync()
        wall = (time.perf_counter() - t) * 1e3
        sts = [e.stats() for e in self.engines]
        return {"ms_host": wall, "ranks": [dict(ms_local_host=lh, **{k: s[k] for k in ("ms_fused", "ms_total", "evals", "n_tiles")})
                                           for lh, s in zip(local, sts)]}

    def fetch(self):
        return self.m.fetch() if self.m else self.engines[0].fetch()

    def same_as_full(self):
        r = self.fetch()
        self.ref.match(LEAN)
        q = self.ref.fetch()
        return r, all(np.array_equal(getattr(r, f), getattr(q, f)) for f in FIELDS)

    def close(self):
        for e in ([self.m] if self.m else self.engines) + [self.ref]:
            e.close()


def sharded_series(args, w, a, bits, npat, nmod, words, pool):
    """The k series (pool given) or the toggle series (pool None) on Ranks; per-rank rows."""
    rk = Ranks(args.shards, args.multi, len(w))
    W, T = len(w), len(a)
    rk.apply("set_asks", a.asks, a.opts)
    rk.apply("set_model_table", bits, npat, nmod, words)
    rk.apply("set_workers", w.a, w.b)
    rk.set_ranges(W)
    rng = np.random.default_rng(2024 if pool is not None else 2025)
    on = np.ones(T, bool)
    if pool is None:
        on[rng.choice(T, 25_000, replace=False)] = False
        rk.apply("set_ask_enabled", np.nonzero(~on)[0], False)
    rk.timed(LEAN)   # warm-up: allocations, first launches
    wa = w.a.copy()
    keys = K if pool is not None else J
    rows = {"full": []}
    rows.update({k: [] for k in keys})
    checked = set()
    for rnd in range(args.rounds):
        for k in keys:
            if pool is None or k == keys[0]:
                rows["full"].append(rk.timed(LEAN))   # refreshes every rank's stored evaluation
            extra = {}
            if pool is not None and k:
                idx = rng.choice(W, k, replace=False).astype(np.uint32)
                fl, up = idx[:k // 2], idx[k // 2:]
                if len(fl):
                    f = wa["flags"][fl] ^ np.where(rng.random(len(fl)) < 0.7, abi.PM_W_ASSIGNED, abi.PM_W_HEALTHY).astype(np.uint32)
                    wa["flags"][fl] = f
                    rk.apply("set_flags", fl, f)
                src = rng.integers(0, len(pool), len(up))
                rk.apply("update_workers", up, pool.a[src].copy(), pool.b[src].copy())
            elif pool is None:
                wk = rk.fetch().worker_ask
                owners = np.bincount(wk[wk != abi.PM_NONE], minlength=T)
                n_off, n_on = (k + 1) // 2, k // 2
                enabled = np.nonzero(on)[0]
                top = enabled[np.argsort(owners[enabled])[::-1][:(n_off + 1) // 2]]
                idle = enabled[owners[enabled] == 0]
                off = np.concatenate([top, rng.choice(idle, min(len(idle), n_off - len(top)), replace=False)])
                en = rng.choice(np.nonzero(~on)[0], min(n_on, int((~on).sum())), replace=False)
                rk.apply("set_ask_enabled", off, False)
                rk.apply("set_ask_enabled", en, True)
                on[off], on[en] = False, True
                extra = {"n_off": len(off), "n_on": len(en)}
            rows[k].append(dict(rk.timed(INCR), **extra))
            _, same = rk.same_as_full()   # every step, against the sibling's full pass
            if not same:
                raise SystemExit(f"{k}: the incremental result differs from the full pass")
            checked.add(k)
    n = rk.n_shards
    rk.close()
    what = f"{n} shard engines on device 0" if not args.multi else f"pm_multi over {n} GPU(s)"
    return rows, checked, f"{T} asks x {W} workers (synth mixed), first fit, fused lean, {what}"


def report_ranks(rows, checked, workload, env, key_name, out_dir, file_name, multi):
    summary = []
    for key, rs in rows.items():
        n = len(rs[0]["ranks"])
        per = []
        for r in range(n):
            rr = [x["ranks"][r] for x in rs]
            d = {"rank": r, "evals": int(rr[-1]["evals"]), "n_tiles": int(rr[-1]["n_tiles"]),
                 "ms_total_median": float(np.median([x["ms_total"] for x in rr]))}
            if multi:
                d["ms_exchange_median"] = float(np.median([x["ms_exchange"] for x in rr]))
                d["exchange_bytes"] = int(rr[-1]["exchange_bytes"])
            else:
                d["ms_local_host_median"] = float(np.median([x["ms_local_host"] for x in rr]))
                d["ms_fused_median"] = float(np.median([x["ms_fused"] for x in rr]))
            per.append(d)
        summary.append({key_name: key, "ms_host_median": float(np.median([x["ms_host"] for x in rs])), "runs": len(rs),
                        "ranks": per, **{k: rs[-1][k] for k in ("n_off", "n_on") if k in rs[-1]}})
    out = {"workload": workload, "card": env, "checked_equal_to_full_pass": [str(c) for c in sorted(checked)],
           "rows": summary}
    if multi and len(summary[0]["ranks"]) < 2:
        out["note"] = "one GPU: multi-GPU numbers not measured"
    print(f"{env.get('name')}  power limit {env.get('power_limit_w')} W  SM {env.get('sm_mhz')}/{env.get('sm_max_mhz')} MHz")
    print(workload)
    cols = "ms_total ms_exchange   xchg_bytes" if multi else "ms_local_host ms_fused ms_total"
    print(f"{key_name:>8} {'rank':>4} {cols} {'evals':>16} {'n_tiles':>9}")
    for s in summary:
        for d in s["ranks"]:
            vals = (f"{d['ms_total_median']:>8.3f} {d['ms_exchange_median']:>11.3f} {d['exchange_bytes']:>12}" if multi else
                    f"{d['ms_local_host_median']:>13.3f} {d['ms_fused_median']:>8.3f} {d['ms_total_median']:>8.3f}")
            print(f"{s[key_name]:>8} {d['rank']:>4} {vals} {d['evals']:>16} {d['n_tiles']:>9}")
    print(json.dumps(out))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, file_name), "w") as f:
            json.dump(out, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workers", type=int, default=1_000_000)
    ap.add_argument("--asks", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--toggle", action="store_true", help="configurations toggled between passes instead of rows written")
    ap.add_argument("--shards", type=int, default=0, help="N shard engines on device 0 (pm_match_local + host merge)")
    ap.add_argument("--multi", action="store_true", help="pm_multi over every visible GPU")
    ap.add_argument("--ask-updates", dest="ask_updates", action="store_true",
                    help="asks replaced between passes (pm_update_asks) instead of rows written; also times the call")
    ap.add_argument("--splice", action="store_true",
                    help="asks removed and inserted anywhere between passes (pm_remove_asks / pm_insert_asks)")
    ap.add_argument("--worker-splice", dest="worker_splice", action="store_true",
                    help="worker rows removed and inserted anywhere between passes (pm_remove_workers / pm_insert_workers)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    w = synth.make_workers(args.workers)
    if args.ask_updates:
        a = synth.make_asks(args.asks, "mixed")
        bits, npat, nmod, words = synth.intern_tables(w, a)
        env = card()
        rows, checked, workload = ask_update_series(args, w, a, bits, npat, nmod, words)
        report(rows, checked, workload, env, "u", args.out, "incremental_ask_update_bench.json")
        return
    if args.splice:
        a = synth.make_asks(args.asks, "mixed")
        bits, npat, nmod, words = synth.intern_tables(w, a)
        env = card()
        rows, checked, workload = splice_series(args, w, a, bits, npat, nmod, words)
        report(rows, checked, workload, env, "case", args.out, "incremental_splice_bench.json")
        return
    if args.worker_splice:
        a = synth.make_asks(args.asks, "mixed")
        bits, npat, nmod, words = synth.intern_tables(w, a)
        env = card()
        pool = synth.make_workers(200_000, seed=synth.SEED_WORKERS + 101)
        rows, checked, workload = worker_splice_series(args, w, a, bits, npat, nmod, words, pool)
        report(rows, checked, workload, env, "case", args.out, "incremental_worker_splice_bench.json")
        return
    if args.shards or args.multi:
        a = synth.make_asks(args.asks, "mixed")
        bits, npat, nmod, words = synth.intern_tables(w, a)
        env = card()
        pool = None if args.toggle else synth.make_workers(200_000, seed=synth.SEED_WORKERS + 101)
        rows, checked, workload = sharded_series(args, w, a, bits, npat, nmod, words, pool)
        name = ("multi" if args.multi else f"shards{args.shards}") + ("_toggle" if args.toggle else "")
        report_ranks(rows, checked, workload, env, "j" if args.toggle else "k", args.out,
                     f"incremental_bench_{name}.json", args.multi)
        return
    if args.toggle:
        a = synth.make_asks(args.asks, "mixed")
        bits, npat, nmod, words = synth.intern_tables(w, a)
        env = card()
        rows, checked, workload = toggle_series(args, w, a, bits, npat, nmod, words, env)
        report(rows, checked, workload, env, "j", args.out, "incremental_toggle_bench.json")
        return

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
                _, same = same_as_full(inc, ref)
                if not same:
                    raise SystemExit(f"k={k}: the incremental result differs from the full pass")
                checked.add(k)
    for e in engines:
        e.close()
    report(rows, checked, f"{T} asks x {W} workers (synth mixed), first fit, fused lean", env, "k", args.out,
           "incremental_bench.json")


U = (1, 100, 1_000)


def own_options(src, opts):
    """Rows `src` (opt_off into `opts`) with only their own option rows, as a caller sends changed asks."""
    rows = src.copy()
    rows["opt_off"] = np.concatenate([[0], np.cumsum(src["n_opts"])[:-1]]).astype(np.uint32)
    own = np.concatenate([opts[o:o + k] for o, k in zip(src["opt_off"], src["n_opts"])] or [opts[:0]])
    return rows, own


def ask_update_series(args, w, a, bits, npat, nmod, words):
    """U asks replaced by other rows of the table (pm_update_asks) between passes: the incremental pass against the full
    one, the result checked equal once per U; then pm_update_asks itself (U rows, host clock around the call and a
    synchronise) at T = the table's asks and at T = 1M."""
    os.environ["PM_TUNE_INCR"] = str(1 << 31)   # read at pm_create: never fall back, so the crossover shows
    inc = Engine(timing=True)
    del os.environ["PM_TUNE_INCR"]
    ref = Engine(timing=True)
    engines = (inc, ref)
    for e in engines:
        e.set_asks(a.asks, a.opts)
        e.set_model_table(bits, npat, nmod, words)
        e.set_workers(w.a, w.b)
        e.match(LEAN)
    W, T = len(w), len(a)
    rng = np.random.default_rng(2026)
    rows = {"full": []}
    rows.update({u: [] for u in U})
    checked = set()
    for rnd in range(args.rounds):
        for u in U:
            rows["full"].append(timed(inc, LEAN))
            idx = np.sort(rng.choice(T, u, replace=False)).astype(np.uint32)
            new, own = own_options(a.asks[rng.integers(0, T, u)], a.opts)
            for e in engines:
                e.update_asks(idx, new, own)
            rows[u].append(timed(inc, INCR))
            if u not in checked:
                _, same = same_as_full(inc, ref)
                if not same:
                    raise SystemExit(f"u={u}: the incremental result differs from the full pass")
                checked.add(u)
    for e in engines:
        e.close()
    calls = []
    for n_asks in (T, 1_000_000):
        big = a if n_asks == T else synth.make_asks(n_asks, "mixed")
        e = Engine(timing=True)
        e.set_asks(big.asks, big.opts)
        for u in U:
            ms = []
            for _ in range(5):
                idx = np.sort(rng.choice(n_asks, u, replace=False)).astype(np.uint32)
                new, own = own_options(big.asks[rng.integers(0, n_asks, u)], big.opts)
                t = time.perf_counter()
                e.update_asks(idx, new, own)
                e.sync()
                ms.append((time.perf_counter() - t) * 1e3)
            calls.append({"n_asks": n_asks, "u": u, "ms_update_asks_median": float(np.median(ms))})
            print(json.dumps(calls[-1]))
        e.close()
    rows["update_asks_calls"] = calls
    return rows, checked, f"{T} asks x {W} workers (synth mixed), first fit, fused lean; u asks replaced per pass"


S = (1, 100, 1_000)


def splice_series(args, w, a, bits, npat, nmod, words):
    """S held asks removed at scattered positions, then S rows inserted at random priorities (pm_remove_asks /
    pm_insert_asks), each followed by one incremental pass; the calls timed; the sibling's pm_set_asks + full pass
    (`route`) timed and its result checked equal."""
    os.environ["PM_TUNE_INCR"] = str(1 << 31)   # read at pm_create: never fall back
    inc = Engine(timing=True)
    del os.environ["PM_TUNE_INCR"]
    ref = Engine(timing=True)
    for e in (inc, ref):
        e.set_asks(a.asks, a.opts)
        e.set_model_table(bits, npat, nmod, words)
        e.set_workers(w.a, w.b)
        e.match(LEAN)
    W = len(w)
    asks = a.asks.copy()   # the current rows, opt_off into a.opts
    rng = np.random.default_rng(2027)
    rows = {"full": []}
    calls, checked = [], set()
    for rnd in range(args.rounds):
        for n in S:
            rows["full"].append(timed(inc, LEAN))
            for case in ("remove", "insert"):
                T = len(asks)
                if case == "remove":
                    held = np.unique(inc.fetch().group_ask)
                    idx = np.sort(rng.choice(held, min(n, len(held)), replace=False)).astype(np.uint32)
                    t = time.perf_counter()
                    inc.remove_asks(idx)
                    inc.sync()
                    asks = np.delete(asks, idx.astype(np.int64))
                else:
                    before = np.sort(rng.integers(0, T + 1, n)).astype(np.uint32)
                    src = a.asks[rng.integers(0, len(a.asks), n)]
                    new, own = own_options(src, a.opts)
                    t = time.perf_counter()
                    inc.insert_asks(before, new, own)
                    inc.sync()
                    asks = np.insert(asks, before.astype(np.int64), src)
                calls.append({"case": case, "s": n, "n_asks": T, "ms_call": (time.perf_counter() - t) * 1e3})
                key = f"{case}_{n}"
                rows.setdefault(key, []).append(timed(inc, INCR))
                t = time.perf_counter()
                ref.set_asks(asks, a.opts)
                r = timed(ref, LEAN)
                r["ms_host"] = (time.perf_counter() - t) * 1e3
                rows.setdefault(f"route_{key}", []).append(r)
                q, got = ref.fetch(), inc.fetch()
                if not all(np.array_equal(getattr(got, f), getattr(q, f)) for f in FIELDS):
                    raise SystemExit(f"{key}: the incremental result differs from pm_set_asks + the full pass")
                checked.add(key)
    for e in (inc, ref):
        e.close()
    for c in calls:
        print(json.dumps(c))
    summary = []
    for case in ("remove", "insert"):
        for n in S:
            ms = [c["ms_call"] for c in calls if c["case"] == case and c["s"] == n]
            summary.append({"case": case, "s": n, "ms_call_median": float(np.median(ms)), "runs": len(ms)})
    rows["splice_calls"] = summary
    return rows, checked, (f"{len(a.asks)} asks x {W} workers (synth mixed), first fit, fused lean; s held asks removed, "
                           f"then s rows inserted, per pass")


def worker_splice_series(args, w, a, bits, npat, nmod, words, pool):
    """S worker rows removed at scattered positions, then S rows inserted at random positions (pm_remove_workers /
    pm_insert_workers), each followed by one incremental pass; the calls timed; the sibling's pm_set_worker_count +
    upload + full pass (`route`) timed and its result checked equal."""
    os.environ["PM_TUNE_INCR"] = str(1 << 31)   # read at pm_create: never fall back
    inc = Engine(timing=True)
    del os.environ["PM_TUNE_INCR"]
    ref = Engine(timing=True)
    for e in (inc, ref):
        e.set_asks(a.asks, a.opts)
        e.set_model_table(bits, npat, nmod, words)
        e.set_workers(w.a, w.b)
        e.match(LEAN)
    wa, wb = w.a.copy(), w.b.copy()   # the current rows
    rng = np.random.default_rng(2028)
    rows = {"full": []}
    calls, checked = [], set()
    for rnd in range(args.rounds):
        for n in S:
            rows["full"].append(timed(inc, LEAN))
            for case in ("remove", "insert"):
                W = len(wa)
                if case == "remove":
                    idx = np.sort(rng.choice(W, n, replace=False)).astype(np.uint32)
                    t = time.perf_counter()
                    inc.remove_workers(idx)
                    inc.sync()
                    wa, wb = np.delete(wa, idx.astype(np.int64)), np.delete(wb, idx.astype(np.int64))
                else:
                    before = np.sort(rng.integers(0, W + 1, n)).astype(np.uint32)
                    src = rng.integers(0, len(pool), n)
                    na, nb = pool.a[src].copy(), pool.b[src].copy()
                    t = time.perf_counter()
                    inc.insert_workers(before, na, nb)
                    inc.sync()
                    b = before.astype(np.int64)
                    wa, wb = np.insert(wa, b, na), np.insert(wb, b, nb)
                calls.append({"case": case, "s": n, "n_workers": W, "ms_call": (time.perf_counter() - t) * 1e3})
                key = f"{case}_{n}"
                rows.setdefault(key, []).append(timed(inc, INCR))
                t = time.perf_counter()
                ref.set_workers(wa, wb)
                r = timed(ref, LEAN)
                r["ms_host"] = (time.perf_counter() - t) * 1e3
                rows.setdefault(f"route_{key}", []).append(r)
                q, got = ref.fetch(), inc.fetch()
                if not all(np.array_equal(getattr(got, f), getattr(q, f)) for f in FIELDS):
                    raise SystemExit(f"{key}: the incremental result differs from pm_set_worker_count + upload + the full pass")
                checked.add(key)
    for e in (inc, ref):
        e.close()
    for c in calls:
        print(json.dumps(c))
    summary = []
    for case in ("remove", "insert"):
        for n in S:
            ms = [c["ms_call"] for c in calls if c["case"] == case and c["s"] == n]
            summary.append({"case": case, "s": n, "ms_call_median": float(np.median(ms)), "runs": len(ms)})
    rows["splice_calls"] = summary
    return rows, checked, (f"{len(a.asks)} asks x {len(w)} workers (synth mixed), first fit, fused lean; s worker rows "
                           f"removed, then s rows inserted, per pass")


def report(rows, checked, workload, env, key_name, out_dir, file_name):
    extra = {k: rows.pop(k) for k in ("update_asks_calls", "splice_calls") if k in rows}
    summary = []
    for key, rs in rows.items():
        summary.append({key_name: key, "ms_device_median": float(np.median([r["ms_device"] for r in rs])),
                        "ms_host_median": float(np.median([r["ms_host"] for r in rs])),
                        "evals": int(rs[-1]["evals"]), "n_tiles": int(rs[-1]["n_tiles"]), "runs": len(rs),
                        **{k: rs[-1][k] for k in ("n_off", "n_on") if k in rs[-1]}})
    out = {"workload": workload, "card": env, "checked_equal_to_full_pass": sorted(checked), "rows": summary}
    out.update(extra)
    print(f"{env.get('name')}  power limit {env.get('power_limit_w')} W  SM {env.get('sm_mhz')}/{env.get('sm_max_mhz')} MHz")
    print(f"{key_name:>16} {'device ms':>10} {'host ms':>9} {'evals':>16} {'n_tiles':>9}")
    for s in summary:
        print(f"{s[key_name]:>16} {s['ms_device_median']:>10.3f} {s['ms_host_median']:>9.3f} {s['evals']:>16} {s['n_tiles']:>9}")
    print(json.dumps(out))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, file_name), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
