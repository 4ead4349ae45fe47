"""Warm-started auction passes (PM_AUCTION_WARM) at 100k asks x 1M workers, BASELINE configs[2]'s instance (the one
tools/auction_scale.py and tests/test_gpu_parity.py build).

One cold pass, then warm passes after 0, 10, 1 000 and 100 000 rewritten worker rows, with the rows drawn from unowned
workers (nothing to release but the raised rows' own competition) and from owned workers (every owner released, and
the release cascades through its class), and after 100 changed caps.  Each warm pass is followed by a cold pass of
the same tables in the same run, so cold and warm times sit side by side.  Per pass: wall ms (host clock around
pm_match, which ends in a device synchronise), ms_fused (CUDA events around the pass), rounds, released asks, evals.
The card's name and power limit are read in the same run.  One JSON line per pass; a summary table on stderr.

--repair: every change set runs a warm pass, a warm repair (PM_AUCTION_WARM | PM_AUCTION_REPAIR: stored prices kept,
changed rows raised, reverse rounds at the end) and a cold pass, alternately, each warm or repair pass after a cold pass
of the current tables and a fresh draw of the same kind and number of changes.  Per pass also: reverse rounds and bids.

--asks: ask-table change sets instead (pm_update_asks / pm_resize_asks): append 1, 100 and 1 000 asks, replace 100,
remove the last 100 asks (most of them hold a worker).  Each runs as a warm pass, a warm repair and a cold pass on the
same tables, alternately, each warm or repair pass after a cold pass of the tables before the change; and as
pm_set_asks + a cold pass, the one way to take such a change without the deltas.

--splice: asks removed and inserted anywhere in the table (pm_remove_asks / pm_insert_asks): remove 1, 100 and 1 000
held asks at scattered positions, insert 1, 100 and 1 000 rows at random priorities (with caps).  Each runs as a warm
pass and a warm repair, each after a cold pass of the tables before the change, with the calls timed.  For comparison
each is also taken the way without the splices: pm_set_asks of the current rows, the caps, pm_auction_restore_slots of
the remapped export (the restore audit), then the same pass from the restored state.

--worker-splice: worker rows removed and inserted anywhere in the table (pm_remove_workers / pm_insert_workers):
remove 1, 100 and 1 000 held workers at scattered positions, insert 1, 100 and 1 000 rows (copies of other rows) at
random positions.  Each runs as a warm pass and a warm repair, each after a reload and a cold pass of the tables
before the change, with the calls timed.  For comparison each is also taken the way without the splices: the export
before the change (pm_auction_state, pm_auction_assignment), the indices remapped on the host, pm_set_worker_count +
the upload of the current rows, pm_auction_restore of the remapped state, then the same pass; `same_as_splice` says
whether that pass gave the same assignment and rounds.

    python tools/auction_warm_bench.py [--repair | --asks | --splice | --worker-splice] [--out results/auction_warm.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from protocol_b200 import abi, synth  # noqa: E402
from protocol_b200.engine import Engine  # noqa: E402

NONE = 0xFFFFFFFF


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as ex:   # noqa: BLE001
        return f"unknown ({ex})"


def instance():
    T, W = 100_000, 1_000_000
    w = synth.make_workers(W, seed=synth.SEED_WORKERS)
    a = synth.make_asks(T, "mixed", seed=synth.SEED_ASKS)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    wb = w.b.copy()
    wb["ext_ask_price"] = np.exp(np.log(10) + synth._unit(synth.SEED_EXT, W, 1) * np.log(200)).astype(np.uint32)
    cap = np.exp(np.log(20) + synth._unit(synth.SEED_EXT, T, 2) * np.log(150)).astype(np.uint32)
    return a, w.a.copy(), wb, bits, npat, nmod, words, cap


def timed(eng, mode):
    t0 = time.perf_counter()
    eng.match(mode)
    ms = (time.perf_counter() - t0) * 1e3
    st = eng.stats()
    _, warm, released = eng.auction_state(prices=False)
    _, rev_rounds, rev_bids = eng.auction_reverse_stats()
    return dict(wall_ms=round(ms, 2), ms_fused=round(st["ms_fused"], 2), rounds=st["n_rounds"], warm=warm,
                released=released, evals=st["evals"], rev_rounds=rev_rounds, rev_bids=rev_bids)


def assigned_of(eng, T):
    res = eng.fetch()
    got = np.full(T, NONE, dtype=np.uint32)
    got[res.group_ask] = res.group_members
    return got


def ask_series(eng, a, cap, record):
    """--asks: the change sets of the task-arrival loop, each as warm, repair, cold and pm_set_asks + cold."""
    rng = np.random.default_rng(3)
    asks, cap = a.asks.copy(), cap.copy()
    opts = a.opts   # every table below indexes these option rows (pm_set_asks gets them whole)

    def draw(n):
        """n new rows, copies of the instance's rows (their patterns are in the model table), with only their own
        option rows, as a caller sends a new task's."""
        src = a.asks[rng.integers(0, len(a.asks), n)]
        rows = src.copy()
        rows["opt_off"] = np.concatenate([[0], np.cumsum(src["n_opts"])[:-1]]).astype(np.uint32)
        own = np.concatenate([a.opts[o:o + k] for o, k in zip(src["opt_off"], src["n_opts"])] or [a.opts[:0]])
        return src, rows, own

    warm = abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM
    modes = [("warm", warm), ("repair", warm | abi.PM_AUCTION_REPAIR)]
    for case, n in (("append", 1), ("append", 100), ("append", 1000), ("replace", 100), ("remove", 100)):
        for name, mode in modes:
            eng.match(abi.PM_MODE_AUCTION)             # the stored state: a cold pass of the current tables
            T = len(asks)
            t0 = time.perf_counter()
            if case == "append":
                src, rows, own = draw(n)
                eng.resize_asks(T + n, rows, own)
                asks = np.concatenate([asks, src])
                cap = np.concatenate([cap, rng.integers(20, 3000, n).astype(np.uint32)])
                eng.set_price_caps(cap)
            elif case == "replace":
                idx = np.sort(rng.choice(T, n, replace=False)).astype(np.uint32)
                src, rows, own = draw(n)
                eng.update_asks(idx, rows, own)
                asks[idx] = src
            else:
                eng.resize_asks(T - n)
                asks, cap = asks[:T - n].copy(), cap[:T - n].copy()
            eng.sync()
            call_ms = round((time.perf_counter() - t0) * 1e3, 2)
            record(f"{name}_{case}", n, dict(timed(eng, mode), call_ms=call_ms))
            record(f"cold_{case}", n, timed(eng, abi.PM_MODE_AUCTION))
        t0 = time.perf_counter()                       # today's only option: the whole table again, then a cold pass
        eng.set_asks(asks, opts)
        eng.set_price_caps(cap)
        r = timed(eng, abi.PM_MODE_AUCTION)
        r["wall_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
        record(f"set_asks_cold_{case}", n, r)


def splice_series(eng, a, cap, record):
    """--splice: held asks removed at scattered positions and rows inserted at random priorities, each change set as a
    warm pass and a warm repair, then the same change taken by pm_set_asks + caps + pm_auction_restore_slots."""
    rng = np.random.default_rng(4)
    asks, cap = a.asks.copy(), cap.copy()
    warm = abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM
    for case, n in (("remove", 1), ("remove", 100), ("remove", 1000), ("insert", 1), ("insert", 100), ("insert", 1000)):
        for name, mode in (("warm", warm), ("repair", warm | abi.PM_AUCTION_REPAIR)):
            eng.set_asks(asks, a.opts)                 # the tables before the change, and a cold pass of them
            eng.set_price_caps(cap)
            eng.match(abi.PM_MODE_AUCTION)
            T = len(asks)
            if case == "remove":
                held = np.flatnonzero(assigned_of(eng, T) != NONE)
                idx = np.sort(rng.choice(held, n, replace=False)).astype(np.uint32)
                t0 = time.perf_counter()
                eng.remove_asks(idx)
                eng.sync()
                new_asks, new_cap = np.delete(asks, idx.astype(np.int64)), np.delete(cap, idx.astype(np.int64))
            else:
                before = np.sort(rng.integers(0, T + 1, n)).astype(np.uint32)
                src = a.asks[rng.integers(0, len(a.asks), n)]
                rows = src.copy()
                rows["opt_off"] = np.concatenate([[0], np.cumsum(src["n_opts"])[:-1]]).astype(np.uint32)
                own = np.concatenate([a.opts[o:o + k] for o, k in zip(src["opt_off"], src["n_opts"])] or [a.opts[:0]])
                b = before.astype(np.int64)
                new_asks = np.insert(asks, b, src)
                new_cap = np.insert(cap, b, rng.integers(20, 3000, n).astype(np.uint32))
                t0 = time.perf_counter()
                eng.insert_asks(before, rows, own)
                eng.set_price_caps(new_cap)
                eng.sync()
            call_ms = round((time.perf_counter() - t0) * 1e3, 2)
            price, _, _ = eng.auction_state()
            slots = eng.auction_slot_assignment()
            r = timed(eng, mode)
            got = assigned_of(eng, len(new_asks))
            record(f"{name}_{case}", n, dict(r, call_ms=call_ms))
            t0 = time.perf_counter()                   # the way without the splices
            eng.set_asks(new_asks, a.opts)
            eng.set_price_caps(new_cap)
            eng.auction_restore_slots(price, slots)
            eng.sync()
            restore_ms = round((time.perf_counter() - t0) * 1e3, 2)
            q = timed(eng, mode)
            same = bool(np.array_equal(assigned_of(eng, len(new_asks)), got) and q["rounds"] == r["rounds"])
            record(f"set_asks_restore_{name}_{case}", n, dict(q, call_ms=restore_ms, same_as_splice=same))
        asks, cap = new_asks, new_cap


def worker_splice_series(eng, wa, wb, record):
    """--worker-splice: held workers removed at scattered positions and rows inserted at random positions, each change
    set as a warm pass and a warm repair, then the same change taken by export + host remap + reload + restore."""
    rng = np.random.default_rng(5)
    wa, wb = wa.copy(), wb.copy()
    warm = abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM
    for case, n in (("remove", 1), ("remove", 100), ("remove", 1000), ("insert", 1), ("insert", 100), ("insert", 1000)):
        for name, mode in (("warm", warm), ("repair", warm | abi.PM_AUCTION_REPAIR)):
            eng.set_workers(wa, wb)                    # the tables before the change, and a cold pass of them
            eng.match(abi.PM_MODE_AUCTION)
            W, T = len(wa), eng.n_asks
            t0 = time.perf_counter()                   # the export the way without the splices starts from
            price0, _, _ = eng.auction_state()
            assigned0 = eng.auction_assignment()
            export_ms = (time.perf_counter() - t0) * 1e3
            held = assigned0 != NONE
            if case == "remove":
                idx = np.sort(rng.choice(assigned0[held], n, replace=False)).astype(np.uint32)
                t0 = time.perf_counter()
                eng.remove_workers(idx)
                eng.sync()
                i = idx.astype(np.int64)
                new_wa, new_wb = np.delete(wa, i), np.delete(wb, i)
            else:
                before = np.sort(rng.integers(0, W + 1, n)).astype(np.uint32)
                src = rng.integers(0, W, n)
                t0 = time.perf_counter()
                eng.insert_workers(before, wa[src], wb[src])
                eng.sync()
                b = before.astype(np.int64)
                new_wa, new_wb = np.insert(wa, b, wa[src]), np.insert(wb, b, wb[src])
            call_ms = round((time.perf_counter() - t0) * 1e3, 2)
            r = timed(eng, mode)
            got = assigned_of(eng, T)
            record(f"{name}_worker_{case}", n, dict(r, call_ms=call_ms))
            t0 = time.perf_counter()                   # the way without the splices
            a = assigned0.astype(np.int64)
            if case == "remove":
                gone = held & np.isin(a, i)
                price = np.delete(price0, i)
                a = np.where(held & ~gone, a - np.searchsorted(i, a), NONE)
            else:
                price = np.insert(price0, b, 0)
                a = np.where(held, a + np.searchsorted(b, a, "right"), NONE)
            eng.set_workers(new_wa, new_wb)
            eng.auction_restore(price, a.astype(np.uint32))
            eng.sync()
            restore_ms = round(export_ms + (time.perf_counter() - t0) * 1e3, 2)
            q = timed(eng, mode)
            same = bool(np.array_equal(assigned_of(eng, T), got) and q["rounds"] == r["rounds"])
            record(f"reload_restore_{name}_worker_{case}", n, dict(q, call_ms=restore_ms, same_as_splice=same))
        wa, wb = new_wa, new_wb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--counts", default="0,10,1000,100000")
    ap.add_argument("--repair", action="store_true", help="also run PM_AUCTION_REPAIR on every change set")
    ap.add_argument("--asks", action="store_true", help="ask-table change sets (pm_update_asks / pm_resize_asks)")
    ap.add_argument("--splice", action="store_true", help="asks removed and inserted anywhere (pm_remove_asks / pm_insert_asks)")
    ap.add_argument("--worker-splice", dest="worker_splice", action="store_true",
                    help="workers removed and inserted anywhere (pm_remove_workers / pm_insert_workers)")
    args = ap.parse_args()
    gpu = card()
    print(f"card: {gpu}", file=sys.stderr)
    a, wa, wb, bits, npat, nmod, words, cap = instance()
    T, W = len(cap), len(wa)
    eng = Engine(timing=True)
    eng.set_asks(a.asks, a.opts)
    eng.set_model_table(bits, npat, nmod, words)
    eng.set_workers(wa, wb)
    eng.set_price_caps(cap)
    rows = []

    def record(case, n, r):
        r = dict(case=case, n=n, **r, card=gpu)
        rows.append(r)
        print(json.dumps(r), flush=True)

    if args.asks or args.splice or args.worker_splice:
        record("cold", 0, timed(eng, abi.PM_MODE_AUCTION))
        if args.worker_splice:
            worker_splice_series(eng, wa, wb, record)
        else:
            (splice_series if args.splice else ask_series)(eng, a, cap, record)
        eng.close()
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(dict(card=gpu, rows=rows), f, indent=1)
        return

    modes = [("warm", abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM)]
    if args.repair:
        modes.append(("repair", abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM | abi.PM_AUCTION_REPAIR))
    record("cold", 0, timed(eng, abi.PM_MODE_AUCTION))
    rng = np.random.default_rng(1)
    for variant in ("unowned", "owned"):
        for n in [int(x) for x in args.counts.split(",")]:
            for name, mode in modes:
                eng.match(abi.PM_MODE_AUCTION)             # the stored state: a cold pass of the current tables
                got = assigned_of(eng, T)
                owned = np.zeros(W, dtype=bool)
                owned[got[got != NONE]] = True
                pool = np.flatnonzero(owned if variant == "owned" else ~owned)
                idx = np.sort(rng.choice(pool, size=min(n, len(pool)), replace=False)).astype(np.uint32)
                if len(idx):
                    b = wb[idx].copy()
                    b["ext_ask_price"] = np.maximum(1, (b["ext_ask_price"] * rng.uniform(0.5, 1.5, len(idx))).astype(np.uint32))
                    wb[idx] = b
                    eng.update_workers(idx, wa[idx], b)
                record(f"{name}_rows_{variant}", int(len(idx)), timed(eng, mode))
            record("cold", 0, timed(eng, abi.PM_MODE_AUCTION))
    for name, mode in modes:
        eng.match(abi.PM_MODE_AUCTION)
        cap2 = cap.copy()                              # 100 caps changed against the stored pass's
        idx = rng.choice(T, 100, replace=False)
        cap2[idx] = np.maximum(1, (cap2[idx] * rng.uniform(0.5, 1.5, 100)).astype(np.uint32))
        eng.set_price_caps(cap2)
        record(f"{name}_caps", int((cap2 != cap).sum()), timed(eng, mode))
        cap = cap2
    record("cold", 0, timed(eng, abi.PM_MODE_AUCTION))
    eng.close()
    print(f"{'case':>22} {'n':>7} {'wall ms':>9} {'ms_fused':>9} {'rounds':>7} {'rev rnds':>8} {'rev bids':>10} {'warm':>5} "
          f"{'released':>9} {'evals':>14}", file=sys.stderr)
    for r in rows:
        print(f"{r['case']:>22} {r['n']:>7} {r['wall_ms']:>9} {r['ms_fused']:>9} {r['rounds']:>7} {r['rev_rounds']:>8} "
              f"{r['rev_bids']:>10} {int(r['warm']):>5} {r['released']:>9} {r['evals']:>14}", file=sys.stderr)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
