"""Auction demands (pm_set_ask_demand) at cfg3 workers: the first 25 000 asks of BASELINE configs[2]'s instance (the one
tools/auction_warm_bench.py builds) with demands drawn from {1, 2, 4, 8} (D ~ 94 000 slots) x 1M workers.

* a cold pass with demands, and the same pass on the twin engine whose ask table repeats each row demand times;
* the cold state exported per slot (pm_auction_slot_assignment) and restored into a fresh engine with the same tables
  and demands (pm_auction_restore_slots): the restore and that engine's first warm pass, against the cold pass;
* from the demand engine's stored state, 1 / 100 / 1 000 demand changes (random asks, each demand moved by -2..+2),
  each followed by a warm pass, then another change of the same size followed by a repair pass (a chain: each step
  starts from the state the previous one left);
* what the twin needs for the 1 000-change step, which inserts and removes rows in the middle of its table:
  pm_set_asks + caps + a cold pass, or pm_set_asks + caps + pm_auction_restore of the remapped state + a warm pass.

Every time is a host clock around a call that ends in a device synchronise.  Prints one JSON line with the card's name
and power limit read in the same run.

    python tools/auction_demand_bench.py
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from auction_warm_bench import card, instance  # noqa: E402
from protocol_b200 import abi  # noqa: E402
from protocol_b200.engine import Engine  # noqa: E402

AUC = abi.PM_MODE_AUCTION
WARM = AUC | abi.PM_AUCTION_WARM
REPAIR = WARM | abi.PM_AUCTION_REPAIR
T = 25_000


def load(asks, opts, wa, wb, bits, npat, nmod, words, cap):
    eng = Engine()
    eng.set_asks(asks, opts)
    eng.set_model_table(bits, npat, nmod, words)
    eng.set_workers(wa, wb)
    eng.set_price_caps(cap)
    return eng


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, (time.perf_counter() - t0) * 1e3


def change(d, n, rng):
    d2 = d.copy()
    for t in rng.choice(len(d), n, replace=False):
        d2[t] = max(1, int(d2[t]) + int(rng.choice([-2, -1, 1, 2])))
    return d2


def main():
    gpu = card()
    a, wa, wb, bits, npat, nmod, words, cap = instance()
    asks, cap = np.ascontiguousarray(a.asks[:T]), cap[:T]
    rng = np.random.default_rng(11)
    d = rng.choice([1, 2, 4, 8], T).astype(np.uint32)
    out = dict(case="demand_cfg3", n_asks=T, n_workers=len(wa), n_slots=int(d.sum()))

    eng = load(asks, a.opts, wa, wb, bits, npat, nmod, words, cap)
    eng.set_ask_demand(d)
    _, out["cold_ms"] = timed(lambda: eng.match(AUC))
    out["cold_rounds"] = eng.stats()["n_rounds"]
    out["cold_gap"] = eng.auction_certificate()["gap"]
    twin = load(np.repeat(asks, d), a.opts, wa, wb, bits, npat, nmod, words, np.repeat(cap, d))
    _, out["twin_cold_ms"] = timed(lambda: twin.match(AUC))
    out["twin_same_prices"] = bool(np.array_equal(eng.auction_state()[0], twin.auction_state()[0]))

    # a restart: the cold state exported per slot and restored into a fresh engine with the same tables and demands
    price, slots = eng.auction_state()[0], eng.auction_slot_assignment()
    moved = load(asks, a.opts, wa, wb, bits, npat, nmod, words, cap)
    moved.set_ask_demand(d)
    rep, ms = timed(lambda: moved.auction_restore_slots(price, slots))
    out["restore_ms"] = round(ms, 1)
    out["restore_held"] = rep["n_held"]
    out["restore_dropped"] = rep["n_dropped_bad"] + rep["n_dropped_shared"] + rep["n_dropped_slack"]
    _, ms = timed(lambda: moved.match(WARM))
    out["restore_first_warm_ms"] = round(ms, 1)
    out["restore_first_warm_started_warm"] = moved.auction_state(prices=False)[1]
    out["restore_first_warm_rounds"] = moved.stats()["n_rounds"]
    moved.close()

    d_twin = d   # the twin's table stays at the first demands
    for n in (1, 100, 1000):
        d = change(d, n, rng)
        _, ms_set = timed(lambda: eng.set_ask_demand(d))
        _, ms = timed(lambda: eng.match(WARM))
        st = eng.auction_state(prices=False)
        out[f"warm_{n}_set_ms"] = round(ms_set, 2)
        out[f"warm_{n}_ms"] = round(ms, 1)
        out[f"warm_{n}_started_warm"], out[f"warm_{n}_released"] = st[1], st[2]
        out[f"warm_{n}_gap"] = eng.auction_certificate()["gap"]
        if n == 1000:   # the twin's way to the same table: rows inserted and removed in the middle
            t_price, t_assigned = twin.auction_state()[0], twin.auction_assignment()
            o_prev = np.concatenate([[0], np.cumsum(d_twin, dtype=np.int64)])
            o_new = np.concatenate([[0], np.cumsum(d, dtype=np.int64)])
            remapped = np.full(int(o_new[-1]), abi.PM_NONE, dtype=np.uint32)
            for t in range(T):
                k = min(int(d_twin[t]), int(d[t]))
                remapped[o_new[t]:o_new[t] + k] = t_assigned[o_prev[t]:o_prev[t] + k]
            twin_asks, twin_cap = np.repeat(asks, d), np.repeat(cap, d)

            def twin_cold():
                twin.set_asks(twin_asks, a.opts)
                twin.set_price_caps(twin_cap)
                twin.match(AUC)
            _, out["twin_1000_set_asks_cold_ms"] = timed(twin_cold)

            def twin_restore_warm():
                twin.set_asks(twin_asks, a.opts)
                twin.set_price_caps(twin_cap)
                twin.auction_restore(t_price, remapped)
                twin.match(WARM)
            _, out["twin_1000_set_asks_restore_warm_ms"] = timed(twin_restore_warm)
        d = change(d, n, rng)
        eng.set_ask_demand(d)
        _, ms = timed(lambda: eng.match(REPAIR))
        st = eng.auction_state(prices=False)
        out[f"repair_{n}_ms"] = round(ms, 1)
        out[f"repair_{n}_started_warm"], out[f"repair_{n}_released"] = st[1], st[2]
        out[f"repair_{n}_gap"] = eng.auction_certificate()["gap"]
    out["cold_ms"], out["twin_cold_ms"] = round(out["cold_ms"], 1), round(out["twin_cold_ms"], 1)
    for k in ("twin_1000_set_asks_cold_ms", "twin_1000_set_asks_restore_warm_ms"):
        out[k] = round(out[k], 1)
    out["card"] = gpu
    eng.close()
    twin.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
