"""The auction state restore (pm_auction_restore) at 100k asks x 1M workers, BASELINE configs[2]'s instance (the one
tools/auction_warm_bench.py and tests/test_gpu_auction_warm.py build).

Engine A runs one cold auction pass and exports its state (pm_auction_state + pm_auction_assignment).  Engine B, a fresh
engine with the same tables, as after a restart, restores it: warm-up calls, then repeated restores timed with a host
clock around each (the call ends in a device synchronise).  Then B's first warm pass from the restored state with no
change, and, from a fresh restore, its warm pass after 1 000 rewritten rows (half of them held, ask price halved), and
the same change once more repaired (PM_AUCTION_REPAIR).  A's cold pass is the comparison.  Prints one JSON line with the card's name and power limit read in the same run.

    python tools/auction_restore_bench.py [--reps 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
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

WARM = abi.PM_MODE_AUCTION | abi.PM_AUCTION_WARM


def load(a, wa, wb, bits, npat, nmod, words, cap):
    eng = Engine()
    eng.set_asks(a.asks, a.opts)
    eng.set_model_table(bits, npat, nmod, words)
    eng.set_workers(wa, wb)
    eng.set_price_caps(cap)
    return eng


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    gpu = card()
    a, wa, wb, bits, npat, nmod, words, cap = instance()
    T, W = len(cap), len(wa)
    eng_a = load(a, wa, wb, bits, npat, nmod, words, cap)
    _, cold_ms = timed(lambda: eng_a.match(abi.PM_MODE_AUCTION))
    price, assigned = eng_a.auction_state()[0], eng_a.auction_assignment()
    cert_a = eng_a.auction_certificate()
    eng_a.close()

    eng_b = load(a, wa, wb, bits, npat, nmod, words, cap)
    for _ in range(args.warmup):
        eng_b.auction_restore(price, assigned)
    ms = []
    for _ in range(args.reps):
        rep, t = timed(lambda: eng_b.auction_restore(price, assigned))
        ms.append(t)
    cert_b = eng_b.auction_certificate()
    _, warm0_ms = timed(lambda: eng_b.match(WARM))
    warm0 = eng_b.auction_state(prices=False)
    rounds0 = eng_b.stats()["n_rounds"]

    eng_b.auction_restore(price, assigned)
    rng = np.random.default_rng(5)
    held = assigned[assigned != abi.PM_NONE]
    idx = np.unique(np.concatenate([rng.choice(held, 500, replace=False), rng.choice(W, 500, replace=False)])).astype(np.uint32)
    b = wb[idx].copy()
    b["ext_ask_price"] = np.maximum(1, b["ext_ask_price"] // 2)
    eng_b.update_workers(idx, wa[idx], b)
    _, warm1k_ms = timed(lambda: eng_b.match(WARM))
    warm1k = eng_b.auction_state(prices=False)
    rounds1k = eng_b.stats()["n_rounds"]
    gap1k = eng_b.auction_certificate()["gap"]
    # the same change again from a fresh restore, repaired instead (PM_AUCTION_REPAIR keeps the stored prices)
    eng_b.update_workers(idx, wa[idx], wb[idx])
    eng_b.auction_restore(price, assigned)
    eng_b.update_workers(idx, wa[idx], b)
    _, repair1k_ms = timed(lambda: eng_b.match(WARM | abi.PM_AUCTION_REPAIR))
    repair1k = eng_b.auction_state(prices=False)
    repair_gap1k = eng_b.auction_certificate()["gap"]
    eng_b.close()
    med = float(np.median(ms))
    print(json.dumps(dict(
        case="restore_cfg3", n_asks=T, n_workers=W, cold_pass_ms=round(cold_ms, 1), restore_ms_median=round(med, 2),
        restore_ms_best=round(min(ms), 2), reps=args.reps, n_held=rep["n_held"],
        dropped=rep["n_dropped_bad"] + rep["n_dropped_shared"] + rep["n_dropped_slack"],
        same_certificate=cert_a == cert_b, warm_0_rows_ms=round(warm0_ms, 1), warm_0_rows_started_warm=warm0[1],
        warm_0_rows_rounds=rounds0, warm_1000_rows_ms=round(warm1k_ms, 1), warm_1000_rows_started_warm=warm1k[1],
        warm_1000_rows_released=warm1k[2], warm_1000_rows_rounds=rounds1k, warm_1000_rows_gap=gap1k,
        repair_1000_rows_ms=round(repair1k_ms, 1), repair_1000_rows_started_warm=repair1k[1],
        repair_1000_rows_released=repair1k[2], repair_1000_rows_gap=repair_gap1k, card=gpu)), flush=True)


if __name__ == "__main__":
    main()
