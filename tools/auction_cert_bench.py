"""The auction certificate (pm_auction_certificate) at 100k asks x 1M workers, BASELINE configs[2]'s instance (the one
tools/auction_warm_bench.py and tests/test_gpu_auction_warm.py build).

One cold auction pass, then the certificate of its stored state: warm-up calls, then repeated calls timed with a host
clock around each (the call ends in a device synchronise).  Prints one JSON line: median and best ms, pairs/s at the
median, the gap and the hold counts, with the card's name and power limit read in the same run.

    python tools/auction_cert_bench.py [--reps 10] [--warmup 2]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    gpu = card()
    a, wa, wb, bits, npat, nmod, words, cap = instance()
    T, W = len(cap), len(wa)
    eng = Engine()
    eng.set_asks(a.asks, a.opts)
    eng.set_model_table(bits, npat, nmod, words)
    eng.set_workers(wa, wb)
    eng.set_price_caps(cap)
    t0 = time.perf_counter()
    eng.match(abi.PM_MODE_AUCTION)
    pass_ms = (time.perf_counter() - t0) * 1e3
    for _ in range(args.warmup):
        eng.auction_certificate()
    ms = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        c = eng.auction_certificate()
        ms.append((time.perf_counter() - t0) * 1e3)
    eng.close()
    med = float(np.median(ms))
    print(json.dumps(dict(
        case="certificate_cfg3", n_asks=T, n_workers=W, auction_pass_ms=round(pass_ms, 1), ms_median=round(med, 2),
        ms_best=round(min(ms), 2), reps=args.reps, pairs_per_s=float(f"{c['evals'] / (med * 1e-3):.4g}"), gap=c["gap"],
        cost=c["cost"], bound=c["bound"], n_held=c["n_held"], n_bad_holds=c["n_bad_holds"], n_shared=c["n_shared"],
        n_priced_unowned=c["n_priced_unowned"], n_slack_over=c["n_slack_over"], max_slack=c["max_slack"],
        card=gpu)), flush=True)


if __name__ == "__main__":
    main()
