"""eps-scaled auction passes at 100k asks x 1M workers, BASELINE configs[2]'s instance (the one tools/auction_scale.py
and tests/test_gpu_auction_warm.py build): is eps-scaling with reverse rounds (PM_AUCTION_REVERSE) worth using?

Passes, alternated --reps times in one run on one engine:
  eps1          the default pass, eps = 1 throughout;
  fwd_64_4      eps-scaled without reverse rounds (64, 16, 4, 1: not sound, DESIGN 6d);
  rev_64_4      with reverse rounds, eps_start 64, eps_div 4;
  rev_1024_8    with reverse rounds, eps_start 1024, eps_div 8;
  rev_1         the bit with eps_start 1 (a single phase: nothing for the reverse rounds to do).
Per pass: wall ms (host clock around pm_match, which ends in a device synchronise), ms_fused (CUDA events around the
pass), ms_reverse (CUDA events around the reverse rounds, pm_stats.ms_build) and its share of ms_fused, forward rounds,
reverse rounds and bids, phases, and the total cost (sum of ask_price held + (cap + 1) for every ask holding nothing).
The card's name, power limit and SM clock are read in the same run.  One JSON line per pass; a summary on stderr.

    python tools/auction_scaling_bench.py [--reps 3] [--out results/auction_scaling.json]
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
CASES = [  # (name, reverse rounds, eps_start, eps_div)
    ("eps1", False, 1, 4),
    ("fwd_64_4", False, 64, 4),
    ("rev_64_4", True, 64, 4),
    ("rev_1024_8", True, 1024, 8),
    ("rev_1", True, 1, 4),
]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
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


def timed(eng, case, ap, cap):
    name, rev, eps_start, eps_div = case
    eng.set_auction_params(cost_scale=1, eps_start=eps_start, eps_div=eps_div)
    mode = abi.PM_MODE_AUCTION | (abi.PM_AUCTION_REVERSE if rev else 0)
    t0 = time.perf_counter()
    eng.match(mode)
    ms = (time.perf_counter() - t0) * 1e3
    st = eng.stats()
    phases, rev_rounds, bids = eng.auction_reverse_stats()
    res = eng.fetch()
    got = np.full(len(cap), NONE, dtype=np.uint32)
    got[res.group_ask] = res.group_members
    held = got != NONE
    cost = int(ap[got[held]].sum() + (cap[~held].astype(np.int64) + 1).sum())
    return dict(case=name, wall_ms=round(ms, 2), ms_fused=round(st["ms_fused"], 2), ms_reverse=round(st["ms_build"], 2),
                reverse_share=round(st["ms_build"] / st["ms_fused"], 4) if st["ms_fused"] else 0.0,
                forward_rounds=st["n_rounds"], reverse_rounds=rev_rounds, reverse_bids=bids, phases=phases,
                total_cost=cost, assigned=int(held.sum()), evals=st["evals"])


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--cases", default=",".join(c[0] for c in CASES))
    p.add_argument("--out", default=None)
    args = p.parse_args()
    gpu = card()
    print(f"card: {gpu}", file=sys.stderr)
    a, wa, wb, bits, npat, nmod, words, cap = instance()
    ap = wb["ext_ask_price"].astype(np.int64)
    eng = Engine(timing=True)
    eng.set_asks(a.asks, a.opts)
    eng.set_model_table(bits, npat, nmod, words)
    eng.set_workers(wa, wb)
    eng.set_price_caps(cap)
    cases = [c for c in CASES if c[0] in args.cases.split(",")]
    rows = []
    for rep in range(args.reps):
        for case in cases:
            r = dict(rep=rep, **timed(eng, case, ap, cap), card=gpu)
            rows.append(r)
            print(json.dumps(r), flush=True)
    eng.close()
    print(f"{'case':>12} {'rep':>3} {'wall ms':>9} {'ms_fused':>9} {'ms_rev':>8} {'share':>6} {'fwd':>6} {'rev':>6} {'bids':>9} "
          f"{'ph':>3} {'total cost':>11}", file=sys.stderr)
    for r in rows:
        print(f"{r['case']:>12} {r['rep']:>3} {r['wall_ms']:>9} {r['ms_fused']:>9} {r['ms_reverse']:>8} {r['reverse_share']:>6} "
              f"{r['forward_rounds']:>6} {r['reverse_rounds']:>6} {r['reverse_bids']:>9} {r['phases']:>3} {r['total_cost']:>11}",
              file=sys.stderr)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=gpu, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
