"""Device time per management pass, by kernel, on one benchmark workload (torch.profiler, CUDA activities).

    python tools/kernel_profile.py [--workload cfg3] [--passes 5] [--warmup 3] [--out DIR]

Builds bench.py's seeded tables, runs `--warmup` untimed materialised first-fit passes, then profiles `--passes` more
and prints one JSON line: per kernel its device time per pass (ms) and launches per pass, the sum over all kernels
and the wall time per pass between two device synchronisations.  Run it on its own, not beside a timed benchmark:
tracing slows the host.  With --out DIR the line is also written to DIR/kernel_profile_<workload>.json.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from protocol_b200 import abi
    from protocol_b200.engine import Engine

    if not torch.cuda.is_available():
        raise SystemExit("kernel_profile.py: no CUDA device")
    w, a, (bits, npat, nmod, words), (T, W, _, desc) = bench.make_tables(args.workload, 1, args.models)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        eng = Engine(device=0, cost_tile_bytes=8 << 30, stream=stream.cuda_stream)
        eng.set_asks(a.asks, a.opts)
        eng.set_model_table(bits, npat, nmod, words)
        eng.set_workers(w.a, w.b)
        mode = abi.PM_MODE_FIRST_FIT | abi.PM_PATH_MATERIALIZED
        for _ in range(args.warmup):
            eng.match(mode)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            for _ in range(args.passes):
                eng.match(mode)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) / args.passes * 1e3
        eng.close()
    per = collections.defaultdict(lambda: [0.0, 0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per[e.name][0] += e.device_time / 1e3 / args.passes   # us -> ms per pass
            per[e.name][1] += 1
    kernels = {k: {"ms_per_pass": round(v[0], 4), "launches_per_pass": v[1] / args.passes}
               for k, v in sorted(per.items(), key=lambda kv: -kv[1][0])}
    line = {"workload": f"{args.workload}: {desc}", "device": torch.cuda.get_device_name(0), "passes": args.passes,
            "ms_device_per_pass": round(sum(v[0] for v in per.values()), 4), "ms_wall_per_pass": round(wall, 4),
            "kernels": kernels}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"kernel_profile_{args.workload}.json"), "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
