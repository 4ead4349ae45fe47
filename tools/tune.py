"""Kernel-shape experiments on an H100: PM_TUNE_* variants, per-kernel CUDA-event times.
usage: python tools/tune.py [n_asks n_workers]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import peaks
from protocol_b200 import abi, synth
from protocol_b200.engine import Engine

T = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000
W = int(sys.argv[2]) if len(sys.argv) > 2 else 100_000
w = synth.make_workers(W)
a = synth.make_asks(T, "mixed")
bits, npat, nmod, words = synth.intern_tables(w, a)
PEAK, PEAK_SOURCE = peaks(torch.cuda.get_device_name(0))   # GB/s of the device's data sheet, None when unknown


def run(env, steps=4, mode=abi.PM_MODE_FIRST_FIT):
    for k in list(os.environ):
        if k.startswith("PM_TUNE_"):
            del os.environ[k]
    os.environ.update(env)
    eng = Engine(timing=True)
    eng.set_asks(a.asks, a.opts)
    eng.set_model_table(bits, npat, nmod, words)
    eng.set_workers(w.a, w.b)
    eng.match(mode)
    acc = {}
    for _ in range(steps):
        eng.match(mode)
        st = eng.stats()
        for k in ("ms_build", "ms_argmin", "ms_fused", "ms_resolve", "ms_total"):
            acc[k] = acc.get(k, 0.0) + st[k] / steps
    out = dict(env=env, **{k: round(v, 3) for k, v in acc.items()})
    if acc["ms_build"]:
        # the bytes the engine counts per pass: 4 or 8 per evaluation, whichever tile ran (padding columns excluded)
        out["bytes_per_eval"] = st["cost_bytes_written"] / st["evals"]
        out["build_GBs"] = round(st["cost_bytes_written"] / 1e9 / acc["ms_build"] * 1e3, 0)
        out["argmin_GBs"] = round(st["cost_bytes_read"] / 1e9 / acc["ms_argmin"] * 1e3, 0)
        if PEAK:
            out["build_frac"] = round(out["build_GBs"] / PEAK, 3)
            out["argmin_frac"] = round(out["argmin_GBs"] / PEAK, 3)
    print(out, flush=True)
    eng.close()


def hbm_ceilings():
    """pure-write and pure-read streams through torch, for context next to the kernels"""
    import torch
    n = (8 << 30) // 8
    x = torch.empty(n, dtype=torch.int64, device="cuda")
    for name, fn, nbytes in (("fill(write)", lambda: x.fill_(7), n * 8), ("sum(read)", lambda: x.sum(), n * 8),
                             ("copy(r+w)", lambda: x[: n // 2].copy_(x[n // 2:]), n * 8)):
        fn(); torch.cuda.synchronize()
        best = 1e9
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1))
        print({"stream": name, "GBs": round(nbytes / best / 1e6, 0)}, flush=True)
    del x
    torch.cuda.empty_cache()


if __name__ == "__main__":
    print({"hbm_peak_GBs": PEAK, "source": PEAK_SOURCE}, flush=True)
    if os.environ.get("TUNE_CEIL"):
        hbm_ceilings()
    for env in ({}, {"PM_TUNE_BUILD": "8"}):   # 8: the int64 tile on the FastRow path
        run(env)
    run({}, mode=abi.PM_MODE_FIRST_FIT | abi.PM_PATH_FUSED)
