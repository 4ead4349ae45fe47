"""Committed golden fixtures (tests/golden/*.npz, made by tests/golden/make_golden.py from the CPU
oracle).  CPU: the oracle still reproduces them and the synthetic generator is stable (checksums).
GPU: the CUDA path reproduces them bit for bit without touching the oracle."""
import os

import numpy as np
import pytest

from protocol_b200 import abi

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
import sys

sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

NAMES = sorted(mg.CASES)


def load(name):
    return np.load(os.path.join(HERE, f"{name}.npz"))


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_golden(name):
    from oracle import pm_oracle as orc

    w, a, bits, npat, nmod, words, prox = mg.build(name)
    z = load(name)
    assert int(np.frombuffer(w.a.tobytes(), dtype=np.uint32).sum(dtype=np.uint64)) == int(z["wa_crc"][0]), "generator drifted"
    assert int(np.frombuffer(a.asks.tobytes(), dtype=np.uint32).sum(dtype=np.uint64)) == int(z["asks_crc"][0])
    g = orc.soa_form_groups(w.a, w.b, a.asks, a.opts, bits, words, addr_rank=w.addr_rank, lat=w.lat, lon=w.lon, proximity=prox)
    assert np.array_equal(g.cfg, z["group_ask"]) and np.array_equal(g.off, z["group_off"])
    assert np.array_equal(g.members, z["group_members"])
    ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, bits, words, 0, len(a), 0, len(w), threads=8)
    assert np.array_equal(ev["row_best"], z["ask_best"]) and np.array_equal(ev["row_count"], z["ask_count"])


def test_priced_golden_has_ties_and_negative_costs():
    """first_fit_priced freezes row minima at Zipf prices and at prices of 2^31 and above (negative packed costs)."""
    z = load("first_fit_priced")
    hi = z["ask_best"][z["ask_count"] > 0] >> 32
    assert (hi == -(1 << 31)).any() and (hi == -1).any() and (hi > 0).any() and (hi != 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("path", [abi.PM_PATH_MATERIALIZED, abi.PM_PATH_FUSED], ids=["materialized", "fused"])
@pytest.mark.parametrize("name", NAMES)
def test_cuda_reproduces_golden(name, path):
    from protocol_b200.engine import Engine

    w, a, bits, npat, nmod, words, prox = mg.build(name)
    z = load(name)
    eng = Engine(cost_tile_bytes=4 << 20)
    eng.set_asks(a.asks, a.opts)
    eng.set_model_table(bits, npat, nmod, words)
    eng.set_workers(w.a, w.b)
    eng.set_addr_rank(w.addr_rank)
    eng.set_locations(w.lat, w.lon)
    eng.match((abi.PM_MODE_PROXIMITY if prox else abi.PM_MODE_FIRST_FIT) | path)
    r = eng.fetch()
    assert np.array_equal(r.group_ask, z["group_ask"]) and np.array_equal(r.group_off, z["group_off"])
    assert np.array_equal(r.group_members, z["group_members"])
    assert np.array_equal(r.ask_best, z["ask_best"]) and np.array_equal(r.ask_count, z["ask_count"])
    eng.close()
