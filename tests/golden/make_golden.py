"""Generates tests/golden/*.npz: expected results of the matching pass on small seeded swarms,
computed by the CPU oracle (oracle/pm_oracle.cpp — itself pinned to the reference's known-answer
tests).  The reference is Rust and cannot run here, so these are oracle outputs, not reference
outputs; they make the -m gpu suite independent of the oracle build on the GPU box and freeze the
expected answers in the repository.  Re-run:  python tests/golden/make_golden.py [name ...]
(no names: every case)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pm_oracle as orc  # noqa: E402
from protocol_b200 import abi, synth  # noqa: E402

CASES = {
    # name: (n_asks, n_workers, kind, group_sizes, proximity, seed_shift, prices)
    "first_fit_solo": (300, 4000, "mixed", None, False, 0, None),
    "first_fit_sizes": (200, 5000, "mixed", [(1, 1), (2, 2), (2, 4), (3, 3), (4, 8)], False, 1, None),
    "proximity_sizes": (100, 2500, "mixed", [(2, 2), (2, 4), (3, 3)], True, 2, None),
    "skewed_infeasible": (400, 3000, "skewed", None, False, 3, None),
    "first_fit_priced": (300, 3000, "mixed", None, False, 4, "zipf_edges"),
}
# "zipf_edges": Zipf prices (many ties), and every 400th candidate worker priced at one of these: at 2^31 and above
# the packed cost (price << 32 | worker) is negative, so those workers are the best of every ask they meet
EDGE_PRICES = [0x80000000, 0xFFFFFFFF, 0x7FFFFFFE, 0x80000001]


def build(name):
    T, W, kind, sizes, prox, shift, prices = CASES[name]
    w = synth.make_workers(W, seed=synth.SEED_WORKERS + shift, with_addresses=True,
                           price="zipf" if prices == "zipf_edges" else prices)
    if prices == "zipf_edges":
        cand = abi.PM_W_HEALTHY | abi.PM_W_P2P
        pick = np.flatnonzero((w.a["flags"] & (cand | abi.PM_W_ASSIGNED)) == cand)[::400]
        w.b["ext_ask_price"][pick] = np.resize(np.array(EDGE_PRICES, dtype=np.uint32), len(pick))
    a = synth.make_asks(T, kind, seed=synth.SEED_ASKS + shift, group_sizes=sizes)
    bits, npat, nmod, words = synth.intern_tables(w, a)
    return w, a, bits, npat, nmod, words, prox


if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    for name in sys.argv[1:] or CASES:
        w, a, bits, npat, nmod, words, prox = build(name)
        g = orc.soa_form_groups(w.a, w.b, a.asks, a.opts, bits, words, addr_rank=w.addr_rank, lat=w.lat, lon=w.lon,
                                proximity=prox)
        ev = orc.soa_eval_matrix(w.a, w.b, a.asks, a.opts, bits, words, 0, len(a), 0, len(w), threads=8)
        np.savez_compressed(os.path.join(here, f"{name}.npz"), group_ask=g.cfg, group_off=g.off, group_members=g.members,
                            ask_best=ev["row_best"], ask_count=ev["row_count"], col_first=ev["col_first"],
                            wa_crc=np.array([int(np.frombuffer(w.a.tobytes(), dtype=np.uint32).sum(dtype=np.uint64))]),
                            asks_crc=np.array([int(np.frombuffer(a.asks.tobytes(), dtype=np.uint32).sum(dtype=np.uint64))]))
        print(name, len(g), "groups")
