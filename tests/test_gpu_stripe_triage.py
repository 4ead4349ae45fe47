"""pm_build_argmin_feat's row triage on hardware: a CTA skips the rows whose every block is dead by its stripe's OR of
feature words and already holds the sentinel (SKIP), stores only the missing sentinel blocks of the other dead rows
(SENTINEL), and runs the block classes on the rest (LIVE) (test_stripe_triage_formulation.py).

One engine and its PM_TUNE_BUILD=8 twin go through passes and table calls (test_gpu_block_class.Checked).  After every
materialised pass every output equals the twin's and the CPU oracle's, and the cost buffer read back through
PM_BUF_COST_TILE equals the expected tile.  The history reaches every row kind in one launch
(test_stripe_triage_formulation.test_the_gpu_history_reaches_every_row_kind): SENTINEL rows with partly
set map bytes (the slots' asks alternate between stripe-dead and LIVE rows from pass to pass), multi-option
stripe-dead rows, disabled asks, a padded last stripe, a ragged last CTA of rows, and a shard with w0 off a stripe
boundary."""
import numpy as np
import pytest

from test_ask_deltas_formulation import own_options
from test_block_class_formulation import cfg3_like, with_disabled
from test_gpu_block_class import Checked
from test_gpu_feature_predicate import FEAT, kernel_of
from test_gpu_tile_overlap import tile_bytes
from test_stripe_triage_formulation import TPass, multi

pytestmark = pytest.mark.gpu


def test_row_kinds_through_a_history():
    t = cfg3_like(1300, 20077, 67)   # 1300 rows: tiles of 512, 512, 276 (a ragged last CTA of rows)
    W = len(t["wa"])
    assert kernel_of(t) == {FEAT}
    p = TPass(t, 0, W)
    assert p.sd.any() and (~p.sd).any() and p.sd[multi(p)].any()
    assert p.ld > p.nw                      # a padded last stripe
    h = Checked(t, tile_bytes(W, 512))
    try:
        for _ in range(2):                  # the first pass finds the map zeroed, the second SKIPs
            h.run_pass()
        # the asks reversed: each slot now holds another ask, so dead rows meet bytes a LIVE row left partly set
        rev = np.arange(len(t["asks"]))[::-1].astype(np.uint32)
        rows = h.t["asks"][rev].copy()
        sent = own_options(rows, h.t["opts"])
        idx = np.arange(len(rows), dtype=np.uint32)
        h.both(lambda x: x.update_asks(idx, *sent))
        h.t["asks"] = rows
        h.run_pass()
        h.run_pass()
        # disabled asks: stripe-dead in every CTA
        on = with_disabled(h.t)
        off = np.flatnonzero(~on).astype(np.uint32)
        h.both(lambda x: x.set_ask_enabled(off, False))
        h.enabled = False
        h.run_pass()
        h.both(lambda x: x.set_ask_enabled(off, True))
        h.enabled = True
        h.run_pass()
        # a shard with w0 off a stripe boundary, then the whole range again
        h.shard = (9001, 8000)
        h.both(lambda x: x.set_shard(*h.shard))
        h.run_pass()
        h.run_pass()
        h.shard = None
        h.both(lambda x: x.set_shard(0, 0))
        h.run_pass()
        assert h.n_checked == 9
    finally:
        h.close()

