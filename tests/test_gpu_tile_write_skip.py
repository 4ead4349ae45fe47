"""pm_build_argmin_feat's skipped stores on hardware: the cost tile the materialised pass leaves (PM_BUF_COST_TILE) must
hold every word the pass computed, although the kernel does not store a warp's 512-byte block when it is all
infeasible and the buffer already holds the sentinel there (TileBuf::held).

One engine goes through a history of passes and table calls.  After each pass the buffer is read back and held
against a simulated one: each tile of the pass writes its rows' 32-bit cost words (Engine.cost_tile's int64 rows,
high word, in the column order) at slot * ld; the padding columns hold kNarrowInfeasible.  Words written otherwise —
by the int64 tile of a price at 0x7FFFFFFF, or by Engine.cost_tile's export — and a reallocated buffer are unknown
to the simulation until a pass writes them again, so a block the kernel skipped over them would show up.  Every
pass's outputs are also held against a PM_TUNE_BUILD=8 twin that runs the same history on the int64 tile."""
import numpy as np
import pytest
import torch

from helpers import load_engine
from protocol_b200 import abi
from protocol_b200.sharded import _DevArray, wrap_device_buffers
from test_ask_deltas_formulation import own_options
from test_column_order_formulation import column_order, features
from test_gpu_narrow_tile import MAT, RESULT_FIELDS, assert_same, make_engine, tables
from test_gpu_tile_overlap import tile_bytes

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FFFFFFF


class SimBuffer:
    """The cost buffer as 32-bit words, with the words whose contents the simulation knows.  The buffer only grows
    (TileBuf::ensure): a request past its capacity reallocates it, and nothing in it is known then."""

    def __init__(self):
        self.words = np.zeros(0, dtype=np.uint32)
        self.known = np.zeros(0, dtype=bool)

    def need(self, nbytes):
        if nbytes > len(self.words) * 4:
            self.words = np.zeros(nbytes // 4, dtype=np.uint32)
            self.known = np.zeros(nbytes // 4, dtype=bool)

    def forget(self, nbytes):
        self.known[:nbytes // 4] = False

    def write_pass(self, tile32, rows):
        """tile32 [T, ld]: the pass's rows; each tile's row i goes to slot i."""
        for t0 in range(0, len(tile32), rows):
            part = tile32[t0:t0 + rows].reshape(-1)
            self.words[:part.size] = part
            self.known[:part.size] = True


def expected_tile(x, t, w0, nw):
    """[T, ld] uint32: the 32-bit tile of a pass over workers [w0, w0 + nw), in the column order, from x's export."""
    ld = -(-nw // 1024) * 1024
    F, n, _ = features(t, w0, nw)
    perm = column_order(F, n, ld)
    hi = (x.cost_tile(0, len(t["asks"]), nw) >> 32).astype(np.uint32)   # worker order
    out = np.full((len(t["asks"]), ld), SENTINEL, dtype=np.uint32)
    out[:, :nw] = hi[:, perm[:nw]]
    return out


def read_buffer(e):
    p, nbytes = e.device_buffer(abi.PM_BUF_COST_TILE)
    return torch.as_tensor(_DevArray(p, nbytes // 4, "<i4"), device="cuda").cpu().numpy().view(np.uint32).copy()


class History:
    """One engine and its PM_TUNE_BUILD=8 twin through the same calls; the twin's exports give the expected tiles."""

    def __init__(self, t, cost_tile_bytes):
        self.t = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in t.items()}
        self.e = make_engine(False, cost_tile_bytes=cost_tile_bytes)
        self.twin = make_engine(True, cost_tile_bytes=cost_tile_bytes)
        for x in (self.e, self.twin):
            load_engine(x, self.t)
        self.sim = SimBuffer()
        self.shard = None
        self.n_checked = 0

    def close(self):
        self.e.close()
        self.twin.close()

    def both(self, fn):
        fn(self.e)
        fn(self.twin)

    def range(self):
        w0, nw = self.shard if self.shard is not None else (0, len(self.t["wa"]))
        return w0, nw, -(-nw // 1024) * 1024

    def outputs(self, x):
        W, T = len(self.t["wa"]), len(self.t["asks"])
        x.match_local(MAT)
        x.sync()
        arr = [a.cpu().numpy().copy() for a in wrap_device_buffers(x, W, T)]
        res = None
        if self.shard is None:
            x.match_finish(MAT)
            res = x.fetch()
        return arr, res

    def run_pass(self, narrow=True):
        got, res = self.outputs(self.e)
        want, res_w = self.outputs(self.twin)
        for a, b, name in zip(got, want, ("first_ask", "ask_best", "ask_count")):
            assert np.array_equal(a, b), f"{name} differs from the int64 tile's"
        if res is not None:
            for f in RESULT_FIELDS:
                assert np.array_equal(getattr(res, f), getattr(res_w, f)), f"{f} differs"
        w0, nw, ld = self.range()
        T = len(self.t["asks"])
        assert self.e.stats()["cost_bytes_written"] == (4 if narrow else 8) * T * nw, "not the expected tile width"
        nbytes = self.e.device_buffer(abi.PM_BUF_COST_TILE)[1]
        self.sim.need(nbytes)
        if not narrow:
            self.sim.forget(nbytes)
            return
        rows = nbytes // (ld * 4)
        buf = read_buffer(self.e)
        self.sim.write_pass(expected_tile(self.twin, self.t, w0, nw), rows)
        k = self.sim.known[:len(buf)]
        assert k[:min(rows, T) * ld].all()   # every slot this pass wrote
        bad = np.flatnonzero((buf != self.sim.words[:len(buf)]) & k)
        assert bad.size == 0, (f"{bad.size} stale words, first at slot {bad[0] // ld} column {bad[0] % ld}: "
                               f"{buf[bad[0]]:#x} != {self.sim.words[bad[0]]:#x}")
        self.n_checked += 1

    def export(self):
        """Engine.cost_tile on the engine itself: int64 rows over the start of its buffer."""
        w0, nw, ld = self.range()
        nbytes = len(self.t["asks"]) * ld * 8
        self.sim.need(nbytes)
        self.e.cost_tile(0, len(self.t["asks"]), nw)
        self.sim.forget(nbytes)


def test_the_tile_stays_exact_through_a_history():
    t = tables(900, 5000, 41)
    W, T = len(t["wa"]), len(t["asks"])
    h = History(t, tile_bytes(W, 256))   # tiles of 256 rows: 256, 256, 256, 132
    rng = np.random.default_rng(7)
    try:
        for _ in range(3):   # the first pass writes every block, the next ones skip
            h.run_pass()
        blocks = (expected_tile(h.twin, h.t, 0, W) == SENTINEL).reshape(T, -1, 128).all(axis=2)
        assert blocks.mean() > 0.5, "few all-infeasible blocks: nothing to skip"
        # the export overwrites the buffer with int64 rows: the next pass must write every block again
        h.export()
        h.run_pass()
        h.run_pass()
        # workers rewritten with other workers' contents and new prices: the column order changes
        src = rng.permutation(W)[:1500]
        na, nb = h.t["wa"][src].copy(), h.t["wb"][src].copy()
        nb["ext_ask_price"] = rng.integers(1, 1 << 20, len(src))
        h.both(lambda x: x.upsert_workers(na, nb, 700))
        h.t["wa"][700:2200], h.t["wb"][700:2200] = na, nb
        h.run_pass()
        # asks replaced by other rows of the table
        idx = rng.integers(0, T, 40).astype(np.uint32)
        rows = h.t["asks"][rng.integers(0, T, 40)].copy()
        sent = own_options(rows, h.t["opts"])
        h.both(lambda x: x.update_asks(idx, *sent))
        for i, r in zip(idx, rows):
            h.t["asks"][i] = r
        h.run_pass()
        # fewer asks than one tile's rows: the rows per tile change (256 -> 100)
        h.both(lambda x: x.resize_asks(100))
        h.t["asks"] = h.t["asks"][:100].copy()
        h.run_pass()
        h.run_pass()
        # a shard: ld changes (5120 -> 3072) and w0 moves off a stripe boundary; then the whole range again
        h.shard = (1234, 2500)
        h.both(lambda x: x.set_shard(*h.shard))
        h.run_pass()
        h.run_pass()
        h.shard = None
        h.both(lambda x: x.set_shard(0, 0))
        h.run_pass()
        # a price of 0x7FFFFFFF: the int64 tile, then back to the 32-bit one
        old = h.t["wb"][17:18].copy()
        top = old.copy()
        top["ext_ask_price"] = 0x7FFFFFFF
        a17 = h.t["wa"][17:18].copy()
        h.both(lambda x: x.upsert_workers(a17, top, 17))
        h.t["wb"][17] = top[0]
        h.run_pass(narrow=False)
        h.both(lambda x: x.upsert_workers(a17, old, 17))
        h.t["wb"][17] = old[0]
        h.run_pass()
        h.run_pass()
        assert h.n_checked == 14
    finally:
        h.close()
    assert_same(h.t, tile_bytes(W, 256))
