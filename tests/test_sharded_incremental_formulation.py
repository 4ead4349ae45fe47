"""The incremental pass on sharded engines (PM_INCREMENTAL on pm_match_local, pm_comm ranks and pm_multi), restated on
the CPU.

N ranks each hold the whole (replicated) tables and evaluate the equal share [r * ceil(W / N), ...) of the workers.
Each keeps the stored evaluation of its own range: the first feasible ask under the mask it was taken with, NONE
outside the range.  Between passes rows are written, W grows and shrinks (so every share's boundaries move), and asks
are toggled.  A rank's pass is full or incremental by its own count: its in-range written rows plus |E| nw / T against
the cutoff.  An incremental pass resets and walks the range's written rows, walks the range's orphans (stored first ask
in D) from the ask after it, and runs the E-pass over the range's workers.  Rows that enter a range on a resize count
as written there; rows that leave it return to NONE.

After every step the concatenated ranges must equal the unsharded first feasible ask, each rank's walk list must be
exactly its in-range written rows (entered rows included) plus its orphans, and nothing outside a range may be set —
whether the ranks agree on full vs incremental or not."""
import numpy as np
import pytest

NONE = 0xFFFFFFFF


def first_feasible(F, mask):
    G = F & mask[:, None]
    return np.where(G.any(0), G.argmax(0), NONE).astype(np.uint32)


def share(W, N, r):
    per = -(-W // N)
    lo = min(r * per, W)
    return lo, min(lo + per, W)


class Rank:
    def __init__(self, N, r, cutoff):
        self.N, self.r, self.cutoff = N, r, cutoff
        self.stored = None          # None: no stored evaluation
        self.eval_mask = None
        self.written = set()        # every written row (the preludes'); the walk takes those in range

    def range(self, W):
        return share(W, self.N, self.r)

    def resize(self, W_old, W_new):
        if self.stored is None:
            return
        a0, a1 = self.range(W_old)
        b0, b1 = self.range(W_new)
        st = np.full(W_new, NONE, np.uint32)
        k = min(W_old, W_new)
        st[:k] = self.stored[:k]
        self.written = {i for i in self.written if i < W_new}
        for i in range(a0, min(a1, W_new)):            # left the range
            if not b0 <= i < b1:
                st[i] = NONE
        for i in range(b0, b1):                        # entered it
            if not a0 <= i < a1:
                self.written.add(i)
        self.written |= set(range(W_old, W_new))       # past the old end: written for the preludes, wherever they lie
        self.stored = st

    def pass_(self, F, mask):
        """Returns (stored range, rows walked in full, pairs evaluated, full?)."""
        T, W = F.shape
        lo, hi = self.range(W)
        nw = hi - lo
        inr = sorted(i for i in self.written if lo <= i < hi)
        if self.stored is not None:
            E = np.nonzero(mask & ~self.eval_mask)[0]
            D = np.nonzero(~mask & self.eval_mask)[0]
        use_incr = self.stored is not None and T and nw and len(inr) + -(-len(E) * nw // T) <= self.cutoff
        if not use_incr:
            st = np.full(W, NONE, np.uint32)
            st[lo:hi] = first_feasible(F[:, lo:hi], mask)
            walked, evals = list(range(lo, hi)), T * nw
        else:
            st = self.stored.copy()
            wmask = np.zeros(W, bool)
            wmask[inr] = True
            rng_mask = np.zeros(W, bool)
            rng_mask[lo:hi] = True
            orphans = np.isin(self.stored, D) & ~wmask & rng_mask
            st[wmask | orphans] = NONE
            evals = 0
            for w in np.nonzero(wmask | orphans)[0]:
                start = 0 if wmask[w] else int(self.stored[w]) + 1
                hit = np.nonzero(F[start:, w] & mask[start:])[0]
                evals += (hit[0] + 1) if len(hit) else T - start
                if len(hit):
                    st[w] = min(st[w], start + hit[0])
            for w in range(lo, hi):                    # the E-pass over the range's workers
                for t in E:
                    if st[w] < t:
                        break
                    evals += 1
                    if F[t, w]:
                        st[w] = min(st[w], t)
                        break
            walked = sorted(np.nonzero(wmask | orphans)[0].tolist())
            assert set(walked) == set(inr) | set(np.nonzero(orphans)[0].tolist())
        self.stored, self.eval_mask, self.written = st, mask.copy(), set()
        return st, walked, evals, not use_incr


def run_history(N, seed, cutoffs=None, steps=50):
    rng = np.random.default_rng(seed)
    T, W = int(rng.integers(5, 30)), int(rng.integers(N, 12 * N + 20))
    F = rng.random((T, W)) < rng.uniform(0.05, 0.4)
    mask = rng.random(T) < 0.7
    ranks = [Rank(N, r, (cutoffs or [10**9] * N)[r]) for r in range(N)]
    kinds, splits = set(), 0
    for step in range(steps):
        op = ["rows", "grow", "shrink", "toggle", "disable_top", "none", "rows_toggle", "one_range"][step % 8]
        entered = [set() for _ in ranks]
        W_old = W
        if op in ("rows", "rows_toggle"):
            cols = np.unique(rng.integers(0, W, int(rng.integers(1, 8))))
            F[:, cols] = rng.random((T, len(cols))) < 0.2
            for rk in ranks:
                rk.written |= set(cols.tolist())
        elif op == "one_range":           # writes into one rank's range only
            lo, hi = share(W, N, int(rng.integers(0, N)))
            if hi > lo:
                cols = np.unique(rng.integers(lo, hi, int(rng.integers(1, hi - lo + 1))))
                F[:, cols] = rng.random((T, len(cols))) < 0.2
                for rk in ranks:
                    rk.written |= set(cols.tolist())
        elif op == "grow":
            W = W + int(rng.integers(1, N + 2))
            F = np.concatenate([F, rng.random((T, W - W_old)) < 0.2], axis=1)
        elif op == "shrink":
            W = max(1, W - int(rng.integers(1, N + 2)))
            F = F[:, :W]
        if op in ("grow", "shrink"):
            for r, rk in enumerate(ranks):
                a0, a1 = share(W_old, N, r)
                b0, b1 = share(W, N, r)
                entered[r] = {i for i in range(b0, b1) if not a0 <= i < a1}
                rk.resize(W_old, W)
        if op in ("toggle", "rows_toggle"):
            idx = rng.choice(T, int(rng.integers(1, max(2, T // 4))), replace=False)
            mask[idx] = rng.random(len(idx)) < 0.5
        elif op == "disable_top" and ranks[0].stored is not None:
            whole = first_feasible(F, mask)
            owners = np.bincount(whole[whole != NONE], minlength=T)
            mask[int(np.argmax(owners))] = False
        expect = first_feasible(F, mask)
        before = [None if rk.stored is None else rk.stored.copy() for rk in ranks]
        written_in = [{i for i in rk.written if share(W, N, r)[0] <= i < share(W, N, r)[1]} for r, rk in enumerate(ranks)]
        eval_masks = [None if rk.eval_mask is None else rk.eval_mask.copy() for rk in ranks]
        got = np.full(W, NONE, np.uint32)
        fulls = []
        for r, rk in enumerate(ranks):
            lo, hi = share(W, N, r)
            st, walked, evals, full = rk.pass_(F, mask)
            fulls.append(full)
            assert (st[:lo] == NONE).all() and (st[hi:] == NONE).all(), f"step {step}: rank {r} set outside its range"
            got[lo:hi] = st[lo:hi]
            if not full:
                D = np.nonzero(~mask & eval_masks[r])[0]
                orphans = {w for w in range(lo, hi) if before[r][w] in set(D.tolist()) and w not in written_in[r]}
                assert set(walked) == written_in[r] | orphans, f"step {step}: rank {r} walk list"
                assert entered[r] <= set(walked), f"step {step}: rank {r} did not walk the rows that entered its range"
                if op == "none":
                    assert walked == [] and evals == 0
        assert np.array_equal(got, expect), f"step {step} ({op})"
        splits += len(set(fulls)) > 1
        kinds.add(op)
    assert len(kinds) == 8
    return splits


@pytest.mark.parametrize("N", [2, 3, 5, 8])
@pytest.mark.parametrize("seed", range(3))
def test_ranges_concatenate_to_the_unsharded_first_feasible_ask(N, seed):
    run_history(N, 100 * N + seed)


@pytest.mark.parametrize("N", [2, 3, 5, 8])
def test_ranks_that_disagree_on_full_vs_incremental(N):
    """Small, uneven cutoffs: in many passes some ranks evaluate their range in full and others walk a few rows."""
    rng = np.random.default_rng(N)
    splits = sum(run_history(N, 7 * N + s, cutoffs=rng.integers(0, 4, N).tolist()) for s in range(3))
    assert splits > 0
