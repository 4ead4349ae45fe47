"""The incremental pass across enabled-configuration changes (pm_set_ask_enabled + PM_INCREMENTAL), restated on the CPU.

1. The update rule, on random feasibility matrices F[t, w] over random histories of toggles and row writes.  The
   stored evaluation holds each worker's first feasible ask f under the mask it was taken with; E = asks enabled since,
   D = asks disabled since.  Written rows are reset and walked over every ask; the orphans (f in D) are reset and walked
   from f + 1; the E-pass walks every worker over E in increasing order, stopping once its current value lies below
   the next ask of E.  Each walk merges with a minimum, in any order.  The result must be the first feasible ask under
   the current mask at every step; the rows walked in full are the written rows plus the orphans.
2. The plugin's upload order: pm_sort_configs, then the stable min_group_size re-sort of available_configurations(),
   applied to an enabled subset, gives that subset of the re-sorted full list — so the engine can hold every
   configuration in one order and switch them on and off."""
import numpy as np
import pytest

from protocol_b200.engine import sort_configs

NONE = 0xFFFFFFFF


def first_feasible(F, mask):
    G = F & mask[:, None]
    return np.where(G.any(0), G.argmax(0), NONE).astype(np.uint32)


def incremental(F, stored, eval_mask, mask, written, rng):
    """One incremental pass; returns (new stored evaluation, rows walked in full, pair evaluations)."""
    T, W = F.shape
    E = np.nonzero(mask & ~eval_mask)[0]
    D = np.nonzero(~mask & eval_mask)[0]
    buf = stored.copy()
    wmask = np.zeros(W, bool)
    wmask[list(written)] = True
    orphans = np.isin(stored, D) & ~wmask
    buf[wmask | orphans] = NONE                  # the resets come first
    evals = 0

    def walks():
        nonlocal evals
        for w in np.nonzero(wmask | orphans)[0]:
            start = 0 if wmask[w] else int(stored[w]) + 1
            hit = np.nonzero(F[start:, w] & mask[start:])[0]
            evals += (hit[0] + 1) if len(hit) else T - start
            if len(hit):
                buf[w] = min(buf[w], start + hit[0])

    def e_pass():
        nonlocal evals
        for w in range(W):
            for t in E:
                if buf[w] < t:                   # nothing of E from here on can lower it
                    break
                evals += 1
                if F[t, w]:
                    buf[w] = min(buf[w], t)
                    break

    for part in ((walks, e_pass) if rng.random() < 0.5 else (e_pass, walks)):
        part()
    return buf, int(wmask.sum() + orphans.sum()), evals


@pytest.mark.parametrize("seed", range(6))
def test_update_rule_equals_first_feasible_under_the_mask(seed):
    rng = np.random.default_rng(seed)
    T, W = int(rng.integers(5, 40)), int(rng.integers(20, 200))
    F = rng.random((T, W)) < rng.uniform(0.05, 0.4)
    mask = rng.random(T) < 0.7
    stored, eval_mask = first_feasible(F, mask), mask.copy()
    kinds = set()
    for step in range(60):
        op = ["toggle", "off_on", "disable_top", "enable0", "rows", "rows_toggle", "none"][step % 7]
        written = set()
        if op in ("toggle", "rows_toggle"):
            idx = rng.choice(T, int(rng.integers(1, max(2, T // 4))), replace=False)
            mask[idx] = rng.random(len(idx)) < 0.5
        elif op == "off_on":              # off and on again between two passes: neither in E nor in D
            j = int(rng.integers(0, T))
            was = mask[j]
            mask[j] = not was
            mask[j] = was
        elif op == "disable_top":         # the first ask of many workers
            owners = np.bincount(stored[stored != NONE], minlength=T)
            mask[int(np.argmax(owners))] = False
        elif op == "enable0":
            mask[0] = True
        if op in ("rows", "rows_toggle"):
            cols = np.unique(rng.integers(0, W, int(rng.integers(1, 10))))
            F[:, cols] = rng.random((T, len(cols))) < 0.2
            written = set(cols.tolist())
        n_en = int((mask & ~eval_mask).sum())
        stored, walked, evals = incremental(F, stored, eval_mask, mask, written, rng)
        eval_mask = mask.copy()
        assert np.array_equal(stored, first_feasible(F, mask)), f"step {step} ({op})"
        if op in ("none", "off_on"):
            assert walked == 0 and evals == 0
        assert evals <= T * walked + n_en * W
        kinds.add(op)
    assert len(kinds) == 7


def test_disabling_the_only_feasible_ask_and_enabling_ask0():
    T, W = 6, 50
    F = np.zeros((T, W), bool)
    F[3] = True                           # ask 3 takes everyone
    F[0, ::2] = True
    mask = np.array([False, True, True, True, True, True])
    stored = first_feasible(F, mask)
    assert (stored == 3).all()
    rng = np.random.default_rng(1)
    mask2 = mask.copy()
    mask2[3] = False                      # every worker is an orphan, and nothing after 3 accepts anyone
    s2, walked, _ = incremental(F, stored, mask, mask2, set(), rng)
    assert walked == W and (s2 == NONE).all()
    mask3 = mask2.copy()
    mask3[0] = True                       # ask 0 ahead of every (former) owner
    s3, walked, evals = incremental(F, s2, mask2, mask3, set(), rng)
    assert walked == 0 and evals == W and np.array_equal(s3, first_feasible(F, mask3))


@pytest.mark.parametrize("seed", range(8))
def test_enabled_subset_keeps_the_order_of_the_full_list(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 300))
    mn = rng.integers(0, 5, n).astype(np.uint32)
    hr = (rng.random(n) < 0.6).astype(np.uint8)
    sealed = sort_configs(mn, hr)                               # pm_plugin_seal_configs

    def resort(idx):                                            # available_configurations: stable, min desc
        return sorted(idx, key=lambda i: -int(mn[i]))

    full = resort(list(sealed))
    for _ in range(20):
        on = set(np.nonzero(rng.random(n) < rng.uniform(0, 1))[0].tolist())
        assert resort([i for i in sealed if i in on]) == [i for i in full if i in on]
