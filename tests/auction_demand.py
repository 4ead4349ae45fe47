"""Ask demands (pm_set_ask_demand, prime_match.h "Auction demands") restated in numpy: the slot offsets, the remap of a
stored slot assignment under a demand change, the per-ask certificate over slots, and the fold of a slot assignment to
the grouped result.  Shared by the demand tests and the engine histories (tests/engine_history.py).

An engine with demands d behaves as its twin, whose ask table repeats row t d[t] times: slot s of ask t is
offsets(d)[t] + k, k < d[t].
"""
from __future__ import annotations

import numpy as np

import auction_warm_checker as wc

NONE = wc.NONE
INF = 0x7FFFFFFFFFFFFFFF   # PM_COST_INF: ask_best of an ask that holds nothing


def offsets(d):
    return np.concatenate([[0], np.cumsum(np.asarray(d, dtype=np.int64))]).astype(np.int64)


def remap(a_slots, d_old, d_new, n_kept=None):
    """pm_set_ask_demand under a stored state: old slot k of ask t stays slot k while k < the new demand; the added
    slots hold nothing.  Returns (new slot assignment, added slots, freed), freed = the workers of removed slots below
    n_kept (every held one when n_kept is None): those count against the warm cutoff."""
    o_old, o_new = offsets(d_old), offsets(d_new)
    out = np.full(int(o_new[-1]), NONE, dtype=np.uint32)
    added, freed = [], 0
    limit = NONE if n_kept is None else int(n_kept)
    for t in range(len(d_old)):
        k = min(int(d_old[t]), int(d_new[t]))
        out[o_new[t]:o_new[t] + k] = a_slots[o_old[t]:o_old[t] + k]
        gone = np.asarray(a_slots[o_old[t] + k:o_old[t + 1]])
        freed += int(np.sum((gone != NONE) & (gone < limit)))
        added.extend(range(int(o_new[t]) + k, int(o_new[t + 1])))
    return out, np.array(added, dtype=np.int64), freed


def demand_certificate(F, ask_price, cap, d, S, price, a_slots):
    """The certificate as the device computes it with demands: the row terms per ask (T x W), weighted by d; holds,
    costs, slacks and ownership per slot."""
    T, W = F.shape
    S = int(S)
    ap = [int(x) for x in np.asarray(ask_price)[:W]]
    pr = [int(x) for x in np.asarray(price)[:W]]
    key = np.array([ap[w] * S + pr[w] for w in range(W)], dtype=np.int64)
    big = np.iinfo(np.int64).max
    rowmin = np.where(F, key[None, :], big).min(axis=1) if W else np.full(T, big, dtype=np.int64)
    row = [min((int(cap[t]) + 1) * S, int(rowmin[t])) for t in range(T)]
    off = offsets(d)
    own = [0] * W
    cost = n_held = n_bad = 0
    slack = []
    for t in range(T):
        for s in range(off[t], off[t + 1]):
            w = int(a_slots[s])
            if w != NONE and w < W:
                n_held += 1
                own[w] += 1
                n_bad += int(not F[t, w])
                cost += ap[w] * S
                slack.append(int(key[w]) - row[t])
            else:
                cost += (int(cap[t]) + 1) * S
                slack.append((int(cap[t]) + 1) * S - row[t])
    bound = sum(int(d[t]) * row[t] for t in range(T)) - sum(pr)
    free = [w for w in range(W) if own[w] == 0 and pr[w] > 0]
    return dict(cost=cost, bound=bound, gap=cost - bound, n_held=n_held, n_bad_holds=n_bad,
                n_shared=sum(1 for o in own if o > 1), n_priced_unowned=len(free),
                priced_unowned_sum=sum(pr[w] for w in free), n_slack_over=sum(1 for s in slack if s > 1),
                max_slack=max(slack) if T else 0, evals=T * W, ask_bound=np.array(row, dtype=np.int64))


def fold_like_device(a_slots, d, ask_price):
    """Held flags per slot and their exclusive scan, counts per ask, groups by the scan of the ask flags, members
    gathered in slot order and sorted per group.  Returns (group_ask, group_off, members, count, best); best is int64
    max for an ask that holds nothing."""
    off = offsets(d)
    a_slots = np.asarray(a_slots)
    held = (a_slots != NONE).astype(np.int64)
    spos = np.concatenate([[0], np.cumsum(held)])
    count = spos[off[1:]] - spos[off[:-1]]
    gidx = np.concatenate([[0], np.cumsum(count > 0)])
    G, M = int(gidx[-1]), int(spos[-1])
    group_ask = np.zeros(G, dtype=np.int64)
    group_off = np.zeros(G + 1, dtype=np.int64)
    members = np.zeros(M, dtype=np.int64)
    best = np.full(len(d), np.iinfo(np.int64).max, dtype=np.int64)
    for t in np.flatnonzero(count):
        g = gidx[t]
        group_ask[g], group_off[g] = t, spos[off[t]]
        ws = a_slots[off[t]:off[t + 1]]
        ws = ws[ws != NONE].astype(np.int64)
        members[spos[off[t]]:spos[off[t]] + len(ws)] = ws
        best[t] = min((int(ask_price[w]) << 32) | int(w) for w in ws)
    group_off[G] = M
    for g in range(G):
        members[group_off[g]:group_off[g + 1]] = np.sort(members[group_off[g]:group_off[g + 1]])
    return group_ask, group_off, members, count, best


def result_arrays(a_slots, d, ask_price, n_workers):
    """Every array pm_fetch_result returns for an auction pass whose slot assignment is a_slots: one group per ask
    holding a worker, in ask order, its members sorted; worker_ask / worker_group per worker; ask_count and ask_best
    (PM_COST_INF for an ask that holds nothing)."""
    group_ask, group_off, members, count, best = fold_like_device(a_slots, d, ask_price)
    wg = np.full(n_workers, NONE, dtype=np.uint32)
    wk = np.full(n_workers, NONE, dtype=np.uint32)
    for g in range(len(group_ask)):
        m = members[group_off[g]:group_off[g + 1]]
        wg[m], wk[m] = g, group_ask[g]
    return dict(worker_group=wg, worker_ask=wk, group_ask=group_ask.astype(np.uint32),
                group_off=group_off.astype(np.uint32), group_members=members.astype(np.uint32),
                ask_best=np.where(count > 0, best, INF).astype(np.int64), ask_count=count.astype(np.uint32))
