# -*- coding: utf-8 -*-
"""Ordering check of a training plan's op list: replay the fork / wait protocol of lfd_train_plan_run with vector clocks and check that
every pair of ops that conflict on a workspace tensor (write vs anything, accumulate vs read) is ordered, and that PACK / ZERO / UNPACK
barriers come after everything before them."""
import lfd._native as nat
from lfd._train import TrainPlan


def check_every_conflict_ordered(ops, what=''):
    """-> number of cross-branch conflicting pairs (each asserted to be ordered)."""
    clock, last, seq, info = [], {}, {}, []
    for i, op in enumerate(ops):
        b = op.get('branch', 0)
        if b in last:
            vc = dict(clock[last[b]])
        else:
            vc = dict(clock[last[0]]) if 0 in last else {}       # fork after the preceding main-stream op
        for w in range(nat.MAX_BRANCHES):
            if (op['wait_mask'] >> w) & 1 and w in last:
                for k, v in clock[last[w]].items():
                    vc[k] = max(vc.get(k, -1), v)
        seq[b] = seq.get(b, -1) + 1
        vc[b] = seq[b]
        clock.append(vc)
        last[b] = i
        roles = TrainPlan._ROLES.get(op['kind'])
        acc = {}
        if roles is not None:
            for j, nm in op.get('off', {}).items():
                if nm is not None:
                    acc.setdefault(nm, set()).add(roles[j])
        info.append((b, seq[b], acc, roles is None))
    by_name = {}
    n_pairs = 0
    for j, (bj, sj, accj, barrier) in enumerate(info):
        if barrier:
            for i in range(j):
                bi, si = info[i][0], info[i][1]
                assert clock[j].get(bi, -1) >= si, (what, 'barrier', i, j)
            continue
        for nm, rj in accj.items():
            for (i, ri) in by_name.get(nm, []):
                bi, si = info[i][0], info[i][1]
                if bi == bj:
                    continue
                conflict = 'W' in ri or 'W' in rj or (('A' in ri) != ('A' in rj)) or (('A' in ri) and ('R' in ri or 'R' in rj))
                if conflict:
                    n_pairs += 1
                    assert clock[j].get(bi, -1) >= si, (what, nm, i, j, ops[i]['kind'], ops[j]['kind'])
            by_name.setdefault(nm, []).append((j, rj))
    return n_pairs
