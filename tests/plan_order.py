# -*- coding: utf-8 -*-
"""Byte-level ordering check of a plan's op list, for inference plans (lfd_plan) and training plans (lfd_train_plan) alike.

The executor (csrc/api.cu, BranchExecutor::enqueue) clears the statistics region on the caller's stream, then enqueues op after op: a
side branch forks after every main-stream op enqueued so far, wait_mask bit w makes an op wait for everything enqueued so far on branch w
(skipped when w is the op's own branch or a side branch that has not started), and every branch joins at the end.  Those rules give every
op a vector clock, hence a happens-before order.  Every op touches byte ranges of the workspace -- read (R), written (W) or accumulated
with atomics (A) -- taken from the records the kernels read, not from the planner's bookkeeping.  Then:
  1. every range lies inside the workspace and starts 256-byte aligned;
  2. two ops on different branches whose ranges overlap, where one writes or one accumulates against a read, are ordered;
  3. liveness: for every read by op r of bytes that op p produced, every other op w that writes overlapping bytes happens before p or
     after r (ops of one branch are ordered by list order).
Inference plans add the GroupNorm statistics slots (disjoint, inside the cleared region, read from the conv that produced the normalised
tensor) and the head's point ranges (each output's levels partition [0, P) as level_geometry lays them out)."""
import lfd._native as nat
from lfd._engine import conv_out, level_geometry
from lfd._train import TrainPlan

ALIGN = 256


class Ops(object):
    """Happens-before of an op list under the executor's fork / wait / join rules."""

    def __init__(self, schedule):
        """schedule: [(branch, wait_mask)] per op."""
        self.branch, self.seq, self.clock = [], [], []
        last, seq = {}, {}
        for i, (b, mask) in enumerate(schedule):
            if b in last:
                vc = dict(self.clock[last[b]])
            else:
                vc = dict(self.clock[last[0]]) if 0 in last else {}      # fork after the main-stream ops enqueued so far
            for w in range(nat.MAX_BRANCHES):
                if (mask >> w) & 1 and w != b and w in last:             # a branch that has not started has nothing to wait for
                    for k, v in self.clock[last[w]].items():
                        vc[k] = max(vc.get(k, -1), v)
            seq[b] = seq.get(b, -1) + 1
            vc[b] = seq[b]
            self.branch.append(b)
            self.seq.append(seq[b])
            self.clock.append(vc)
            last[b] = i

    def before(self, a, b):
        """Op a happens before op b."""
        return a is not None and b is not None and a < b and self.clock[b].get(self.branch[a], -1) >= self.seq[a]


def _check(what, order, acc, reads, ws_bytes, barriers=()):
    """acc[i]: [(lo, hi, role)] of op i; reads: [(r, lo, hi, p, residual)] -- op r reads bytes op p produced (p None: produced before the
    list); residual: r may write its output over them in place (an element-wise read-modify-write).
    -> number of cross-branch overlapping conflicting pairs (each asserted to be ordered)."""
    flat = []
    for i, ranges in enumerate(acc):
        for lo, hi, role in ranges:
            assert 0 <= lo < hi <= ws_bytes, (what, 'op %d: bytes [%d, %d) outside the workspace of %d' % (i, lo, hi, ws_bytes))
            assert lo % ALIGN == 0, (what, 'op %d: a region at byte %d is not %d-byte aligned' % (i, lo, ALIGN))
            flat.append((lo, hi, role, i))
    for j in barriers:           # PACK / ZERO / UNPACK: everything before them precedes them
        for i in range(j):
            assert order.before(i, j), (what, 'barrier', i, j)
    flat.sort()
    n_pairs = 0
    for x, (lo, hi, ri, i) in enumerate(flat):
        for lo2, hi2, rj, j in flat[x + 1:]:
            if lo2 >= hi:
                break
            if order.branch[i] == order.branch[j] or not ('W' in (ri, rj) or {ri, rj} == {'A', 'R'}):
                continue
            n_pairs += 1
            a, b = min(i, j), max(i, j)
            assert order.before(a, b), (what, 'ops %d and %d conflict on [%d, %d) and [%d, %d) and are not ordered' % (a, b, lo, hi, lo2, hi2))
    writes = [(lo, hi, i) for lo, hi, role, i in flat if role == 'W']
    for r, lo, hi, p, residual in reads:
        for wlo, whi, w in writes:
            if wlo < hi and lo < whi and w != p and not (w == r and residual and (wlo, whi) == (lo, hi)):
                assert order.before(w, p) or order.before(r, w), \
                    (what, 'op %d reads [%d, %d) that op %s produced, op %d overwrites [%d, %d) in between' % (r, lo, hi, p, w, wlo, whi))
    return n_pairs


# ------------------------------------------------------------------------------------------------------------------ inference plans
def op_ranges(o):
    """The workspace bytes an lfd_op record touches, as its kernel reads the fields -> {operand: (lo, hi, role)}."""
    N, out_c = o.N, o.tail_cout or o.Cout
    r = {}
    if o.in_off >= 0:
        r['in'] = (o.in_off, o.in_off + N * o.H * o.W * o.Cin * 2, 'R')
    if o.out_off >= 0:
        r['out'] = (o.out_off, o.out_off + N * o.Ho * o.Wo * out_c * 2, 'W')
    if o.res_off >= 0:
        r['res'] = (o.res_off, o.res_off + N * o.Ho * o.Wo * out_c * 2, 'R')
    if o.ds_cout:
        r['out2'] = (o.ds_out_off, o.ds_out_off + N * o.Ho * o.Wo * o.ds_cout * 2, 'W')
    if o.stats_off >= 0:
        r['stats'] = (o.stats_off, o.stats_off + N * o.gn_groups * 16, 'A' if o.kind == nat.OP_CONV else 'R')
    return r


def _stem_size(model, H, W):
    for conv, _, _ in model._backbone.stem_layers():
        H, W = conv_out(H, conv.kernel_size[0], conv.stride[0]), conv_out(W, conv.kernel_size[0], conv.stride[0])
    return H, W


def check_inference_plan(plan, model, what=''):
    """Rules 1-3 on the records of plan._op_array after the statistics memset, the GroupNorm slots and the head's point ranges.
    Producers are found through the op list's tensor names; the bytes a name stands for must be the same for the producer and every
    reader.  -> number of cross-branch overlapping conflicting pairs, all ordered."""
    recs = list(plan._op_array)
    ops = plan._ops
    assert len(recs) == len(ops)
    order = Ops([(0, 0)] + [(o.branch, o.wait_mask) for o in recs])      # op 0: the statistics memset
    acc = [[(0, plan.stats_bytes, 'W')] if plan.stats_bytes else []]
    rng = [op_ranges(o) for o in recs]
    acc += [list(r.values()) for r in rng]
    producer = {}
    for i, op in enumerate(ops):
        for k in ('out', 'out2'):
            if op.get(k) is not None:
                assert op[k] not in producer, (what, 'tensor %s written twice' % op[k])
                producer[op[k]] = (i, k)
    reads = []
    for i, op in enumerate(ops):
        for k, f in (('inp', 'in'), ('res', 'res')):
            name = op.get(k)
            assert (name is None) == (f not in rng[i]), (what, 'op %d: %s' % (i, f))
            if name is None:
                continue
            p, pk = producer[name]
            assert p < i, (what, 'op %d reads %s before op %d writes it' % (i, name, p))
            assert rng[i][f][:2] == rng[p][pk][:2], (what, 'op %d reads %s as bytes %s, op %d wrote %s' % (i, name, rng[i][f][:2], p, rng[p][pk][:2]))
            reads.append((1 + i, rng[i][f][0], rng[i][f][1], 1 + p, f == 'res'))
    # GroupNorm statistics: one slot per GN conv, disjoint, inside the cleared region; a reader reads its input's producer's slot
    slots = sorted(rng[i]['stats'][:2] for i, o in enumerate(recs) if o.kind == nat.OP_CONV and 'stats' in rng[i])
    for (lo, hi), (lo2, _) in zip(slots, slots[1:]):
        assert hi <= lo2, (what, 'GroupNorm statistics slots overlap', (lo, hi), lo2)
    assert all(hi <= plan.stats_bytes for _, hi in slots), (what, 'a GroupNorm statistics slot outside the cleared region')
    for i, o in enumerate(recs):
        if o.kind in (nat.OP_GN_APPLY, nat.OP_HEAD_FINAL) and o.gn_groups:
            p = producer[ops[i]['inp']][0]
            assert recs[p].kind == nat.OP_CONV and recs[p].gn_groups == o.gn_groups and rng[p]['stats'][:2] == rng[i]['stats'][:2], \
                (what, 'op %d does not read the statistics of op %d, which produced its input' % (i, p))
            reads.append((1 + i, rng[i]['stats'][0], rng[i]['stats'][1], 1 + p, False))
        elif o.kind == nat.OP_CONV and o.gn_groups:
            assert o.stats_off >= 0, (what, 'op %d: GroupNorm conv without statistics' % i)
    # head outputs: per output, the levels' point ranges partition [0, P) as level_geometry lays them out
    sizes, P, offs = level_geometry(model._backbone, model._head, *_stem_size(model, plan.H, plan.W))
    assert P == plan.P
    want = sorted((offs[l], offs[l] + h * w, h, w) for l, (h, w) in enumerate(sizes))
    for field in ('n_cls', 'n_reg'):
        got = sorted((o.point_off, o.point_off + o.H * o.W, o.H, o.W) for o in recs if o.kind == nat.OP_HEAD_FINAL and getattr(o, field) > 0)
        assert got == want, (what, field, 'point ranges', got, want)
    return _check(what, order, acc, reads, plan.workspace_bytes)


# ------------------------------------------------------------------------------------------------------------------ training plans
def check_training_ops(plan, ops, what=''):
    """Rules 1-3 on one op list of a TrainPlan (fwd_ops or bwd_ops): named operands take the bytes of their workspace region, a frozen
    prefix's LFD_TOP_INFER op the bytes its lfd_op record gives (its scratch tensors share one recycled region), a ZERO its span.  The
    producer of a read is the last earlier op that wrote or accumulated into the same tensor, or cleared its bytes; PACK / ZERO / UNPACK are
    barriers.
    -> number of cross-branch overlapping conflicting pairs, all ordered."""
    order = Ops([(op.get('branch', 0), op['wait_mask']) for op in ops])
    infer = [op for op in ops if op['kind'] == nat.TOP_INFER]
    prefix = iter(plan._prefix['arr'] if infer else ())
    acc, reads, barriers, made, zeros = [], [], [], {}, []      # made: tensor -> its last writer / accumulator; zeros: (lo, hi, op)
    for i, op in enumerate(ops):
        roles = TrainPlan._ROLES.get(op['kind'])
        ranges = []
        if roles is None:
            barriers.append(i)
            if op['kind'] == nat.TOP_ZERO:
                ranges.append((op['off'][0], op['off'][0] + op['off'][1], 'W', None, False))
                zeros.append(ranges[-1][:2] + (i,))
        elif op['kind'] == nat.TOP_INFER:
            rec = op_ranges(next(prefix))
            for j, f in ((0, 'in'), (1, 'out'), (2, 'res'), (3, 'out2')):
                name = op['off'].get(j)
                assert (name is None) == (f not in rec), (what, i, f)
                if name is not None:
                    assert rec[f][0] == plan._off[name], (what, i, name)
                    ranges.append(rec[f] + (name, j == 2))
        else:
            for j, name in op.get('off', {}).items():
                if name is not None:
                    lo = plan._off[name]
                    ranges.append((lo, lo + plan._sizes[name], roles[j], name, op['kind'] == nat.TOP_CONV and j == 2))
        for lo, hi, role, name, residual in ranges:
            if role == 'R':
                p = max([made.get(name, -1)] + [k for a, b, k in zeros if a <= lo and hi <= b])
                reads.append((i, lo, hi, p if p >= 0 else None, residual))
        for lo, hi, role, name, _ in ranges:
            if role != 'R' and name is not None:
                made[name] = i
        acc.append([rg[:3] for rg in ranges])
    assert next(prefix, None) is None, (what, 'fewer LFD_TOP_INFER ops than prefix records')
    return _check(what, order, acc, reads, plan.workspace_bytes, barriers)
