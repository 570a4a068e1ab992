"""The thread kernel's key-ordered ready-flow frontier and its one-pass channel winners, on a model (no GPU).

The small-frontier half of ramp_lookahead_thread.cuh keeps the ready flow entries in descending key order (a completed
class's flows, stored in that order in the blob, are merged in; survivor compaction keeps it) and finds the channel
winners in one pass: an entry wins unless every group of its set is claimed by an entry with a larger key, and in key
order those are exactly the entries before its run of equal keys.  These tests check that this gives the winners and the
t_comm of the pairwise rule (tests/quotient_model.py) on every frontier the goldens' quotients and random DAGs reach, and
on random frontiers with key ties and overlapping group sets, and that neither depends on the order of the frontier.
"""
import math

import numpy as np
import pytest

from conftest import golden_files
from golden_io import Golden
import quotient_model as qm
from ddls_b200.quotient import quotient as native_quotient

MAX_SIZE = 3000          # classes + entries of the quotients the Python tick loop below is run on


def pairwise(front):
    """front: [(key, groups, rem)] in any order -> (indices of the winners, t_comm)."""
    win = []
    for k, (key, gm, _) in enumerate(front):
        open_groups = gm
        for key2, gm2, _ in front:
            if key2 > key:
                open_groups &= ~gm2
        if open_groups:
            win.append(k)
    return win, min([front[k][2] for k in win], default=math.inf)


def one_pass(front):
    """front in descending key order -> (indices of the winners, t_comm), as the kernel's phase D walks it."""
    win, seen, claimed = [], 0, 0
    for k, (key, gm, _) in enumerate(front):
        assert k == 0 or front[k - 1][0] >= key, 'frontier not in key order'
        if k > 0 and key != front[k - 1][0]:
            claimed = seen
        if gm & ~claimed:
            win.append(k)
        seen |= gm
    return win, min([front[k][2] for k in win], default=math.inf)


def check_frontier(front, rng):
    """One-pass on the key-ordered frontier == pairwise, whatever the order of equal keys or of the frontier."""
    want_win, want_t = pairwise(front)
    want = sorted((front[k][0], front[k][1], front[k][2]) for k in want_win)
    for _ in range(3):
        perm = list(rng.permutation(len(front)))
        shuffled = [front[k] for k in perm]
        w, t = pairwise(shuffled)
        assert t == want_t and sorted(shuffled[k] for k in w) == want
        ordered = sorted(shuffled, key=lambda e: -e[0])          # stable: equal keys keep the shuffled order
        w, t = one_pass(ordered)
        assert t == want_t and sorted(ordered[k] for k in w) == want


def run_key_ordered(q, rng):
    """tests/quotient_model.run_lookahead_quotient with the kernel's frontier discipline: flows merged in key order,
    winners by one pass, completed entries' children in slot order.  Checks every frontier against the pairwise rule."""
    N, E = q.n_ops, q.n_deps
    row = q.row_ptr
    in_deg = np.bincount(q.dep_dst, minlength=N) if E else np.zeros(N, dtype=np.int64)
    par_done = [0] * N
    key = [int(k) for k in q.dep_key]
    grp = [int(q.dep_group_mask[e]) if q.masks_valid else (0 if int(q.dep_channel[e]) == 0xFFFFFFFF else 1 << int(q.dep_channel[e]))
           for e in range(E)]
    # the blob's order: each class's flows by descending key (stable), then its non-flows
    out_flows = [sorted([e for e in range(int(row[c]), int(row[c + 1])) if q.dep_is_flow[e]], key=lambda e: -key[e])
                 for c in range(N)]
    ops = [(i, float(q.op_cost[i]) + 0.0) for i in range(N) if in_deg[i] == 0]
    flows, nf = [], []
    trace_n, trace_tick = [], []
    t = 0.0
    ops_completed = deps_completed = 0
    n_frontiers = 0
    while True:
        wkey = {}
        for op, _ in ops:
            wkey[int(q.op_worker[op])] = max(wkey.get(int(q.op_worker[op]), 0), int(q.op_key[op]))
        winners = [(op, rem) for op, rem in ops if wkey[int(q.op_worker[op])] == int(q.op_key[op])]
        t_op = min([rem for _, rem in winners], default=math.inf)
        any_nf = len(nf) > 0
        if any_nf:
            t_comm = 0.0
        else:
            front = [(key[e], grp[e], rem) for e, rem in flows]
            check_frontier(front, rng)
            _, t_comm = one_pass(front)
            n_frontiers += len(front) > 0
        tick = t_comm if t_comm < t_op else t_op
        t += tick
        trace_n.append(sum(int(q.op_weight[op]) for op, _ in winners))
        trace_tick.append(tick)
        ops_next = []

        def complete_dep(e):
            child = int(q.dep_dst[e])
            old = par_done[child]
            par_done[child] = old + int(q.dep_inc[e])
            if old < int(q.op_threshold[child]) <= par_done[child]:
                ops_next.append((child, float(q.op_cost[child]) + 0.0))
        if any_nf:
            for e in nf:
                complete_dep(e)
            deps_completed += len(nf)
            nf = []
        else:
            done = [e for e, rem in flows if rem <= tick]
            flows = [(e, rem - tick) for e, rem in flows if rem > tick]
            for e in done:
                complete_dep(e)
            deps_completed += len(done)
        win_set = {op for op, _ in winners}
        for op, rem in ops:
            if op in win_set:
                if rem <= tick:
                    ops_completed += 1
                    run = [(e, float(q.dep_run_time[e]) + 0.0) for e in out_flows[op]]
                    flows = sorted(flows + run, key=lambda f: -key[f[0]])      # the merge (order of equal keys is free)
                    nf.extend(e for e in range(int(row[op]), int(row[op + 1])) if not q.dep_is_flow[e])
                    continue
                rem = rem - tick
            ops_next.append((op, rem))
        ops = ops_next
        if (ops_completed == N and deps_completed == E) or math.isinf(tick):
            break
    return dict(n_ticks=len(trace_tick), jct=t * float(q.num_training_steps), trace_n_active=np.array(trace_n, dtype=np.int32),
                trace_tick=np.array(trace_tick, dtype=np.float64)), n_frontiers


def check_quotient(q, rng):
    want = qm.run_lookahead_quotient(q)
    got, n = run_key_ordered(q, rng)
    assert got['n_ticks'] == want['n_ticks'] and got['jct'] == want['jct']
    np.testing.assert_array_equal(got['trace_tick'], want['trace_tick'])
    np.testing.assert_array_equal(got['trace_n_active'], want['trace_n_active'])
    return n


@pytest.mark.parametrize('fname', golden_files())
def test_one_pass_winners_on_golden_quotients(fname):
    rng = np.random.default_rng(7)
    checked = 0
    for t in Golden(fname).templates:
        for q in (native_quotient(t), qm.identity_quotient(t)):
            if q.n_ops + q.n_deps <= MAX_SIZE:
                checked += check_quotient(q, rng)
    if checked == 0:
        pytest.skip(f'no quotient of {fname} is small enough for the Python tick loop')


@pytest.mark.parametrize('degree', [2, 4, 8, 16])
def test_one_pass_winners_on_the_bench_quotients(degree):
    """The bench's ResNet-50-like job on the 4x4x4 RAMP: the quotients every step of bench.py runs."""
    from ddls_b200 import synth
    from ddls_b200.template_builder import RampShape, build_template
    q = native_quotient(build_template(synth.resnet_like_graph(), degree, RampShape(4, 4, 4)))
    assert check_quotient(q, np.random.default_rng(degree)) > 500


def test_one_pass_winners_on_random_dags():
    from ddls_b200.template_builder import random_dag_template
    rng = np.random.default_rng(1234)
    n = 0
    for size, w in zip(rng.integers(2, 200, size=40), rng.integers(1, 9, size=40)):
        t = random_dag_template(rng, int(size), n_workers=int(w))
        for q in (native_quotient(t), qm.identity_quotient(t)):
            n += check_quotient(q, rng)
    assert n > 1000


def test_one_pass_winners_on_random_frontiers():
    """Key ties, overlapping group sets, empty sets (no channel), equal remaining times, up to 16 entries."""
    rng = np.random.default_rng(11)
    for _ in range(4000):
        F = int(rng.integers(1, 17))
        keys = rng.integers(1, int(rng.integers(2, 8)), size=F)
        front = [(int(k), int(rng.integers(0, 16)) & int(rng.integers(0, 16)), float(rng.integers(0, 5)) / 4)
                 for k in keys]
        check_frontier(front, rng)
