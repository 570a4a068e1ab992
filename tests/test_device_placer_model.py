"""CPU: the formulation ramp_env_place_kernel computes (ddls_b200/csrc/ramp_env.cuh), restated in numpy over many cluster states at
once -- every op's placement a candidate block index, parent collective placement before first fit, candidates in the host's
enumeration order, free memory updated in the C++'s order -- against ramp_first_fit_place_many and the reference's recorded
decisions; and the canonical mask the kernel looks templates up by against the template key of the host's placer."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from ddls_b200 import synth
from ddls_b200.batched import A100_MEMORY, _Model, candidate_blocks, canonical_mask, place_smem_per_warp, placer_tables

HERE = os.path.dirname(os.path.abspath(__file__))


def kernel_model(tables, degree, cand_ptr, blocks, busy, free_mem):
    """busy [n, W] bool, free_mem [n, W]: per state, the candidate index of every op (-1 when the job cannot be placed) and ok."""
    n_states, W = busy.shape
    n_ops = len(tables['topo'])
    sp = tables['splits'][degree]
    mem = free_mem.astype(np.float64).copy()
    where = np.full((n_states, n_ops), -1, dtype=np.int64)
    ok = np.ones(n_states, dtype=bool)
    rows = np.arange(n_states)
    by_degree = {d: np.array(blocks[cand_ptr[d]:cand_ptr[d + 1]], dtype=np.int64).reshape(-1, d)
                 for d in range(1, len(cand_ptr) - 1) if cand_ptr[d + 1] > cand_ptr[d]}
    for op in tables['topo']:
        split, need = int(sp[op]), float(tables['need'][op])
        c = np.full(n_states, -1, dtype=np.int64)
        for pa in tables['parents'][tables['par_ptr'][op]:tables['par_ptr'][op + 1]]:
            if sp[pa] != split or split not in by_degree:              # no block of `split` servers: the parent failed
                continue
            open_ = ok & (c < 0)
            srv = by_degree[split][np.maximum(where[:, pa] - cand_ptr[split], 0)]
            avail = np.zeros(n_states)
            for j in range(split):                                    # the C++'s summation order
                avail = avail + mem[rows, srv[:, j]]
            take = open_ & (avail >= need)
            c[take] = where[take, pa]
        op_size = need / split
        ff = ok & (c < 0)
        if ff.any():
            if split not in by_degree:
                ok[ff] = False
            else:
                bd = by_degree[split]
                fit = ~busy[:, bd].any(axis=2) & (mem[:, bd] >= op_size).all(axis=2)
                has = fit.any(axis=1)
                c[ff & has] = cand_ptr[split] + fit.argmax(axis=1)[ff & has]
                ok[ff & ~has] = False
        live = ok & (c >= 0)
        if live.any():
            srv = by_degree[split][c[live] - cand_ptr[split]]
            r = rows[live][:, None]
            mem[r, srv] = mem[r, srv] - op_size
        where[:, op] = np.where(ok, c, -1)
    return where, ok


def union_masks(where, ok, blocks, n_words):
    out = np.zeros((len(ok), n_words), dtype=np.uint64)
    for k in np.nonzero(ok)[0]:
        for c in set(where[k].tolist()):
            for s in blocks[c]:
                out[k, s >> 6] |= np.uint64(1 << (s & 63))
    return out


def kernel_canonical(words, shape, n_words):
    """The kernel's construction: a presence flag per axis value, exclusive prefix sums as ranks, one bit per used server."""
    C_, R, S = shape
    used = [s for s in range(C_ * R * S) if (int(words[s >> 6]) >> (s & 63)) & 1]
    rank = np.zeros(C_ + R + S, dtype=np.int64)
    for s in used:
        rank[s // (R * S)] = rank[C_ + (s // S) % R] = rank[C_ + R + s % S] = 1
    rank = np.concatenate([np.cumsum(rank[a:b]) - rank[a:b] for a, b in ((0, C_), (C_, C_ + R), (C_ + R, C_ + R + S))])
    out = [0] * n_words
    for s in used:
        j = (rank[s // (R * S)] * R + rank[C_ + (s // S) % R]) * S + rank[C_ + R + s % S]
        out[j >> 6] |= 1 << int(j & 63)
    return tuple(out)


def native_place_many(g, splits, shape, states, n_words):
    from ddls_b200 import engine
    from ddls_b200.expand import _FwdGraph
    L = engine.load_library()
    L.ramp_first_fit_place_many.restype = C.c_int
    L.ramp_first_fit_place_many.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    mem = np.ascontiguousarray([a + p for a, p in zip(g.act, g.par)], dtype=np.float64)
    zero = np.zeros(g.n)
    es = np.ascontiguousarray([u for u, _ in g.edges], dtype=np.int32)
    ed = np.ascontiguousarray([v for _, v in g.edges], dtype=np.int32)
    cg = _FwdGraph(g.n, len(g.edges), zero.ctypes.data, zero.ctypes.data, mem.ctypes.data, zero.ctypes.data, es.ctypes.data, ed.ctypes.data)
    sp = np.ascontiguousarray(splits, dtype=np.int32)
    states = np.ascontiguousarray(states, dtype=np.uint64)
    masks = np.zeros((len(states), n_words), dtype=np.uint64)
    ok = np.zeros(len(states), dtype=np.uint8)
    assert L.ramp_first_fit_place_many(C.byref(cg), sp.ctypes.data, (C.c_int32 * 3)(*shape), A100_MEMORY, len(states), n_words,
                                       states.ctypes.data, masks.ctypes.data, ok.ctypes.data) == 0
    return masks, ok.astype(bool)


def two_source_graph():
    """Two input ops feeding one chain, with small ops that split fewer ways than the degree."""
    g = synth.ForwardGraph(name='two_source')
    for i, f in enumerate([0.004, 0.3, 0.05, 0.2, 0.012, 0.09]):
        g.add('Linear', f, 2 * f, 2e8 * (i + 1), 1e8)
    g.edges += [(1, 3), (2, 3), (3, 4), (4, 5), (2, 6), (5, 6)]
    return g


def memory_graph(parent_fits: bool):
    """A parent on 4 servers whose child needs their whole free memory: parent collective placement takes the parent's block when
    parent_fits (the child's bytes equal what the parent left free there) and falls through to first fit, onto another block, when
    the child needs 4 bytes more."""
    g = synth.ForwardGraph(name='mem_fit' if parent_fits else 'mem_nofit')
    g.add('Linear', 0.04, 0.08, 40e9, 0.0)                          # 4 sub-ops of 10 GB
    child = 4 * A100_MEMORY - 40e9
    g.add('Linear', 0.04, 0.08, child if parent_fits else child + 4.0, 0.0)
    g.add('Linear', 0.01, 0.02, 1e6, 0.0)
    g.edges += [(1, 2), (2, 3)]
    return g


def graphs():
    return {'res2': synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3),
            'chain6': synth.chain_graph(6, 'chain6'), 'tfm1': synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4),
            'bert': synth.transformer_like_graph(n_layers=12, name='bert_base_like', seed=2),
            'two_source': two_source_graph(), 'mem_fit': memory_graph(True), 'mem_nofit': memory_graph(False)}


def random_states(rng, W, n_words, n):
    busy = rng.random((n, W)) < rng.uniform(0.0, 0.95, size=(n, 1))
    busy[:8] = False                                                # the empty cluster
    states = np.zeros((n, n_words), dtype=np.uint64)
    for s in range(W):
        states[:, s >> 6] |= busy[:, s].astype(np.uint64) << np.uint64(s & 63)
    return busy, states


CASES = [(name, shape) for shape in ((4, 4, 4), (8, 8, 4)) for name in ('res2', 'chain6', 'tfm1', 'bert', 'two_source')] + \
        [('mem_fit', (4, 4, 4)), ('mem_nofit', (4, 4, 4))]


@pytest.mark.parametrize('name,shape', CASES, ids=lambda x: x if isinstance(x, str) else 'x'.join(map(str, x)))
def test_kernel_formulation_equals_native_placer(name, shape):
    """Every degree the action set has, several thousand random busy states: the same server set for every placed job, the same
    failures, and a canonical mask that identifies the host's template key exactly."""
    g = graphs()[name]
    W, D = int(np.prod(shape)), 16
    n_words = (W + 63) // 64
    model = _Model(g, 0.01, 50)
    tables = placer_tables([model], D)
    cand_ptr, blocks = candidate_blocks(shape, D)
    rng = np.random.default_rng(abs(hash((name, shape))) % 2**32)
    n = 3000 if W <= 64 else 1500
    busy, states = random_states(rng, W, n_words, n)
    n_failed = n_uneven = 0
    key_of_mask, mask_of_key = {}, {}
    for d in [1] + list(range(2, D + 1, 2)):
        where, ok = kernel_model(tables, d, cand_ptr, blocks, busy, np.full((n, W), A100_MEMORY))
        got = union_masks(where, ok, blocks, n_words)
        want, want_ok = native_place_many(g, model.splits(d), shape, states, n_words)
        np.testing.assert_array_equal(ok, want_ok, err_msg=f'degree {d}')
        np.testing.assert_array_equal(got[ok], want[ok], err_msg=f'degree {d}')
        n_failed += int((~ok).sum())
        n_uneven += len(set(model.splits(d))) > 1
        for k in np.unique(np.nonzero(ok)[0][:400]):
            coords = [((s // (shape[1] * shape[2])), (s // shape[2]) % shape[1], s % shape[2])
                      for s in range(W) if (int(got[k, s >> 6]) >> (s & 63)) & 1]
            ranks = [{v: i for i, v in enumerate(sorted({c[ax] for c in coords}))} for ax in range(3)]
            tkey = (d, tuple((ranks[0][c[0]], ranks[1][c[1]], ranks[2][c[2]]) for c in coords))   # _place_many's key
            cm = canonical_mask(coords, shape, n_words)
            assert kernel_canonical(got[k], shape, n_words) == cm
            assert mask_of_key.setdefault(tkey, cm) == cm and key_of_mask.setdefault((d, cm), tkey) == tkey
    assert n_failed > 0
    if name in ('bert', 'two_source'):
        assert n_uneven > 0


def test_memory_graphs_take_both_sides_of_the_parent_test():
    """On the empty cluster the child shares its parent's block exactly when parent_fits; otherwise first fit moves it."""
    shape, D = (4, 4, 4), 4
    cand_ptr, blocks = candidate_blocks(shape, D)
    for fits in (True, False):
        model = _Model(memory_graph(fits), 0.01, 50)
        assert model.splits(4)[:2] == [4, 4]
        tables = placer_tables([model], D)
        where, ok = kernel_model(tables, 4, cand_ptr, blocks, np.zeros((1, 64), dtype=bool), np.full((1, 64), A100_MEMORY))
        assert ok[0] and (where[0, 1] == where[0, 0]) == fits


def test_kernel_formulation_reproduces_reference_decisions():
    """tests/fixtures/placer_cases.json: the reference's RampFirstFitOpPlacer on busy clusters with per-server free memory."""
    cases = json.load(open(os.path.join(HERE, 'fixtures', 'placer_cases.json')))
    from ddls_b200.placer import backward_op_id, partitioned_op_id
    for i, c in enumerate(cases):
        shape = tuple(c['shape'])
        R, S = shape[1], shape[2]
        W = int(np.prod(shape))
        n = len(c['nodes'])
        g = synth.ForwardGraph(name=f'case{i}')
        for m in c['mem']:
            g.add('Linear', 0.0, 0.0, m, 0.0)
        g.edges = [(int(u), int(v)) for u, v in c['edges']]
        split_of = dict(zip(c['mp_split_ids'], c['mp_splits']))
        sp = [split_of.get(str(k), 1) for k in range(1, n + 1)]
        tables = placer_tables([_Model(g, 0.01, 50)], 1)
        tables['splits'] = np.asarray([sp, sp], dtype=np.int32)         # the recorded splits at "degree 1"
        cand_ptr, blocks = candidate_blocks(shape, max(sp))
        idx = lambda sv: (sv[0] * R + sv[1]) * S + sv[2]
        busy = np.zeros((1, W), dtype=bool)
        free = np.zeros((1, W))
        for sv, m, j in c['ramp']:
            busy[0, idx(sv)] = bool(j)
            free[0, idx(sv)] = m
        where, ok = kernel_model(tables, 1, cand_ptr, blocks, busy, free)
        if c['placement'] is None:
            assert not ok[0], i
            continue
        assert ok[0], i
        got = {}
        for op in range(n):
            fwd, bwd = str(op + 1), backward_op_id(str(op + 1), n)
            for j, s in enumerate(blocks[where[0, op]]):
                coord = [s // (R * S), (s // S) % R, s % S]
                if sp[op] > 1:
                    got[partitioned_op_id(fwd, j)] = got[partitioned_op_id(bwd, j)] = coord
                else:
                    got[fwd] = got[bwd] = coord
        assert got == c['placement'], i


def test_placer_tables_follow_the_graph():
    g = two_source_graph()
    t = placer_tables([_Model(g, 0.01, 50), _Model(synth.chain_graph(3, 'c3'), 0.01, 50)], 4)
    assert t['op_ptr'].tolist() == [0, 6, 9]
    assert t['topo'][:6].tolist() == [0, 1, 2, 5, 3, 4] or t['topo'][:6].tolist() == [0, 1, 2, 3, 4, 5]
    assert t['parents'][t['par_ptr'][2]:t['par_ptr'][3]].tolist() == [0, 1]            # edge order
    assert t['parents'][t['par_ptr'][5]:t['par_ptr'][6]].tolist() == [1, 4]
    assert t['topo'][6:].tolist() == [0, 1, 2]
    assert t['splits'].shape == (5, 9) and (t['splits'] >= 1).all()


def test_shared_memory_budget_matches_header():
    src = open(os.path.join(HERE, '..', 'include', 'ramp_b200.h')).read()
    from ddls_b200 import batched
    assert f'#define RAMP_ENV_PLACE_SMEM_PER_WARP {batched.PLACE_SMEM_PER_WARP}' in src
    assert place_smem_per_warp(64, 100) == 8 * 72 + 400
    assert place_smem_per_warp(256, 2544) == batched.PLACE_SMEM_PER_WARP
    assert place_smem_per_warp(256, 2545) > batched.PLACE_SMEM_PER_WARP
