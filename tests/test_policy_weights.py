"""CPU: the weight blob of the device GNN policy (ddls_b200/policy.py) -- key order = the checkpoint order of the reference's GNNPolicy
module tree (restated in tests/gnn_reference.py with the reference's parameter names), sizes = what the C ABI expects
(ramp_policy_weight_count is host-only code), and malformed checkpoints are rejected with the offending key."""
import ctypes as C

import numpy as np
import pytest

from ddls_b200 import policy as P


@pytest.mark.parametrize('overrides,n_actions', [({}, 17), ({}, 9), (dict(num_rounds=3, out_features_msg=24, out_features_hidden=40,
                                                                       out_features_node=12, out_features_graph=6, fcnet_hiddens=(128,)), 5)])
def test_blob_layout_matches_the_module_tree_and_the_c_abi(overrides, n_actions):
    from gnn_reference import GNNPolicy
    cfg = dict(P.DEFAULT_CONFIG); cfg.update(overrides)
    ref = GNNPolicy(cfg, n_actions)
    sd = ref.state_dict()
    assert list(sd.keys()) == list(P.weight_keys(cfg))
    shapes = P.weight_shapes(cfg, n_actions)
    assert {k: tuple(v.shape) for k, v in sd.items()} == shapes
    blob = P.pack_weights(sd, cfg, n_actions)
    assert blob.dtype == np.float32 and blob.ndim == 1
    L = P._engine.load_library()
    P._bind(L)
    c = P._Config(cfg['in_features_node'], cfg['in_features_edge'], cfg['in_features_graph'], n_actions, cfg['out_features_msg'],
                  cfg['out_features_hidden'], cfg['out_features_node'], cfg['out_features_graph'], cfg['num_rounds'],
                  tuple(cfg['fcnet_hiddens'])[0], 0, 0, 1, 3)
    assert L.ramp_policy_weight_count(C.byref(c)) == len(blob) == sum(int(np.prod(s)) for s in shapes.values())
    # the blob is the parameters in key order, row-major
    off = 0
    for k in P.weight_keys(cfg):
        n = int(np.prod(shapes[k]))
        np.testing.assert_array_equal(blob[off:off + n], sd[k].detach().numpy().ravel())
        off += n


def test_malformed_checkpoints_are_rejected():
    cfg = dict(P.DEFAULT_CONFIG)
    sd = P.random_state_dict(cfg, 17, seed=1)
    missing = dict(sd); del missing['graph_module.1.bias']
    with pytest.raises(KeyError, match='graph_module.1.bias'):
        P.pack_weights(missing, cfg, 17)
    bad = dict(sd); bad['logit_module._logits._model.0.weight'] = np.zeros((9, 256), dtype=np.float32)
    with pytest.raises(ValueError, match='logit_module._logits'):
        P.pack_weights(bad, cfg, 17)
    L = P._engine.load_library()
    P._bind(L)
    c = P._Config(5, 2, 17, 17, 32, 64, 16, 8, 1, 256, 0, 0, 1, 3)            # num_rounds < 2 (gnn.py:40-41)
    assert L.ramp_policy_weight_count(C.byref(c)) == -1


# ---- check_config's bounds (ramp_policy.cu), through ramp_policy_weight_count: host-only code ----
BASE = dict(P.DEFAULT_CONFIG)
BOUNDS = [  # (field, lowest admitted, highest admitted, rejected values)
    ('in_features_node', 1, 128, (0, 129)),
    ('in_features_edge', 1, 128, (0, 129)),
    ('in_features_graph', 1, 96, (0, 97)),
    ('out_features_msg', 2, 128, (0, 1, 3, 127, 129, 130)),
    ('out_features_hidden', 1, 128, (0, 129)),
    ('out_features_node', 1, 96, (0, 97)),
    ('out_features_graph', 1, 32, (0, 33)),
    ('n_actions', 1, 32, (0, 33)),
    ('num_rounds', 2, 8, (1, 9)),
    ('fcnet_hidden', 32, 512, (0, 31, 33, 100, 513, 544)),
    ('aggregator_activation', 0, 1, (-1, 2)),
    ('fcnet_activation', 0, 2, (-1, 1, 3)),
    ('n_models', 1, 1 << 20, (0, -1)),
]


def _count(**kw):
    cfg = dict(BASE, fcnet_hiddens=(kw.pop('fcnet_hidden', 256),))
    n_actions, n_models = kw.pop('n_actions', 17), kw.pop('n_models', 3)
    agg, fca = kw.pop('aggregator_activation', 0), kw.pop('fcnet_activation', 0)
    cfg.update(kw)
    c = P.c_config(cfg, n_actions, n_models)
    c.aggregator_activation, c.fcnet_activation = agg, fca
    L = P._engine.load_library()
    P._bind(L)
    return L.ramp_policy_weight_count(C.byref(c)), cfg, n_actions


@pytest.mark.parametrize('field,lo,hi,rejected', BOUNDS, ids=[b[0] for b in BOUNDS])
def test_weight_count_at_every_bound_of_the_configuration(field, lo, hi, rejected):
    """At the lowest and highest admitted value of each field the count is the sum of weight_shapes; one past either side
    (and, for the even / multiple-of-32 fields, the nearest values in between) is refused with -1."""
    for v in (lo, hi):
        got, cfg, A = _count(**{field: v})
        assert got == sum(int(np.prod(s)) for s in P.weight_shapes(cfg, A).values()), (field, v)
    for v in rejected:
        assert _count(**{field: v})[0] == -1, (field, v)


def test_weight_count_at_the_largest_configuration():
    """Every width at its maximum together (in_features_graph + n_actions = 128, fin = 128, 8 rounds, 512 hidden units)."""
    big = dict(in_features_node=128, in_features_edge=128, in_features_graph=96, out_features_msg=128, out_features_hidden=128,
               out_features_node=96, out_features_graph=32, num_rounds=8)
    got, cfg, A = _count(n_actions=32, fcnet_hidden=512, **big)
    assert got == sum(int(np.prod(s)) for s in P.weight_shapes(cfg, A).values())
    small = dict(in_features_node=1, in_features_edge=1, in_features_graph=1, out_features_msg=2, out_features_hidden=1,
                 out_features_node=1, out_features_graph=1, num_rounds=2)
    got, cfg, A = _count(n_actions=1, fcnet_hidden=32, **small)
    assert got == sum(int(np.prod(s)) for s in P.weight_shapes(cfg, A).values())


# ---- the float64 numpy reference (gnn_reference.embed64 / head64) against the module restatement run in float64 ----
REF_CONFIGS = {
    'yaml': ({}, 17),
    'max': (dict(in_features_node=128, in_features_edge=128, in_features_graph=96, out_features_msg=128, out_features_hidden=128,
                 out_features_node=96, out_features_graph=32, num_rounds=8, fcnet_hiddens=(128,), aggregator_activation='leaky_relu',
                 fcnet_activation='tanh'), 32),
    'min': (dict(in_features_node=1, in_features_edge=1, in_features_graph=1, out_features_msg=2, out_features_hidden=1,
                 out_features_node=1, out_features_graph=1, fcnet_hiddens=(32,)), 1),
    'odd': (dict(in_features_node=33, in_features_edge=3, in_features_graph=63, out_features_msg=66, out_features_hidden=65,
                 out_features_node=95, out_features_graph=31, num_rounds=3, fcnet_hiddens=(96,), aggregator_activation='leaky_relu'), 2),
    'unmasked': (dict(apply_action_mask=False), 9),
}


def _small_graphs(rng):
    """node count, src, dst: zero in-degree, self-loops, duplicate edges, an isolated node, one node, one edge"""
    return [(1, [], []), (2, [0], [1]),
            (6, [0, 0, 1, 2, 2, 3, 3, 3], [1, 1, 2, 2, 3, 0, 3, 1]),                       # node 4 isolated, node 5 only sends
            (40, rng.integers(0, 40, 120), rng.integers(0, 30, 120))]                     # nodes 30..39: zero in-degree


@pytest.mark.parametrize('name', list(REF_CONFIGS))
def test_fp64_reference_equals_the_module_restatement_in_float64(name):
    import torch
    from gnn_reference import GNNPolicy, embed64, head64
    over, A = REF_CONFIGS[name]
    cfg = dict(P.DEFAULT_CONFIG); cfg.update(over)
    sd = P.random_state_dict(cfg, A, seed=3)                                # min's single relu unit is live under seed 3
    ref = GNNPolicy(cfg, A).double()
    ref.load_state_dict({k: torch.from_numpy(v.astype(np.float64)) for k, v in sd.items()}, strict=True)
    rng = np.random.default_rng(1)
    embs = []
    for n, src, dst in _small_graphs(rng):
        src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
        nf = rng.standard_normal((n, cfg['in_features_node']))
        ef = rng.standard_normal((len(src), cfg['in_features_edge']))
        got = embed64(sd, cfg, nf, ef, src, dst)
        with torch.no_grad():
            want = ref.embed(torch.from_numpy(nf), torch.from_numpy(ef), torch.from_numpy(src), torch.from_numpy(dst)).numpy()
        assert got.dtype == want.dtype == np.float64
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
        embs.append(got)
    assert np.ptp(np.concatenate(embs)) > 1e-3
    n = 64
    model = rng.integers(0, len(embs), n)
    gf = rng.standard_normal((n, cfg['in_features_graph']))
    mask = (rng.random((n, A)) < 0.7).astype(np.float64)
    mask[0], mask[1] = 0, 1
    rows = np.stack(embs)[model]
    logits, value = head64(sd, cfg, rows, gf, mask)
    with torch.no_grad():
        wl, wv = ref(torch.from_numpy(rows), torch.from_numpy(np.concatenate([gf, mask], 1)), torch.from_numpy(mask))
    assert wl.dtype == torch.float64
    np.testing.assert_allclose(logits, wl.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(value, wv.numpy(), rtol=1e-12, atol=1e-12)
