"""CPU: tests/tie_reference.py -- forced branches against autograd through a network whose pre-activation sits one ulp of its
bias on either side of 0, explain() on planted flips and planted non-flips, and the near-ties of ResNet-50's static graph."""
import numpy as np
import pytest
import torch

from ppo_reference import params64, policy64
from tie_reference import Tie, deltas, explain, grad64, near_ties, sites


class _G:
    def __init__(self, nf, ef, src, dst):
        self.nf, self.ef, self.src, self.dst = nf, ef, np.asarray(src), np.asarray(dst)


def _cfg(act='relu'):
    from ddls_b200 import policy as P
    return dict(P.DEFAULT_CONFIG, aggregator_activation=act, fcnet_activation=act)


def _setup(act='relu', n=6, seed=3):
    from ddls_b200 import policy as P
    c = _cfg(act)
    rng = np.random.default_rng(seed)
    src, dst = [0, 0, 1, 2, 3], [1, 2, 3, 3, 1]
    g = _G(rng.standard_normal((5, 5)), rng.standard_normal((5, 2)), src, dst)        # node 4: no in-edge, no out-edge
    A = 5
    sd = P.random_state_dict(c, A, seed=seed)
    params = {k: np.asarray(v.numpy() if hasattr(v, 'numpy') else v, np.float64) for k, v in sd.items()}
    model = np.zeros(n, np.int32)
    gf = rng.standard_normal((n, c['in_features_graph']))
    mask = np.ones((n, A), np.uint8)
    mask[:, 3] = 0
    action = rng.integers(0, 3, n)
    adv = rng.standard_normal(n)

    def loss(logits, value):
        from pg_reference import pg_loss64
        return pg_loss64(logits, action, adv)[0] + 0.3 * (value ** 2).sum()
    return c, [g], params, model, gf, mask, loss


def _pre(params, c, graphs, model, gf, mask, site):
    mod, m, r, i, u = site
    for s in sites(params, c, graphs, model, gf, mask):
        if s[:3] == (mod, m, r):
            return s[3][i, u]
    raise KeyError(site)


def _bias_key(site):
    mod, _, r, _, _ = site
    name = {'node': 'node_module', 'edge': 'edge_module', 'own': 'reduce_module', 'msg': 'reduce_module'}.get(mod)
    if name:
        return f'gnn_module.layers.{r}.{name}.1.bias'
    return f'logit_module.{"_hidden_layers" if mod == "hidden" else "_value_branch_separate"}.0._model.0.bias'


@pytest.mark.parametrize('act', ['relu', 'leaky_relu'])
@pytest.mark.parametrize('site', [('msg', 0, 0, 3, 5), ('own', 0, 1, 1, 7), ('edge', 0, 1, 2, 4), ('node', 0, 0, 3, 9),
                                  ('hidden', -1, -1, 2, 17), ('value', -1, -1, 4, 200)])
def test_forced_branch_is_autograd_one_ulp_away(act, site):
    """move the site's bias until its pre-activation changes sign between two adjacent doubles b- < b+ of the bias: the gradient
    at b- with the positive branch forced is autograd's at b+, and at b+ with the other branch forced autograd's at b-"""
    c, graphs, params, model, gf, mask, loss = _setup(act)
    key, u = _bias_key(site), site[4]
    a = _pre(params, c, graphs, model, gf, mask, site)

    def with_bias(b):
        q = dict(params)
        q[key] = params[key].copy()
        q[key][u] = b
        return q
    b0 = params[key][u] - a
    lo, hi = b0 - 1e-9, b0 + 1e-9
    assert _pre(with_bias(lo), c, graphs, model, gf, mask, site) <= 0 < _pre(with_bias(hi), c, graphs, model, gf, mask, site)
    while np.nextafter(lo, np.inf) < hi:
        mid = lo + (hi - lo) / 2
        if mid in (lo, hi):
            break
        if _pre(with_bias(mid), c, graphs, model, gf, mask, site) > 0:
            hi = mid
        else:
            lo = mid
    assert hi == np.nextafter(lo, np.inf)
    pre_lo, pre_hi = (_pre(with_bias(b), c, graphs, model, gf, mask, site) for b in (lo, hi))
    assert pre_lo <= 0 < pre_hi and pre_hi - pre_lo <= 4 * np.spacing(abs(hi))
    item_site = site
    for b_nat, b_forced, on in ((hi, lo, True), (lo, hi, False)):
        want = grad64(with_bias(b_nat), c, graphs, model, gf, mask, loss)[0]
        got = grad64(with_bias(b_forced), c, graphs, model, gf, mask, loss, forced={item_site: on})[0]
        unforced = grad64(with_bias(b_forced), c, graphs, model, gf, mask, loss)[0]
        scale = max(np.abs(g).max() for g in want.values())
        for k in want:
            np.testing.assert_allclose(got[k], want[k], rtol=0, atol=1e-9 * scale, err_msg=k)
        moved = max(np.abs(unforced[k] - want[k]).max() for k in want)
        assert moved > 1e-6 * scale                                    # the flip matters: the pin is not vacuous


def _planted(seed):
    c, graphs, params, model, gf, mask, loss = _setup('relu', n=12, seed=seed)
    ties = near_ties(params, c, graphs, model, gf, mask, tau=0.05)
    g64, gl, gv = grad64(params, c, graphs, model, gf, mask, loss)
    ds = deltas(params, c, graphs, model, gf, mask, gl, gv, ties)
    g32 = grad64(params, c, graphs, model, gf, mask, loss, dtype=torch.float32)[0]
    e32 = {k: np.linalg.norm(g32[k] - g64[k]) / max(np.linalg.norm(g64[k]), 1e-300) for k in g64}
    return c, graphs, params, model, gf, mask, loss, ties, g64, ds, e32


def _rel(d, g64):
    return max(np.linalg.norm(d[k]) / np.linalg.norm(g64[k]) for k in g64 if np.linalg.norm(g64[k]) > 0)


def test_deltas_are_the_flipped_gradients():
    """D_i (upstream gradient at the unflipped forward, GNN ties through d emb, read-out ties on their row) against the whole
    batch's float64 gradient with the branch flipped, less the unflipped one"""
    c, graphs, params, model, gf, mask, loss, ties, g64, ds, e32 = _planted(7)
    mods = {t.site[0] for t in ties}
    assert {'msg', 'hidden'} <= mods, mods
    for t, d in list(zip(ties, ds))[:12]:
        full = grad64(params, c, graphs, model, gf, mask, loss, forced=t.flipped())[0]
        want = {k: full[k] - g64[k] for k in g64}
        scale = max(np.abs(x).max() for x in want.values())
        for k in want:                  # the forward moved by about the margin: the upstream gradient by about as much
            np.testing.assert_allclose(d[k], want[k], rtol=0, atol=max(0.05 * scale, 1e-12), err_msg=f'{t}: {k}')


def test_explain_recovers_a_planted_flip():
    c, graphs, params, model, gf, mask, loss, ties, g64, ds, e32 = _planted(7)
    big = [i for i, d in enumerate(ds) if _rel(d, g64) > 1e-2]
    assert len(big) >= 3
    rng = np.random.default_rng(0)
    for j in big[:3]:
        noise = {k: 1e-7 * np.linalg.norm(g64[k]) / np.sqrt(g64[k].size) * rng.standard_normal(g64[k].shape) for k in g64}
        g = {k: g64[k] + ds[j][k] + noise[k] for k in g64}
        S, resid = explain(g, g64, ds, e32, ties)
        assert S == [j], (S, j, str(ties[j]))
        assert max(resid.values()) <= 1e-4
    j, i = big[0], big[1]                                             # two flips at once
    S, _ = explain({k: g64[k] + ds[j][k] + ds[i][k] for k in g64}, g64, ds, e32, ties)
    assert sorted(S) == sorted([i, j])
    S, resid = explain(g64, g64, ds, e32, ties)                        # nothing to explain
    assert S == [] and max(resid.values()) == 0.0


def test_explain_refuses_a_perturbation_that_is_no_flip():
    """a perturbation with a planted flip's norm per tensor, in a random direction: no set of flips accounts for it"""
    c, graphs, params, model, gf, mask, loss, ties, g64, ds, e32 = _planted(7)
    rng = np.random.default_rng(1)
    big = [i for i, d in enumerate(ds) if _rel(d, g64) > 1e-2]
    for j in big[:3]:
        pert = {}
        for k in g64:
            r = rng.standard_normal(g64[k].shape)
            pert[k] = r * (np.linalg.norm(ds[j][k]) / np.linalg.norm(r))
        with pytest.raises(AssertionError, match='not explained'):
            explain({k: g64[k] + pert[k] for k in g64}, g64, ds, e32, ties)
    with pytest.raises(AssertionError, match='not explained'):         # the right flip with the wrong sign
        explain({k: g64[k] - ds[big[0]][k] for k in g64}, g64, ds, e32, ties)


def test_near_ties_of_resnet50_at_seed_4():
    """the bench's ResNet-50 static graph (330 nodes, 361 edges) at random_state_dict(DEFAULT_CONFIG, 17, seed=4): three
    reduce-module message items within 1e-5 of a tie, and none at seed 2; no edge-module item near one"""
    from ddls_b200 import policy as P, workload
    from ddls_b200.observation import static_observation
    st = static_observation(workload.make_graph('resnet'))
    g = _G(st['node_features'], st['edge_features'], st['edges_src'], st['edges_dst'])
    assert (len(g.nf), len(g.src)) == (330, 361)
    rows = (np.zeros(1, np.int32), np.zeros((1, 17)), np.ones((1, 17), np.uint8))

    def gnn_ties(seed, tau):
        sd = P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=seed)
        return [t for t in near_ties(sd, P.DEFAULT_CONFIG, [g], *rows, tau=tau) if t.site[1] >= 0]
    close = gnn_ties(4, 1e-5)
    assert [t.site for t in close] == [('msg', 0, 1, 295, 1), ('msg', 0, 0, 9, 7), ('msg', 0, 0, 8, 30)]
    np.testing.assert_allclose([t.margin for t in close], [6.0e-6, 8.9e-6, 9.8e-6], rtol=0.02)
    assert len(gnn_ties(4, 1e-4)) == 20
    edge_margin = min(s[4].min() for s in sites(P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=4), P.DEFAULT_CONFIG, [g], *rows)
                      if s[0] == 'edge')
    assert edge_margin >= 3.5e-2
    assert gnn_ties(2, 1e-5) == []
    assert str(close[0]).startswith('msg model 0 round 1 edge 295 unit 1')


def test_no_forced_branch_is_the_plain_forward():
    c, graphs, params, model, gf, mask, loss = _setup('relu')
    p = params64(params, requires_grad=False)
    a = policy64(p, c, graphs, model, gf, mask)
    b = policy64(p, c, graphs, model, gf, mask, forced={})
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    with pytest.raises(ValueError, match='tanh'):
        c2 = dict(c, aggregator_activation='tanh')
        policy64(p, c2, graphs, model, gf, mask, forced={('msg', 0, 0, 0, 0): True})
    t = Tie(('hidden', -1, -1, 3, 7), -1e-9, 1e-8)
    assert t.flipped() == {('hidden', -1, -1, 3, 7): True} and str(t).startswith('hidden row 3 unit 7')


def test_identical_rows_flip_together():
    """two identical rows share every read-out tie: flips() makes one candidate of the pair, and explain() finds the pair where
    each row's flip alone would be refused (their advantages have opposite signs, so one row's D_i overshoots)"""
    from pg_reference import pg_loss64
    from tie_reference import flips
    c, graphs, params, model, gf, mask, _ = _setup('relu', n=8, seed=7)
    gf[5] = gf[2]
    action = np.array([0, 1, 2, 0, 1, 2, 0, 1])
    adv = np.array([0.5, -1.0, 1.3, 0.2, -0.7, -1.1, 0.9, 0.4])

    def loss(logits, value):
        return pg_loss64(logits, action, adv)[0]
    ties = near_ties(params, c, graphs, model, gf, mask, tau=0.05)
    g64, gl, gv = grad64(params, c, graphs, model, gf, mask, loss)
    ds = deltas(params, c, graphs, model, gf, mask, gl, gv, ties)
    e32 = {k: 0.0 for k in g64}
    cands, cds = flips(ties, ds)
    pairs = [i for i, f in enumerate(cands) if f.ties[0].site[0] == 'hidden' and {t.site[3] for t in f.ties} == {2, 5}]
    assert pairs and len(cands) < len(ties)
    j = max(pairs, key=lambda i: _rel(cds[i], g64))
    assert _rel(cds[j], g64) > 1e-3
    S, resid = explain({k: g64[k] + cds[j][k] for k in g64}, g64, cds, e32, cands)
    assert S == [j] and max(resid.values()) <= 1e-4
    assert str(cands[j]).startswith('hidden rows 2, 5 unit')
