"""CPU: the read-out the algorithm configs set (scripts/ramp_job_partitioning_configs/algo/{ppo,impala,pg,es}.yaml: fcnet_hiddens
[action_space.n]; vf_share_layers False under ppo.yaml, RLlib's default True under the others):

- ramp_policy_weight_count equals the sum of weight_shapes at H = n_actions, shared or not, and at the two yaml models (5,668 and
  5,243 weights at 17 actions); widths other than a multiple of 32 or n_actions, and vf_share_layers outside {0, 1}, are refused;
- pack_weights / unpack_weights round-trip both key sets and refuse the other one, naming the key;
- tests/shared_vf_reference.py's head64 (numpy) and policy64 (torch), the separate-branch restatements with the value hidden layer
  tied to the policy's, equal its module restatement GNNPolicy with vf_share_layers=True in float64, and the PPO, IMPALA and PG
  losses' gradients through policy64 equal autograd through that module; fold() of a tied gradient is the shared one."""
import ctypes as C

import numpy as np
import pytest
import torch

from ddls_b200 import policy as P


def _lib():
    L = P._engine.load_library()
    P._bind(L)
    return L


def _count(c, A, n_models=3):
    return _lib().ramp_policy_weight_count(C.byref(P.c_config(c, A, n_models)))


def _model(A, shared):
    return dict(P.DEFAULT_CONFIG, fcnet_hiddens=(A,), vf_share_layers=bool(shared))


def _sum(c, A):
    return sum(int(np.prod(s)) for s in P.weight_shapes(c, A).values())


@pytest.mark.parametrize('shared', [0, 1])
@pytest.mark.parametrize('A', [1, 17, 31])
def test_weight_count_at_hidden_width_n_actions(A, shared):
    c = _model(A, shared)
    assert _count(c, A) == _sum(c, A) > 0
    assert P.c_config(c, A, 3).vf_share_layers == shared
    keys = P.weight_keys(c)
    assert ('logit_module._value_branch_separate.0._model.0.weight' in keys) == (not shared)
    assert P.weight_shapes(c, A)['logit_module._value_branch._model.0.weight'] == (1, A)


def test_weight_count_of_the_yaml_models():
    for algo, n in (('ppo', 5668), ('impala', 5243), ('pg', 5243), ('es', 5243)):
        c = P.algo_model_config(algo, 17)
        assert c['fcnet_hiddens'] == (17,) and c['vf_share_layers'] == (algo != 'ppo')
        assert _count(c, 17) == _sum(c, 17) == n, algo
    assert _count(P.DEFAULT_CONFIG, 17) == 21920                        # gnn.yaml's [256], today's model, unchanged
    with pytest.raises(ValueError, match='apex_dqn'):
        P.algo_model_config('apex_dqn', 17)


def test_refused_widths_and_sharing_values():
    L = _lib()
    for H in (16, 18, 0, 31, 33, 100, 513, 544):
        c = P.c_config(dict(P.DEFAULT_CONFIG, fcnet_hiddens=(H,)), 17, 3)
        assert L.ramp_policy_weight_count(C.byref(c)) == -1, H
        h = C.c_void_p()
        assert L.ramp_policy_create(0, C.byref(c), C.byref(h)) != 0, H              # refused before any device call
        assert b'multiple of 32' in L.ramp_last_error(), H
    for v in (2, -1):
        c = P.c_config(_model(17, 1), 17, 3)
        c.vf_share_layers = v
        assert L.ramp_policy_weight_count(C.byref(c)) == -1, v
    # a positional configuration without the field (as older callers build it) is the separate value branch
    c = P._Config(5, 2, 17, 17, 32, 64, 16, 8, 2, 256, 0, 0, 1, 3)
    assert c.vf_share_layers == 0 and L.ramp_policy_weight_count(C.byref(c)) == 21920


@pytest.mark.parametrize('shared', [0, 1])
def test_pack_unpack_round_trip_and_the_other_key_set_is_refused(shared):
    A = 17
    c, other = _model(A, shared), _model(A, 1 - shared)
    sd = P.random_state_dict(c, A, seed=3)
    assert list(sd) == list(P.weight_keys(c))
    blob = P.pack_weights(sd, c, A)
    assert len(blob) == _count(c, A)
    back = P.unpack_weights(blob, c, A)
    assert list(back) == list(sd)
    for k in sd:
        np.testing.assert_array_equal(back[k], sd[k])
    wrong = P.random_state_dict(other, A, seed=3)
    key = 'logit_module._value_branch_separate.0._model.0.weight'
    with pytest.raises(KeyError, match=key.replace('.', r'\.')):
        P.pack_weights(wrong, c, A)
    with pytest.raises(ValueError):
        P.unpack_weights(P.pack_weights(wrong, other, A), c, A)


def test_the_shared_value_layer_reads_the_policy_hidden_layer():
    """with vf_share_layers the value is vb + vW . h, h the policy's hidden activations: the numpy head64 equals that by hand"""
    from shared_vf_reference import head64
    A = 17
    c = _model(A, 1)
    sd = P.random_state_dict(c, A, seed=5)
    rng = np.random.default_rng(1)
    n = 40
    emb = rng.standard_normal((n, c['out_features_node']))
    gf = rng.standard_normal((n, c['in_features_graph']))
    mask = (rng.random((n, A)) < 0.6).astype(np.float64)
    logits, value = head64(sd, c, emb, gf, mask)
    w = {k: v.astype(np.float64) for k, v in sd.items()}
    x = np.concatenate([gf, mask], 1)
    mu, var = x.mean(1, keepdims=True), x.var(1, keepdims=True)
    g = ((x - mu) / np.sqrt(var + 1e-5) * w['graph_module.0.weight'] + w['graph_module.0.bias']) @ w['graph_module.1.weight'].T \
        + w['graph_module.1.bias']
    h = np.maximum(np.concatenate([emb, g], 1) @ w['logit_module._hidden_layers.0._model.0.weight'].T
                   + w['logit_module._hidden_layers.0._model.0.bias'], 0)
    want = h @ w['logit_module._value_branch._model.0.weight'][0] + w['logit_module._value_branch._model.0.bias'][0]
    np.testing.assert_allclose(value, want, rtol=1e-13, atol=1e-13)


class _G:
    def __init__(self, n, src, dst, c, rng):
        self.n, self.src, self.dst = n, np.asarray(src, np.int64), np.asarray(dst, np.int64)
        self.nf = rng.standard_normal((n, c['in_features_node']))
        self.ef = rng.standard_normal((len(src), c['in_features_edge']))


def _setup(A=17, n=24, seed=0, shared=1, activation='relu'):
    c = dict(_model(A, shared), fcnet_activation=activation)
    rng = np.random.default_rng(seed)
    gs = [_G(1, [], [], c, rng), _G(4, [0, 1, 1, 2], [1, 2, 3, 3], c, rng), _G(7, [0, 2, 4, 5, 6, 6], [1, 1, 3, 3, 3, 0], c, rng)]
    sd = P.random_state_dict(c, A, seed=seed + 1)
    model = rng.integers(0, len(gs), n)
    gf = rng.standard_normal((n, c['in_features_graph']))
    mask = (rng.random((n, A)) < 0.6).astype(np.float64)
    mask[np.arange(n), rng.integers(0, A, n)] = 1
    return c, A, gs, sd, model, gf, mask, rng


def _module(c, A, sd, gs, model, gf, mask):
    """the module restatement GNNPolicy (RLlib FullyConnectedNetwork with vf_share_layers) in float64: logits, value, parameters"""
    from shared_vf_reference import GNNPolicy
    ref = GNNPolicy(c, A).double()
    assert hasattr(ref.logit_module, '_value_branch_separate') != bool(c.get('vf_share_layers'))
    ref.load_state_dict({k: torch.tensor(np.asarray(v), dtype=torch.float64) for k, v in sd.items()})
    emb = torch.stack([ref.embed(torch.tensor(gs[m].nf), torch.tensor(gs[m].ef), torch.tensor(gs[m].src), torch.tensor(gs[m].dst))
                       for m in model])
    logits, value = ref(emb, torch.tensor(np.concatenate([gf, mask], 1)), torch.tensor(mask))
    return logits, value, dict(ref.named_parameters())


@pytest.mark.parametrize('activation', ['relu', 'tanh'])
def test_head64_equals_the_module_with_shared_value_layers(activation):
    from gnn_reference import embed64
    from shared_vf_reference import head64
    c, A, gs, sd, model, gf, mask, _ = _setup(activation=activation)
    logits, value, named = _module(c, A, sd, gs, model, gf, mask)
    assert not any('_value_branch_separate' in k for k in named) and set(named) == set(sd)
    emb = np.stack([embed64(sd, c, g.nf, g.ef, g.src, g.dst) for g in gs])[model]
    l64, v64 = head64(sd, c, emb, gf, mask)
    valid = mask > 0
    np.testing.assert_allclose(l64[valid], logits.detach().numpy()[valid], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(v64, value.detach().numpy(), rtol=1e-12, atol=1e-12)


def _loss_grads(loss_of, c, A, gs, sd, model, gf, mask):
    """loss_of(logits, value) through policy64 and through the module, both float64: their gradients by key"""
    from ppo_reference import params64
    from shared_vf_reference import policy64
    p = params64(sd)
    logits, value = policy64(p, c, gs, model, gf, mask)
    def grads(loss, params):
        gs_ = torch.autograd.grad(loss, params, allow_unused=True)
        return [torch.zeros_like(x) if d is None else d for x, d in zip(params, gs_)]
    g = dict(zip(p, grads(loss_of(logits, value), list(p.values()))))
    l2, v2, named = _module(c, A, sd, gs, model, gf, mask)
    torch.testing.assert_close(l2, logits, rtol=1e-12, atol=1e-9)
    torch.testing.assert_close(v2, value, rtol=1e-12, atol=1e-12)
    g2 = dict(zip(p, grads(loss_of(l2, v2), [named[k] for k in p])))
    return g, g2


def _check(g, g2):
    for k in g:
        torch.testing.assert_close(g[k], g2[k], rtol=1e-9, atol=1e-12, msg=k)
    hk = 'logit_module._hidden_layers.0._model.0.weight'
    assert g[hk].abs().max() > 0


def test_ppo_loss_gradient_with_shared_value_layers():
    from ddls_b200.learn import PPOConfig
    from ppo_reference import params64, ppo_loss64
    from shared_vf_reference import policy64
    c, A, gs, sd, model, gf, mask, rng = _setup(shared=1)
    logits, _ = policy64(params64(sd, requires_grad=False), c, gs, model, gf, mask)
    old = logits.numpy().copy()
    old[mask > 0] += 0.5 * rng.standard_normal(int((mask > 0).sum()))
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    adv, vt = rng.standard_normal(len(model)), rng.standard_normal(len(model))
    cfg = PPOConfig(vf_clip_param=10.0)
    g, g2 = _loss_grads(lambda l, v: ppo_loss64(l, v, action, old, adv, vt, cfg)[0], c, A, gs, sd, model, gf, mask)
    _check(g, g2)
    # the value loss alone reaches the shared hidden layer (and, with separate branches, it would not)
    cfg0 = PPOConfig(vf_clip_param=10.0, vf_loss_coeff=1.0, entropy_coeff=0.0, kl_coeff=0.0)
    gv, _ = _loss_grads(lambda l, v: ppo_loss64(l.detach(), v, action, old, adv, vt, cfg0)[0], c, A, gs, sd, model, gf, mask)
    assert gv['logit_module._hidden_layers.0._model.0.weight'].abs().max() > 0


def test_impala_loss_gradient_with_shared_value_layers():
    from ddls_b200.learn import IMPALAConfig
    from impala_reference import impala_loss64
    n_frag, L = 6, 4
    c, A, gs, sd, model, gf, mask, rng = _setup(shared=1, n=n_frag * L)
    mrow = model.reshape(n_frag, L).astype(np.int32).copy()
    mrow[1, 2] = -1                                                     # a row without a decision
    batch = dict(model=mrow, action=np.array([rng.choice(np.flatnonzero(m)) for m in mask]).reshape(n_frag, L),
                 behaviour_logp=rng.normal(-1.5, 0.3, (n_frag, L)), reward=rng.standard_normal((n_frag, L)),
                 done=(rng.random((n_frag, L)) < 0.2).astype(np.uint8))
    cfg = IMPALAConfig()
    g, g2 = _loss_grads(lambda l, v: impala_loss64(l, v, batch, cfg)[0], c, A, gs, sd, model, gf, mask)
    _check(g, g2)


def test_pg_loss_gradient_with_shared_value_layers():
    from pg_reference import pg_loss64
    c, A, gs, sd, model, gf, mask, rng = _setup(shared=1)
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    adv = rng.standard_normal(len(model))
    g, g2 = _loss_grads(lambda l, v: pg_loss64(l, action, adv)[0], c, A, gs, sd, model, gf, mask)
    _check(g, g2)
    assert g['logit_module._value_branch._model.0.weight'].abs().max() == 0                 # PG has no value term


def test_fold_of_the_tied_separate_gradient_is_the_shared_gradient():
    """the gradient of the separate-branch form at expand(params), each tensor on its own, folded, equals autograd through the
    tied tensors: what check_explained relies on"""
    from ddls_b200.learn import PPOConfig
    from ppo_reference import params64, policy64, ppo_loss64
    from shared_vf_reference import expand, fold, separate_config
    c, A, gs, sd, model, gf, mask, rng = _setup(shared=1)
    cx = separate_config(c)
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    old = rng.standard_normal(mask.shape)
    adv, vt = rng.standard_normal(len(model)), rng.standard_normal(len(model))
    cfg = PPOConfig(vf_clip_param=10.0)
    px = params64(expand(sd))
    loss = ppo_loss64(*policy64(px, cx, gs, model, gf, mask), action, old, adv, vt, cfg)[0]
    gx = fold({k: g.numpy() for k, g in zip(px, torch.autograd.grad(loss, list(px.values())))})
    p = params64(sd)
    loss = ppo_loss64(*policy64(expand(p), cx, gs, model, gf, mask), action, old, adv, vt, cfg)[0]
    g = {k: v.numpy() for k, v in zip(p, torch.autograd.grad(loss, list(p.values())))}
    assert set(gx) == set(g)
    for k in g:
        np.testing.assert_allclose(gx[k], g[k], rtol=1e-12, atol=1e-14, err_msg=k)
