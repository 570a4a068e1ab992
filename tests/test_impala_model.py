"""CPU: the IMPALA restatement (tests/impala_reference.py) pinned on its own -- V-trace against GAE and a hand-computed case,
clipping, done cuts, the fragment and batch layout, and the loss's gradient in the form the head-gradient kernel computes."""
import dataclasses

import numpy as np
import pytest
import torch

from impala_reference import fragments, impala_loss64, train_batches, vtrace64
from ppo_reference import gae64


@dataclasses.dataclass
class Cfg:
    gamma: float = 0.99
    vtrace_clip_rho_threshold: float = 1.0
    vtrace_clip_pg_rho_threshold: float = 1.0
    vf_loss_coeff: float = 0.5
    entropy_coeff: float = 0.01


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def _segment(T, B, seed):
    """a recorded segment with episodes that end at random steps (done stays set, nothing queued after it) and rows with nothing queued"""
    rng = np.random.default_rng(seed)
    end = rng.integers(1, T + 3, B)
    t = np.arange(T)[:, None]
    done = t >= end[None, :] - 1
    alive = np.concatenate([np.ones((1, B), bool), ~done[:-1]], 0)
    model = np.where(alive & (rng.random((T, B)) > 0.1), 0, -1)
    value = np.where(model >= 0, rng.standard_normal((T, B)), 0.0)
    reward = rng.standard_normal((T, B))
    return reward, value, done, model


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_on_policy_vtrace_is_gae_with_lambda_one(seed):
    """log rho = 0 and thresholds >= 1: vs - V equals GAE(lambda = 1) on rows 0 .. L-2, bootstrapped with V_{L-1}"""
    L, B, gamma = 7, 40, 0.97
    reward, value, done, model = _segment(L, B, seed)
    vs, pg = vtrace64(_t(np.zeros((L - 1, B))), _t((1.0 - done[:-1]) * gamma), _t(reward[:-1]), _t(value[:-1]), _t(value[-1]),
                      1.0, 1.0)
    adv, _, rows = gae64(reward[:-1], value[:-1], done[:-1], model[:-1], value[-1], gamma, 1.0, 1)
    np.testing.assert_allclose((vs.numpy() - value[:-1])[rows], adv, rtol=1e-12, atol=1e-12)
    # on-policy pg_adv is r + gamma' vs_{t+1} - V = vs_t - V_t (c = 1 makes the recursion GAE's)
    np.testing.assert_allclose(pg.numpy()[rows], adv, rtol=1e-12, atol=1e-12)


def test_three_steps_by_hand():
    r, V, boot, g = [1.0, 0.0, 2.0], [0.5, -1.0, 0.25], 3.0, 0.5
    rho = [2.0, 0.5, 1.5]
    vs, pg = vtrace64(_t(np.log(rho))[:, None], _t([g, g, g])[:, None], _t(r)[:, None], _t(V)[:, None], _t([boot]), 1.0, 1.0)
    # clip 1: rho-bar = c = min(rho, 1) = 1, 0.5, 1
    d2 = 1.0 * (2.0 + 0.5 * 3.0 - 0.25)                     # 3.25
    a2 = d2
    d1 = 0.5 * (0.0 + 0.5 * 0.25 - (-1.0))                  # 0.5625
    a1 = d1 + 0.5 * 0.5 * a2                                # 1.375
    d0 = 1.0 * (1.0 + 0.5 * -1.0 - 0.5)                     # 0
    a0 = d0 + 0.5 * 1.0 * a1                                # 0.6875
    want_vs = [0.5 + a0, -1.0 + a1, 0.25 + a2]
    np.testing.assert_allclose(vs.numpy()[:, 0], want_vs, rtol=0, atol=1e-15)
    want_pg = [1.0 * (1.0 + 0.5 * want_vs[1] - 0.5), 0.5 * (0.0 + 0.5 * want_vs[2] + 1.0), 1.0 * (2.0 + 0.5 * boot - 0.25)]
    np.testing.assert_allclose(pg.numpy()[:, 0], want_pg, rtol=0, atol=1e-15)


def test_clipping_thresholds():
    """rho above each threshold is clipped to it; c stays capped at 1 when clip_rho > 1"""
    rng = np.random.default_rng(3)
    T, B = 6, 30
    log_rho = rng.normal(0.0, 1.0, (T, B))
    disc = np.full((T, B), 0.9)
    r, V, boot = rng.standard_normal((T, B)), rng.standard_normal((T, B)), rng.standard_normal(B)
    for cr, cp in ((1.0, 1.0), (2.0, 0.5), (0.7, 3.0)):
        vs, pg = vtrace64(_t(log_rho), _t(disc), _t(r), _t(V), _t(boot), cr, cp)
        rho = np.exp(log_rho)
        rb, c, rp = np.minimum(rho, cr), np.minimum(rho, 1.0), np.minimum(rho, cp)
        v1 = np.concatenate([V[1:], boot[None]])
        acc, want = np.zeros(B), np.zeros((T, B))
        for t in range(T - 1, -1, -1):
            acc = rb[t] * (r[t] + disc[t] * v1[t] - V[t]) + disc[t] * c[t] * acc
            want[t] = V[t] + acc
        np.testing.assert_allclose(vs.numpy(), want, rtol=1e-12, atol=1e-12)
        vs1 = np.concatenate([want[1:], boot[None]])
        np.testing.assert_allclose(pg.numpy(), rp * (r + disc * vs1 - V), rtol=1e-12, atol=1e-12)
        assert (rho > max(cr, cp, 1.0)).any() and (rho < min(cr, cp, 1.0)).any()
    # c capped at 1: with clip_rho 2 the result differs from c = min(rho, 2)
    vs2, _ = vtrace64(_t(log_rho), _t(disc), _t(r), _t(V), _t(boot), 2.0, 1.0)
    rho = np.exp(log_rho)
    acc, bad = np.zeros(B), np.zeros((T, B))
    v1 = np.concatenate([V[1:], boot[None]])
    for t in range(T - 1, -1, -1):
        acc = np.minimum(rho[t], 2.0) * (r[t] + disc[t] * v1[t] - V[t]) + disc[t] * np.minimum(rho[t], 2.0) * acc
        bad[t] = V[t] + acc
    assert np.abs(vs2.numpy() - bad).max() > 1e-3


def test_a_done_row_cuts_the_recursion():
    rng = np.random.default_rng(4)
    T = 8
    r, V, lr = rng.standard_normal(T), rng.standard_normal(T), rng.normal(0, 0.3, T)
    disc = np.full(T, 0.95)
    disc[3] = 0.0                                                          # done at t = 3
    args = [_t(lr)[:, None], _t(disc)[:, None], _t(r)[:, None], _t(V)[:, None]]
    vs, pg = vtrace64(*args, _t([0.7]))
    r2, V2 = r.copy(), V.copy()
    r2[4:] += 5.0
    V2[4:] -= 3.0
    vs2, pg2 = vtrace64(args[0], args[1], _t(r2)[:, None], _t(V2)[:, None], _t([-9.0]))
    np.testing.assert_array_equal(vs.numpy()[:4], vs2.numpy()[:4])
    np.testing.assert_array_equal(pg.numpy()[:4], pg2.numpy()[:4])
    assert vs.numpy()[3, 0] == V[3] + min(np.exp(lr[3]), 1.0) * (r[3] - V[3])


def _traj(T, B, A=3, seed=0):
    rng = np.random.default_rng(seed)
    reward, value, done, model = _segment(T, B, seed)
    live = np.concatenate([np.ones((1, B), bool), ~done[:-1]], 0) & (model >= 0)
    return dict(model=model.astype(np.int32), live=live, graph_features_dynamic=rng.standard_normal((T, B, 11)).astype(np.float32),
                action_mask=np.ones((T, B, A), np.uint8), action=rng.integers(0, A, (T, B)).astype(np.int32),
                logp=rng.standard_normal((T, B)).astype(np.float32), reward=reward, done=done)


@pytest.mark.parametrize('T,L', [(8, 8), (8, 2), (12, 4), (6, 1)])
def test_fragment_layout(T, L):
    B = 5
    tr = _traj(T, B)
    static = [np.arange(6, dtype=np.float32)]
    fr = fragments(tr, static, 1, L)
    assert fr['model'].shape == (T // L * B, L)
    for f in range(T // L * B):
        j, b = divmod(f, B)
        for t in range(L):
            s = j * L + t
            assert fr['reward'][f, t] == tr['reward'][s, b] and fr['action'][f, t] == tr['action'][s, b]
            assert fr['model'][f, t] == (tr['model'][s, b] if tr['live'][s, b] else -1)
            np.testing.assert_array_equal(fr['graph_features'][f, t, :9], tr['graph_features_dynamic'][s, b, :9])
            np.testing.assert_array_equal(fr['graph_features'][f, t, 9:15], static[0])


def test_train_batches():
    assert train_batches(64, 8, 200) == [(0, 25), (25, 50), (50, 64)]          # a short last batch
    assert train_batches(10, 16, 20) == [(k, k + 1) for k in range(10)]         # F = 1
    assert train_batches(6, 4, 400) == [(0, 6)]                                 # one batch holds every fragment
    assert train_batches(1024, 16, 200) == [(k, min(k + 12, 1024)) for k in range(0, 1024, 12)]
    assert len(train_batches(1024, 16, 200)) == 86


def test_loss_gradient_is_the_kernel_form():
    """d total / d logits = -pg_adv (onehot(a) - p) + ent_coeff p (log p + H) and d total / d V = vf_coeff (V - vs) on loss rows,
    0 on row L-1 and on rows without decision; the mean-entropy statistic is over the loss rows"""
    rng = np.random.default_rng(6)
    n, L, A = 5, 4, 6
    cfg = Cfg(vtrace_clip_rho_threshold=1.3, vtrace_clip_pg_rho_threshold=0.8)
    model = np.zeros((n, L), np.int32)
    model[1, 2] = model[3, 0] = -1
    batch = dict(model=model, action=rng.integers(0, A, (n, L)), behaviour_logp=rng.normal(-1.5, 0.3, (n, L)),
                 reward=rng.standard_normal((n, L)), done=(rng.random((n, L)) < 0.2).astype(np.uint8))
    logits = torch.tensor(rng.standard_normal((n * L, A)), requires_grad=True)
    value = torch.tensor(rng.standard_normal(n * L), requires_grad=True)
    total, st, out = impala_loss64(logits, value, batch, cfg)
    gl, gv = torch.autograd.grad(total, [logits, value])
    p = torch.softmax(logits, 1).detach().numpy()
    lp = np.log(p)
    H = -(p * lp).sum(1)
    a = batch['action'].reshape(-1)
    valid = ((model >= 0) & (np.arange(L)[None, :] < L - 1)).reshape(-1)
    pga, vs = out['pg_advantages'].reshape(-1), out['vs'].reshape(-1)
    onehot = np.eye(A)[a]
    want_l = (-pga[:, None] * (onehot - p) + cfg.entropy_coeff * p * (lp + H[:, None])) * valid[:, None]
    want_v = cfg.vf_loss_coeff * (value.detach().numpy() - vs) * valid
    np.testing.assert_allclose(gl.numpy(), want_l, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(gv.numpy(), want_v, rtol=1e-12, atol=1e-14)
    assert st['rows'] == valid.sum()
    assert abs(st['entropy'] - H[valid].mean()) < 1e-12
    np.testing.assert_array_equal(out['log_rho'].reshape(-1)[model.reshape(-1) < 0], 0.0)
