"""CPU: the float64 restatements the PPO learner is tested against (tests/ppo_reference.py), and the rules its kernels apply
(ddls_b200/csrc/ramp_policy_learn.cuh), pinned to torch:

- policy64's gradient of the PPO loss equals torch.autograd through the module restatement GNNPolicy (tests/gnn_reference.py) run
  in float64;
- the head-gradient kernel's closed form of d loss / d logits and d loss / d value equals autograd of ppo_loss64;
- the Adam kernel's update rule equals torch.optim.Adam + clip_grad_norm_;
- gae64 equals RLlib's discount_cumsum formulation episode by episode;
- state_dict() / pack_weights round-trip;
- the learn-call replay: shuffle_order is a permutation, one pass of one minibatch is adam_step on ppo_loss64's gradient, a short
  last minibatch is a mean over its own rows, the float64 and float32 replays agree to fp32 rounding, update_kl's branches."""
import numpy as np
import pytest
import torch

from ddls_b200 import policy as P
from ddls_b200.learn import PPOConfig


class _G:
    def __init__(self, n, src, dst, c, rng):
        self.n, self.src, self.dst = n, np.asarray(src, np.int64), np.asarray(dst, np.int64)
        self.nf = rng.standard_normal((n, c['in_features_node']))
        self.ef = rng.standard_normal((len(src), c['in_features_edge']))


def _setup(config=None, A=9, n=24, seed=0):
    c = dict(P.DEFAULT_CONFIG)
    c.update(config or {})
    rng = np.random.default_rng(seed)
    gs = [_G(1, [], [], c, rng), _G(4, [0, 1, 1, 2], [1, 2, 3, 3], c, rng), _G(7, [0, 2, 4, 5, 6, 6], [1, 1, 3, 3, 3, 0], c, rng)]
    sd = P.random_state_dict(c, A, seed=seed + 1)
    model = rng.integers(0, len(gs), n)
    gf = rng.standard_normal((n, c['in_features_graph']))
    mask = (rng.random((n, A)) < 0.6).astype(np.float64)
    mask[np.arange(n), rng.integers(0, A, n)] = 1
    return c, A, gs, sd, model, gf, mask, rng


def _batch(rng, logits, mask, noise=0.5):
    n, A = mask.shape
    old = logits.detach().numpy().copy()
    old[mask > 0] += noise * rng.standard_normal(int((mask > 0).sum()))
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    return old, action, rng.standard_normal(n), rng.standard_normal(n)


@pytest.mark.parametrize('config', [{}, dict(num_rounds=3, aggregator_activation='leaky_relu', fcnet_activation='tanh')])
def test_policy64_gradient_equals_autograd_on_gnn_policy(config):
    from gnn_reference import GNNPolicy
    from ppo_reference import params64, policy64, ppo_loss64
    c, A, gs, sd, model, gf, mask, rng = _setup(config)
    p = params64(sd)
    logits, value = policy64(p, c, gs, model, gf, mask)
    old, action, adv, vt = _batch(rng, logits, mask)
    cfg = PPOConfig(vf_clip_param=1.0)
    loss, _ = ppo_loss64(logits, value, action, old, adv, vt, cfg)
    g = torch.autograd.grad(loss, list(p.values()))
    ref = GNNPolicy(c, A).double()
    ref.load_state_dict({k: torch.tensor(np.asarray(v), dtype=torch.float64) for k, v in sd.items()})
    emb = torch.stack([ref.embed(torch.tensor(gs[m].nf), torch.tensor(gs[m].ef), torch.tensor(gs[m].src), torch.tensor(gs[m].dst))
                       for m in model])
    l2, v2 = ref(emb, torch.tensor(np.concatenate([gf, mask], 1)), torch.tensor(mask))
    torch.testing.assert_close(l2, logits, rtol=1e-12, atol=1e-9)
    loss2, _ = ppo_loss64(l2, v2, action, old, adv, vt, cfg)
    g2 = torch.autograd.grad(loss2, [dict(ref.named_parameters())[k] for k in p])
    for k, a, b in zip(p, g, g2):
        torch.testing.assert_close(a, b, rtol=1e-9, atol=1e-12, msg=k)


def kernel_upstream(logits, value, action, old, adv, vt, cfg):
    """d loss / d logits and d loss / d value as ramp_policy_head_grad_kernel forms them, in float64"""
    n = len(value)

    def log_softmax(x):
        x = x - x.max(1, keepdims=True)
        return x - np.log(np.exp(x).sum(1, keepdims=True))
    lp, olp = log_softmax(logits), log_softmax(old)
    pr, oq = np.exp(lp), np.exp(olp)
    rows = np.arange(n)
    ratio = np.exp(lp[rows, action] - olp[rows, action])
    s1, s2 = adv * ratio, adv * np.clip(ratio, 1 - cfg.clip_param, 1 + cfg.clip_param)
    gs = np.where(s2 < s1, 0.0, adv * ratio)
    ent = -np.where(pr > 0, pr * lp, 0).sum(1)
    onehot = np.zeros_like(pr)
    onehot[rows, action] = 1
    dl = (-gs[:, None] * (onehot - pr) + cfg.entropy_coeff * pr * (lp + ent[:, None]) + cfg.kl_coeff * (pr - oq)) / n
    d = value - vt
    dv = np.where(d * d <= cfg.vf_clip_param, cfg.vf_loss_coeff * 2 * d, 0.0) / n
    return dl, dv


@pytest.mark.parametrize('noise', [0.0, 0.5])
def test_kernel_upstream_gradient_equals_autograd(noise):
    from ppo_reference import ppo_loss64
    rng = np.random.default_rng(3)
    n, A = 40, 9
    mask = (rng.random((n, A)) < 0.6)
    mask[np.arange(n), rng.integers(0, A, n)] = True
    raw = rng.standard_normal((n, A))
    logits = torch.tensor(raw + np.where(mask, 0.0, float(np.finfo(np.float32).min)), requires_grad=True)
    value = torch.tensor(rng.standard_normal(n), requires_grad=True)
    old = logits.detach().numpy().copy()
    old[mask] += noise * rng.standard_normal(int(mask.sum()))
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    adv, vt = rng.standard_normal(n), value.detach().numpy() + rng.standard_normal(n)
    cfg = PPOConfig(vf_clip_param=0.8)
    loss, stats = ppo_loss64(logits, value, action, old, adv, vt, cfg)
    gl, gv = torch.autograd.grad(loss, [logits, value])
    dl, dv = kernel_upstream(logits.detach().numpy(), value.detach().numpy(), action, old, adv, vt, cfg)
    np.testing.assert_allclose(dl, gl.numpy(), rtol=1e-9, atol=1e-13)
    np.testing.assert_allclose(dv, gv.numpy(), rtol=1e-9, atol=1e-13)
    assert (dl[~mask] == 0).all()                                       # masked actions: exactly 0, never NaN
    assert (stats['clip_frac'] > 0) == (noise > 0)


@pytest.mark.parametrize('grad_clip', [0.05, 0.0, 100.0])
def test_adam_rule_equals_torch(grad_clip):
    from ppo_reference import adam_step
    rng = np.random.default_rng(1)
    cfg = PPOConfig(grad_clip=grad_clip)
    w, m, v = rng.standard_normal(500).astype(np.float32), None, None
    for step in range(3):
        g = rng.standard_normal(500).astype(np.float32)
        norm = float(np.sqrt((g.astype(np.float64) ** 2).sum()))
        coef = np.float32(min(1.0, grad_clip / (norm + 1e-6))) if grad_clip > 0 else np.float32(1)
        gc = g * coef
        m0 = np.zeros_like(w) if m is None else m
        v0 = np.zeros_like(w) if v is None else v
        mm = m0 + np.float32(1 - cfg.adam_beta1) * (gc - m0)
        vv = v0 * np.float32(cfg.adam_beta2) + np.float32(1 - cfg.adam_beta2) * gc * gc
        t = step + 1
        step_size = np.float32(cfg.lr / (1 - cfg.adam_beta1 ** t))
        bc2 = np.float32(np.sqrt(1 - cfg.adam_beta2 ** t))
        mine = w - step_size * (mm / (np.sqrt(vv) / bc2 + np.float32(cfg.adam_eps)))
        want, m, v, tnorm = adam_step(w, g, m, v, step, cfg)
        np.testing.assert_allclose(mine, want, rtol=1e-6, atol=1e-9)
        scale = float(np.abs(gc).max())                                 # where (g - m) cancels, a few ulps of the gradient
        np.testing.assert_allclose(mm, m, rtol=1e-6, atol=1e-7 * scale)
        np.testing.assert_allclose(vv, v, rtol=1e-6, atol=1e-7 * scale * scale)
        assert abs(tnorm - norm) <= 1e-5 * norm
        w = want


def test_gae_equals_discount_cumsum_per_episode():
    from scipy.signal import lfilter
    from ppo_reference import gae64, standardize64
    rng = np.random.default_rng(7)
    T, B, gamma, lam = 9, 6, 0.997, 0.95
    done = np.zeros((T, B), bool)
    for b, t in enumerate([8, 3, 0, -1, 5, -1]):                      # -1: the segment ends before the episode does
        if t >= 0:
            done[t:, b] = True                                          # a finished episode stays done
    reward, value, boot = rng.standard_normal((T, B)), rng.standard_normal((T, B)), rng.standard_normal(B)
    model = np.zeros((T, B), int)
    adv, vt, rows = gae64(reward, value, done, model, boot, gamma, lam, 1)
    want = np.zeros((T, B))
    for b in range(B):
        end = int(np.flatnonzero(done[:, b])[0]) + 1 if done[:, b].any() else T
        last_r = 0.0 if done[:, b].any() else boot[b]
        vpred = np.concatenate([value[:end, b], [last_r]])
        delta = reward[:end, b] + gamma * vpred[1:] - vpred[:-1]
        want[:end, b] = lfilter([1], [1, -gamma * lam], delta[::-1])[::-1]          # RLlib discount_cumsum
        assert rows[:end, b].all() and not rows[end:, b].any()
    np.testing.assert_allclose(adv, want[rows], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(vt, (want + value)[rows], rtol=1e-12, atol=1e-12)
    s = standardize64(adv)
    assert abs(s.mean()) < 1e-12 and abs(s.std() - 1) < 1e-12


def test_state_dict_round_trip():
    for config, A in (({}, 17), (dict(num_rounds=3, fcnet_hiddens=(64,), out_features_msg=10), 5)):
        c = dict(P.DEFAULT_CONFIG)
        c.update(config)
        sd = P.random_state_dict(c, A, seed=9)
        blob = P.pack_weights(sd, c, A)
        back = P.unpack_weights(blob, c, A)
        assert list(back) == list(P.weight_keys(c))
        for k in sd:
            np.testing.assert_array_equal(back[k], sd[k])
        np.testing.assert_array_equal(P.pack_weights(back, c, A), blob)
    with pytest.raises(ValueError):
        P.unpack_weights(blob[:-1], c, A)


@pytest.mark.parametrize('seed', [0, 2 ** 64 - 1])
def test_shuffle_order_is_a_permutation(seed):
    from ppo_reference import shuffle_order
    for n in range(1, 2101):
        orders = [shuffle_order(seed, p, n) for p in (0, 1)]
        for o in orders:
            assert o.dtype == np.int64 and len(o) == n
            np.testing.assert_array_equal(np.sort(o), np.arange(n), err_msg=f'n={n}')
        if n >= 4:                                                      # 3! = 6 orders: two passes may meet below that
            assert (orders[0] != orders[1]).any(), n
    assert (shuffle_order(seed, 2, 2100) != shuffle_order(seed ^ 1, 2, 2100)).any()


def _replay_setup(n=24, seed=0):
    """a GNNPolicy-sized problem on three small graphs (one of one node): rows with collection-like old logits"""
    from ppo_reference import params64, policy64
    c, A, gs, sd, model, gf, mask, rng = _setup(n=n, seed=seed)
    with torch.no_grad():
        logits, value = policy64(params64(sd, requires_grad=False), c, gs, model, gf, mask)
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    batch = dict(model=model, graph_features=gf, action_mask=mask, action=action, advantage=rng.standard_normal(n),
                 value_target=value.numpy() + rng.standard_normal(n))
    return c, A, gs, sd, batch


def _flat(d):
    return np.concatenate([np.asarray(v, np.float64).ravel() for v in d.values()])


@pytest.mark.parametrize('dtype', [torch.float64, torch.float32])
def test_replay_of_one_minibatch_is_one_adam_step(dtype):
    """one pass of one minibatch holding the batch: the replay's step is adam_step on ppo_loss64's autograd gradient at the
    starting weights, whose old logits are the current ones (ratio 1, KL 0)"""
    from ppo_reference import adam_step, learn_replay, params64, policy64, ppo_loss64
    c, A, gs, sd, b = _replay_setup()
    n = len(b['model'])
    cfg = PPOConfig(num_sgd_iter=1, sgd_minibatch_size=n, grad_clip=0.05, vf_clip_param=1.0, seed=3)
    out = learn_replay(sd, c, gs, b, cfg, dtype=dtype)
    p = params64(sd, dtype=dtype)
    logits, value = policy64(p, c, gs, b['model'], b['graph_features'], b['action_mask'])
    loss, want = ppo_loss64(logits, value, b['action'], logits.detach(), b['advantage'], b['value_target'], cfg)
    g = torch.cat([x.reshape(-1) for x in torch.autograd.grad(loss, list(p.values()))]).numpy()
    npdt = np.float64 if dtype == torch.float64 else np.float32
    w, m, v, norm = adam_step(_flat(sd).astype(npdt), g, None, None, 0, cfg)
    assert norm > cfg.grad_clip                                         # clipped
    rtol = 1e-10 if dtype == torch.float64 else 1e-5                  # the replay sums its rows in shuffled order
    np.testing.assert_allclose(_flat(out['weights']), w, rtol=rtol, atol=rtol * np.abs(w).max())
    np.testing.assert_allclose(out['m'], m, rtol=rtol, atol=rtol * np.abs(m).max())
    assert out['step'] == 1 and out['minibatches'][0][0]['rows'] == n
    st = out['stats']
    assert st['kl'] == pytest.approx(0.0, abs=1e-6) and st['clip_frac'] == 0.0
    for k in ('total_loss', 'policy_loss', 'vf_loss', 'entropy'):
        assert st[k] == pytest.approx(want[k], rel=rtol, abs=rtol), k
    assert st['grad_gnorm'] == pytest.approx(norm, rel=rtol)
    assert out['kl_coeff'] == cfg.kl_coeff * 0.5                      # KL 0 < kl_target / 2


def test_replay_short_last_minibatch_is_a_mean_over_its_rows():
    """24 rows in slices of 10: 10, 10 and a last slice of 4, whose loss is the mean over its 4 rows.  lr 0 keeps the weights,
    so every slice's statistics are ppo_loss64's on its rows at the starting weights; Adam's moments still take each slice's
    gradient, so the last step's m, v are the short slice's mean gradient"""
    import dataclasses
    from ppo_reference import adam_step, learn_replay, params64, policy64, ppo_loss64, shuffle_order
    c, A, gs, sd, b = _replay_setup()
    n, mb = len(b['model']), 10
    cfg = PPOConfig(num_sgd_iter=2, sgd_minibatch_size=mb, lr=0.0, vf_clip_param=1.0, seed=11)
    out = learn_replay(sd, c, gs, b, cfg)
    assert [[s['rows'] for s in ps] for ps in out['minibatches']] == [[10, 10, 4]] * 2 and out['step'] == 6
    np.testing.assert_array_equal(_flat(out['weights']), _flat(sd))
    p = params64(sd)
    with torch.no_grad():
        old, _ = policy64(p, c, gs, b['model'], b['graph_features'], b['action_mask'])
    w, m, v, step = _flat(sd), None, None, 0
    for ps in range(2):
        order = shuffle_order(cfg.seed, ps, n)
        for k, s in enumerate(range(0, n, mb)):
            idx = order[s:s + mb]
            pk = params64(sd)
            logits, value = policy64(pk, c, gs, b['model'][idx], b['graph_features'][idx], b['action_mask'][idx])
            loss, want = ppo_loss64(logits, value, b['action'][idx], old[torch.as_tensor(idx)], b['advantage'][idx],
                                    b['value_target'][idx], cfg)
            got = out['minibatches'][ps][k]
            for key in ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'kl', 'clip_frac'):
                assert got[key] == pytest.approx(want[key], rel=1e-12, abs=1e-14), (ps, k, key)
            g = torch.cat([x.reshape(-1) for x in torch.autograd.grad(loss, list(pk.values()))]).numpy()
            w, m, v, _ = adam_step(w, g, m, v, step, cfg)
            step += 1
    np.testing.assert_allclose(out['m'], m, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(out['v'], v, rtol=1e-12, atol=1e-20)
    # the short slice's gradient is its sum over 4 rows / 4: divided by mb it would be 0.4 of it
    short = order[20:]
    wrong = ppo_loss64(*policy64(params64(sd), c, gs, b['model'][short], b['graph_features'][short], b['action_mask'][short]),
                       b['action'][short], old[torch.as_tensor(short)], b['advantage'][short], b['value_target'][short], cfg)[1]
    assert out['minibatches'][1][2]['total_loss'] == pytest.approx(wrong['total_loss'], rel=1e-12)
    assert abs(out['minibatches'][1][2]['total_loss'] * 4 / mb - wrong['total_loss']) > 1e-3 * abs(wrong['total_loss'])
    # the mean over the last pass is over its three slices, not weighted by rows
    assert out['stats']['total_loss'] == pytest.approx(np.mean([s['total_loss'] for s in out['minibatches'][1]]), rel=1e-14)
    cfg2 = dataclasses.replace(cfg, lr=1e-3)
    assert out['step'] == learn_replay(sd, c, gs, b, cfg2)['step']


def test_replay_float64_and_float32_agree_to_fp32_rounding():
    """three passes over 30 rows in slices of 7 (the last of 2), clipping and value clipping on: per weight tensor the float32
    replay's net update is within 1e-4 of the float64 one's, plus the rounding of the fp32 weights that hold it (two ulps per
    element; on a LayerNorm gain near 1 an update of 1e-3 is only some 10^4 ulps)"""
    from ppo_reference import learn_replay
    c, A, gs, sd, b = _replay_setup(n=30, seed=4)
    cfg = PPOConfig(num_sgd_iter=3, sgd_minibatch_size=7, grad_clip=0.5, vf_clip_param=1.0, lr=1e-3, seed=2)
    r64, r32 = learn_replay(sd, c, gs, b, cfg), learn_replay(sd, c, gs, b, cfg, dtype=torch.float32)
    assert r64['step'] == r32['step'] == 15
    assert [s['rows'] for s in r64['minibatches'][0]] == [7, 7, 7, 7, 2]
    worst, bad = (0.0, None), {}
    for k, w0 in sd.items():
        d64 = r64['weights'][k] - np.asarray(w0, np.float64)
        d32 = r32['weights'][k].astype(np.float64) - np.asarray(w0, np.float64)
        nrm, err = np.linalg.norm(d64), np.linalg.norm(d32 - d64)
        assert nrm > 0, k
        worst = max(worst, (err / nrm, k))
        if err > 1e-4 * nrm + 2 * np.linalg.norm(np.spacing(r32['weights'][k])):
            bad[k] = err / nrm
    print(f'float32 replay: largest relative error of a net update {worst[0]:.2e} ({worst[1]})')
    assert not bad, bad
    for k in ('total_loss', 'kl', 'entropy'):
        assert r32['stats'][k] == pytest.approx(r64['stats'][k], rel=1e-4, abs=1e-7), k


def test_update_kl_branches():
    """x1.5 strictly above twice the target, x0.5 strictly below half of it, unchanged between and at both edges"""
    from ppo_reference import update_kl
    t, c = 0.01, 0.2
    assert update_kl(c, np.nextafter(2 * t, 1), t) == c * 1.5
    assert update_kl(c, 2 * t, t) == c
    assert update_kl(c, t, t) == c
    assert update_kl(c, 0.5 * t, t) == c
    assert update_kl(c, np.nextafter(0.5 * t, 0), t) == c * 0.5
    assert update_kl(c, 0.0, t) == c * 0.5
