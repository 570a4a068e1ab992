"""CPU: the PG restatement (tests/pg_reference.py) pinned on its own -- the discounted returns against scipy's lfilter per episode
and against GAE with lambda 1 and no values, the loss's gradient against autograd through the module restatement GNNPolicy
(tests/gnn_reference.py) and in the form the head-gradient kernel computes it, and one Adam step against torch.optim.Adam."""
import numpy as np
import pytest
import torch
from scipy.signal import lfilter

from ddls_b200 import policy as P
from ddls_b200.learn import PGConfig


def _segment(T, B, seed):
    """a recorded segment: episodes end at random steps, some after the segment does (truncated), rows with nothing queued"""
    rng = np.random.default_rng(seed)
    end = rng.integers(1, T + 3, B)
    t = np.arange(T)[:, None]
    done = t == end[None, :] - 1
    done = np.cumsum(done, 0) > 0                                       # done stays set after the episode ends
    alive = np.concatenate([np.ones((1, B), bool), ~done[:-1]], 0)
    model = np.where(alive & (rng.random((T, B)) > 0.1), 0, -1)
    reward = rng.standard_normal((T, B))
    return reward, done, model, end


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_returns_are_lfilter_per_episode(seed):
    from pg_reference import discounted_returns
    T, B, gamma = 9, 12, 0.99
    reward, done, model, end = _segment(T, B, seed)
    assert (end > T).any() and (end <= T).any()                        # truncated and finished episodes
    adv, adv64, rows = discounted_returns(reward, done, model, gamma, 1)
    want = np.zeros((T, B))
    for b in range(B):
        n = min(int(end[b]), T)                                         # the trajectory: up to its done, or the segment's end
        y = lfilter([1.0], [1.0, -gamma], np.append(reward[:n, b], 0.0)[::-1])[::-1][:-1]
        want[:n, b] = y
        if end[b] > T:                                                  # last_r 0: a truncated episode's last return is its reward
            assert y[-1] == reward[n - 1, b]
    np.testing.assert_array_equal(adv64, want[rows])
    np.testing.assert_array_equal(adv, want[rows].astype(np.float32))
    assert not rows[~np.concatenate([np.ones((1, B), bool), ~done[:-1]], 0)].any()   # rows after done are out of the batch
    assert not rows[model < 0].any()


def test_returns_hand_computed():
    from pg_reference import discounted_returns
    reward = np.array([[1.0], [2.0], [3.0], [5.0]])
    done = np.array([[0], [1], [1], [1]], bool)                        # the episode ends at t = 1; t = 2, 3 are dead rows
    adv, _, rows = discounted_returns(reward, done, np.zeros((4, 1), int), 0.5, 1)
    np.testing.assert_array_equal(rows[:, 0], [True, True, False, False])
    np.testing.assert_array_equal(adv, [1.0 + 0.5 * 2.0, 2.0])
    adv, _, _ = discounted_returns(reward, np.zeros((4, 1), bool), np.zeros((4, 1), int), 0.5, 1)
    np.testing.assert_array_equal(adv, [1 + 0.5 * (2 + 0.5 * (3 + 0.5 * 5)), 2 + 0.5 * (3 + 0.5 * 5), 3 + 0.5 * 5, 5.0])


@pytest.mark.parametrize('seed', [3, 4])
def test_returns_equal_gae_without_values_bit_for_bit(seed):
    """the device computes the returns with ramp_ppo_gae_kernel's recursion, lambda 1, V = 0 and a 0 bootstrap: gae64 restates that
    recursion and must give lfilter's bits"""
    from pg_reference import discounted_returns
    from ppo_reference import gae64
    T, B, gamma = 11, 16, 0.99
    reward, done, model, _ = _segment(T, B, seed)
    _, adv64, rows = discounted_returns(reward, done, model, gamma, 1)
    g, vt, grows = gae64(reward, np.zeros((T, B)), done, model, np.zeros(B), gamma, 1.0, 1)
    np.testing.assert_array_equal(grows, rows)
    np.testing.assert_array_equal(g, adv64)
    np.testing.assert_array_equal(vt, adv64)


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
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    return c, A, gs, sd, model, gf, mask, action, rng.standard_normal(n)


@pytest.mark.parametrize('config', [{}, dict(num_rounds=3, aggregator_activation='leaky_relu', fcnet_activation='tanh')])
def test_loss_gradient_equals_autograd_on_gnn_policy(config):
    from gnn_reference import GNNPolicy
    from pg_reference import pg_loss64
    from ppo_reference import params64, policy64
    c, A, gs, sd, model, gf, mask, action, adv = _setup(config)
    p = params64(sd)
    logits, _ = policy64(p, c, gs, model, gf, mask)
    loss, _ = pg_loss64(logits, action, adv)
    g = torch.autograd.grad(loss, list(p.values()), allow_unused=True)
    ref = GNNPolicy(c, A).double()
    ref.load_state_dict({k: torch.tensor(np.asarray(v), dtype=torch.float64) for k, v in sd.items()})
    emb = torch.stack([ref.embed(torch.tensor(gs[m].nf), torch.tensor(gs[m].ef), torch.tensor(gs[m].src), torch.tensor(gs[m].dst))
                       for m in model])
    l2, _ = ref(emb, torch.tensor(np.concatenate([gf, mask], 1)), torch.tensor(mask))
    loss2, _ = pg_loss64(l2, action, adv)
    torch.testing.assert_close(loss2, loss, rtol=1e-12, atol=1e-12)
    params = dict(ref.named_parameters())
    g2 = torch.autograd.grad(loss2, [params[k] for k in p], allow_unused=True)
    for k, a, b in zip(p, g, g2):
        if a is None or b is None:                                      # the value branch: no gradient from PG's loss
            assert a is None and b is None, k
            assert 'value_branch' in k, k
            continue
        torch.testing.assert_close(a, b, rtol=1e-9, atol=1e-12, msg=k)


def test_kernel_upstream_gradient_equals_autograd():
    """the head-gradient kernel's PG mode: d logits = -(adv / n) (onehot(a) - softmax), exactly 0 on masked actions"""
    from pg_reference import pg_loss64
    rng = np.random.default_rng(3)
    n, A = 40, 9
    mask = rng.random((n, A)) < 0.6
    mask[np.arange(n), rng.integers(0, A, n)] = True
    logits = torch.tensor(rng.standard_normal((n, A)) + np.where(mask, 0.0, float(np.finfo(np.float32).min)), requires_grad=True)
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask])
    adv = rng.standard_normal(n)
    loss, stats = pg_loss64(logits, action, adv)
    gl, = torch.autograd.grad(loss, [logits])
    x = logits.detach().numpy()
    x = x - x.max(1, keepdims=True)
    lp = x - np.log(np.exp(x).sum(1, keepdims=True))
    pr = np.exp(lp)
    onehot = np.zeros_like(pr)
    onehot[np.arange(n), action] = 1
    dl = -(adv / n)[:, None] * (onehot - pr)
    np.testing.assert_allclose(dl, gl.numpy(), rtol=1e-9, atol=1e-13)
    assert (dl[~mask] == 0).all()
    assert stats['policy_loss'] == pytest.approx(-np.mean(lp[np.arange(n), action] * adv), rel=1e-12)


@pytest.mark.parametrize('grad_clip', [0.0, 0.05])
def test_replay_step_equals_torch_adam(grad_clip):
    """pg_learn_replay's float64 step equals torch.optim.Adam (+ clip_grad_norm_) on the module parameters in float64, from fresh
    moments and from a running state"""
    from pg_reference import pg_learn_replay, pg_loss64
    from ppo_reference import policy64
    c, A, gs, sd, model, gf, mask, action, adv = _setup(n=20, seed=5)
    cfg = PGConfig(lr=1e-2, grad_clip=grad_clip)
    batch = dict(model=model, graph_features=gf, action_mask=mask, action=action, advantage=adv)
    params = {k: np.asarray(v.detach().numpy() if hasattr(v, 'detach') else v, np.float64) for k, v in sd.items()}
    p = {k: torch.nn.Parameter(torch.tensor(v)) for k, v in params.items()}
    opt = torch.optim.Adam(list(p.values()), lr=cfg.lr, betas=(cfg.adam_beta1, cfg.adam_beta2), eps=cfg.adam_eps, foreach=False)
    state = None
    for it in range(2):
        r = pg_learn_replay(params, c, gs, batch, cfg, state)
        opt.zero_grad()
        logits, _ = policy64(p, c, gs, model, gf, mask)
        loss, _ = pg_loss64(logits, action, adv)
        loss.backward()
        if grad_clip > 0:
            torch.nn.utils.clip_grad_norm_([x for x in p.values() if x.grad is not None], grad_clip)
        opt.step()
        for k in params:
            np.testing.assert_allclose(r['weights'][k], p[k].detach().numpy(), rtol=1e-12, atol=1e-14, err_msg=k)
        assert r['step'] == it + 1
        assert r['stats']['policy_loss'] == pytest.approx(loss.item(), rel=1e-12)
        params = {k: np.asarray(v) for k, v in r['weights'].items()}
        state = (r['m'], r['v'], r['step'])


def test_replay_of_an_empty_batch_is_no_step():
    from pg_reference import pg_learn_replay
    c, A, gs, sd, *_ = _setup(n=4)
    params = {k: np.asarray(v.detach().numpy() if hasattr(v, 'detach') else v, np.float64) for k, v in sd.items()}
    empty = dict(model=np.zeros(0, int), graph_features=np.zeros((0, c['in_features_graph'])), action_mask=np.zeros((0, A)),
                 action=np.zeros(0, int), advantage=np.zeros(0))
    m = np.ones(sum(v.size for v in params.values()))
    r = pg_learn_replay(params, c, gs, empty, PGConfig(), (m, m, 7))
    assert r['step'] == 7 and r['stats']['rows'] == 0
    for k in params:
        np.testing.assert_array_equal(r['weights'][k], params[k])


def test_config_defaults():
    cfg = PGConfig()
    assert (cfg.gamma, cfg.lr, cfg.grad_clip) == (0.99, 1e-4, 0.0)
    assert (cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps) == (0.9, 0.999, 1e-8)
