"""-m gpu: the device GNN policy's two kernels (ddls_b200/csrc/ramp_policy.cu: ramp_gnn_embed_kernel, ramp_policy_head_kernel)
against the float64 restatement of the reference's GNNPolicy (tests/gnn_reference.py: embed64 / head64), at the widths, depths and
graph shapes check_config admits, and the action selection draw for draw.

Tolerance: |cuda - ref| <= 1e-5 + 1e-5 |ref|, element by element, on embeddings, unmasked logits and values.  The kernels are fp32;
a torch fp32 restatement differs from its float64 copy by at most ~1.4e-7 on these configurations, and a serial fp32 mean of
20,000 post-activation values (the embed kernel's node mean) by ~1.6e-6, so the bound has about 6x headroom on the largest graph.
Masked logits are -FLT_MAX exactly (logit + max(log 0, finfo(float32).min) rounds to it in fp32).

The policy is driven through DeviceGNNPolicy's own methods on raw graphs (RawPolicy below), so that node, edge and graph widths are
free; the read-out runs through decide(), which returns the logits, value, log-probability and action of every row."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL = 1e-5
NEG_FLT_MAX_BITS = 0xff7fffff
SMEM_LIMIT = 200 * 1024
GOLDEN_RATIO64, ROW_KEY64 = 0x9E3779B97F4A7C15, 0xD1342543DE82EF95

YAML = {}
MAX = dict(in_features_node=128, in_features_edge=128, in_features_graph=96, out_features_msg=128, out_features_hidden=128,
           out_features_node=96, out_features_graph=32, num_rounds=8, fcnet_hiddens=(128,), aggregator_activation='leaky_relu',
           fcnet_activation='tanh')
MIN = dict(in_features_node=1, in_features_edge=1, in_features_graph=1, out_features_msg=2, out_features_hidden=1, out_features_node=1,
           out_features_graph=1, fcnet_hiddens=(32,))
ODD = dict(in_features_node=33, in_features_edge=3, in_features_graph=63, out_features_msg=66, out_features_hidden=65,
           out_features_node=95, out_features_graph=31, num_rounds=3, fcnet_hiddens=(96,), aggregator_activation='leaky_relu')
WIDE_FC = dict(fcnet_hiddens=(512,), fcnet_activation='tanh')
UNMASKED = dict(apply_action_mask=False)

# id: (overrides of gnn.yaml, n_actions, head kernel shared memory in bytes or None, with the two largest graphs)
CONFIGS = {
    'yaml': (YAML, 17, None, True),
    'max': (MAX, 32, 174_852, True),
    'min': (MIN, 1, None, False),
    'odd': (ODD, 2, 115_596, False),
    'wide-fc': (WIDE_FC, 17, 148_920, False),
    'unmasked': (UNMASKED, 9, None, False),
}
SEED = 3                       # under seed 3 min's single relu unit is live (several other seeds leave every embedding at zero)


def _cfg(overrides):
    from ddls_b200 import policy as P
    c = dict(P.DEFAULT_CONFIG)
    c.update(overrides)
    return c


def head_smem_bytes(c, n_actions, warps=8):
    """head_smem_floats (ramp_policy.cu) in bytes"""
    gin, og, fin, H, A = c['in_features_graph'] + n_actions, c['out_features_graph'], c['out_features_node'] + c['out_features_graph'], \
        tuple(c['fcnet_hiddens'])[0], n_actions
    return 4 * (2 * gin + og * gin + og + 2 * fin * H + 2 * H + A * H + A + H + 1 + warps * 2 * 128)


class Graph:
    def __init__(self, name, n, src, dst):
        self.name, self.n = name, n
        self.src, self.dst = np.asarray(src, dtype=np.int32), np.asarray(dst, dtype=np.int32)

    def features(self, c, rng):
        self.nf = rng.standard_normal((self.n, c['in_features_node'])).astype(np.float32)
        self.ef = rng.standard_normal((len(self.src), c['in_features_edge'])).astype(np.float32)
        self.gs = rng.standard_normal(6).astype(np.float32)
        return self


def graphs(big):
    rng = np.random.default_rng(17)
    src, dst = rng.integers(0, 300, 840), rng.integers(0, 300, 840)
    loops = rng.integers(0, 300, 30)
    dup = rng.integers(0, 840, 30)
    out = [Graph('single', 1, [], []), Graph('pair', 2, [0], [1]), Graph('chain40', 40, np.arange(39), np.arange(1, 40)),
           Graph('multi300', 300, np.concatenate([src, loops, src[dup]]), np.concatenate([dst, loops, dst[dup]]))]
    if big:
        out += [Graph('star4096', 4097, np.arange(1, 4097), np.zeros(4096)),
                Graph('random20k', 20000, rng.integers(0, 20000, 60000), rng.integers(0, 20000, 60000))]
    return out


def _raw_policy_class():
    from ddls_b200 import policy as P

    class RawPolicy(P.DeviceGNNPolicy):
        """DeviceGNNPolicy on raw graphs (Graph above) of any width check_config admits; the product class builds its job types
        from synth graphs with gnn.yaml's observation widths."""

        def __init__(self, c, n_actions, gs, state_dict, device=0):
            self.config, self.n_actions, self.n_models = dict(c), int(n_actions), len(gs)
            self._L = P._engine.load_library()
            P._bind(self._L)
            self._cfg = P.c_config(self.config, self.n_actions, self.n_models)
            self._h = C.c_void_p()
            P._engine._check(self._L.ramp_policy_create(device, C.byref(self._cfg), C.byref(self._h)))
            for m, g in enumerate(gs):
                self.set_model(m, g.nf, g.ef, g.src, g.dst, g.gs)
            self.set_weights(state_dict)
    return RawPolicy


def raw_policy(c, n_actions, gs, sd):
    return _raw_policy_class()(c, n_actions, gs, sd)


def check_close(got, want, what):
    """|got - want| <= TOL + TOL |want| element by element; returns the largest absolute error"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    err = np.abs(got - want)
    bad = err > TOL + TOL * np.abs(want)
    assert not bad.any(), f'{what}: {int(bad.sum())} of {bad.size} outside the bound, worst {err.max():.3e} at ' \
                          f'{np.unravel_index(np.argmax(err), err.shape)} (got {got.flat[np.argmax(err)]!r}, want {want.flat[np.argmax(err)]!r})'
    return float(err.max()) if err.size else 0.0


class Case:
    pass


@pytest.fixture(scope='module', params=list(CONFIGS))
def case(request):
    """One policy per configuration with every graph registered as its own model (each CTA of the embed kernel indexes its model),
    and the float64 embeddings of each."""
    from ddls_b200 import policy as P
    from gnn_reference import embed64
    over, A, _, big = CONFIGS[request.param]
    k = Case()
    k.id, k.c, k.A = request.param, _cfg(over), A
    rng = np.random.default_rng(5)
    k.graphs = [g.features(k.c, rng) for g in graphs(big)]
    k.sd = P.random_state_dict(k.c, A, seed=SEED)
    k.emb64 = np.stack([embed64(k.sd, k.c, g.nf, g.ef, g.src, g.dst) for g in k.graphs])
    k.pol = raw_policy(k.c, A, k.graphs, k.sd)
    yield k
    k.pol.close()


def batch(k, n, seed):
    """n rows: random models, N(0, 1) graph features, masks at p = 0.7, and the special rows all masked / only action 0 / only
    action A - 1 / all valid at the start and at the end of the batch"""
    rng = np.random.default_rng(seed)
    model = rng.integers(0, k.pol.n_models, n).astype(np.int32)
    gf = rng.standard_normal((n, k.c['in_features_graph'])).astype(np.float32)
    mask = (rng.random((n, k.A)) < 0.7).astype(np.uint8)
    special = np.zeros((4, k.A), dtype=np.uint8)
    special[1, 0] = special[2, k.A - 1] = 1
    special[3] = 1
    for i, row in enumerate(special):
        if i < n:
            mask[i] = row
        if n > 8:
            mask[n - 4 + i] = row
    return model, gf, mask


def log_softmax_at(logits, action):
    l = logits.astype(np.float64)
    mx = l.max(1)
    return l[np.arange(len(l)), action] - mx - np.log(np.exp(l - mx[:, None]).sum(1))


def splitmix64(x):
    x = x + np.uint64(GOLDEN_RATIO64)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def expected_draws(logits, seed):
    """The head kernel's categorical draw restated on the host from the fp32 logits it returned: row b draws
    U = (splitmix64(seed ^ b * 0xD1342543DE82EF95) >> 40) 2^-24 and takes the first action i with e_i > 0 and cum_i > U sum(e),
    e_i = exp(l_i - max) (float64 here), else the greedy action.  near: rows whose nearest boundary lies within 1e-5 sum(e) of
    U sum(e), where the kernel's fp32 sums may legitimately land on the other side."""
    u01 = uniform24([seed], len(logits))[0].astype(np.float64) * 2.0 ** -24
    l = logits.astype(np.float64)
    e = np.exp(l - l.max(1, keepdims=True))
    cum = np.cumsum(e, 1)
    tot = cum[:, -1]
    u = u01 * tot
    ok = (e > 0) & (cum > u[:, None])
    action = np.where(ok.any(1), ok.argmax(1), np.argmax(logits, 1))
    near = np.minimum(np.abs(cum - u[:, None]).min(1), u) <= 1e-5 * tot
    return action, near


def check_readout(k, model, gf, mask, out, what):
    """logits / value against head64 on the float64 embeddings; masked logits -FLT_MAX bit for bit; returns the largest errors"""
    from gnn_reference import head64
    logits, value = out[0], out[1]
    wl, wv = head64(k.sd, k.c, k.emb64[model], gf, mask)
    valid = mask.astype(bool) | (not k.c['apply_action_mask'])
    el = check_close(logits[valid], wl[valid], f'{what} logits')
    if k.c['apply_action_mask'] and (~valid).any():
        assert (logits[~valid].view(np.uint32) == NEG_FLT_MAX_BITS).all(), f'{what}: a masked logit is not -FLT_MAX'
    ev = check_close(value, wv, f'{what} value')
    return el, ev


# ---- configuration capacity ----

def test_head_shared_memory_and_the_capacity_edge():
    from ddls_b200 import policy as P
    for name, (over, A, smem, _) in CONFIGS.items():
        b = head_smem_bytes(_cfg(over), A)
        assert b <= SMEM_LIMIT, name
        if smem is not None:
            assert b == smem, name
    L = P._engine.load_library()
    P._bind(L)
    over_edge = dict(MAX, fcnet_hiddens=(160,))
    assert head_smem_bytes(_cfg(over_edge), 32) == 212_100 > SMEM_LIMIT
    h = C.c_void_p()
    assert L.ramp_policy_create(0, C.byref(P.c_config(_cfg(over_edge), 32, 1)), C.byref(h)) == -3      # RAMP_ERR_CAPACITY
    assert b'shared memory' in L.ramp_last_error()
    assert L.ramp_policy_create(0, C.byref(P.c_config(_cfg(MAX), 32, 1)), C.byref(h)) == 0
    L.ramp_policy_destroy(h)


# ---- the embed kernel ----

def test_embeddings_match_fp64(case):
    emb = case.pol.embed()
    assert np.abs(case.emb64).max() > 1e-3
    for m, g in enumerate(case.graphs):
        err = check_close(emb[m], case.emb64[m], f'{case.id} {g.name} embedding')
        print(f'[policy-err] {case.id:9s} {g.name:10s} embedding max |err| {err:.3e} (max |ref| {np.abs(case.emb64[m]).max():.3f})')
        if g.name == 'star4096':
            # every leaf has in-degree 0 and ends each round at zero, so the node mean is the centre's state / 4,097, far below the
            # absolute part of the bound: the node sum (the centre's mean over its 4,097-message mailbox) is held to it instead
            err = check_close(emb[m].astype(np.float64) * g.n, case.emb64[m] * g.n, f'{case.id} star centre')
            print(f'[policy-err] {case.id:9s} star centre state max |err| {err:.3e} (max |ref| {np.abs(case.emb64[m] * g.n).max():.3f})')


# ---- the head kernel: read-out and greedy selection ----

@pytest.mark.parametrize('n', [1, 7, 8, 9, 2111, 2112, 2113, 50000])
def test_decide_matches_fp64(case, n):
    """The grid is capped at 2 x 132 CTAs of 8 warps: 2,112 rows per pass, the rest go round the persistent loop."""
    model, gf, mask = batch(case, n, seed=n)
    out = case.pol.decide(model, gf, mask)
    el, ev = check_readout(case, model, gf, mask, out, f'{case.id} n={n}')
    logits, _, logp, action = out
    np.testing.assert_array_equal(action, np.argmax(logits, 1))                            # the first maximal logit
    if case.c['apply_action_mask']:
        assert mask[np.arange(n), action][mask.any(1)].all()
    np.testing.assert_allclose(logp, log_softmax_at(logits, action), rtol=0, atol=1e-5)
    np.testing.assert_array_equal(case.pol.forward(model, gf, mask)[0], logits)            # forward is the same read-out
    if n == 50000:
        print(f'[policy-err] {case.id:9s} read-out   logits max |err| {el:.3e}, value max |err| {ev:.3e}')


def test_rows_outside_the_models_are_zero_and_leave_their_neighbours_alone(case):
    n = 2113
    model, gf, mask = batch(case, n, seed=77)
    base = case.pol.decide(model, gf, mask, sample=True, seed=991)
    bad = np.array([0, 5, 2104, 2111, n - 1])
    model2 = model.copy()
    model2[bad[::2]], model2[bad[1::2]] = -1, case.pol.n_models
    got = case.pol.decide(model2, gf, mask, sample=True, seed=991)
    keep = np.setdiff1d(np.arange(n), bad)
    for a, b in zip(got, base):
        np.testing.assert_array_equal(a[keep], b[keep])
        assert (a[bad] == 0).all()


def test_greedy_ties_go_to_the_first_index():
    """Logit rows i < j copied with equal biases give bitwise-equal logits (same per-lane products, same reduction order); the
    action is i, or j where i is masked.  Pairs straddle lane 16 of the butterfly and reach lane 31."""
    from ddls_b200 import policy as P
    c, A = _cfg(MAX), 32
    rng = np.random.default_rng(8)
    gs = [g.features(c, rng) for g in graphs(False)]
    sd = P.random_state_dict(c, A, seed=SEED)
    pol = raw_policy(c, A, gs, sd)
    n = 512
    model = rng.integers(0, len(gs), n).astype(np.int32)
    gf = rng.standard_normal((n, c['in_features_graph'])).astype(np.float32)
    W, b = 'logit_module._logits._model.0.weight', 'logit_module._logits._model.0.bias'
    for i, j in [(15, 16), (0, 16), (7, 23), (15, 31), (30, 31), (0, 31)]:
        s = {key: v.copy() for key, v in sd.items()}
        s[W][j] = s[W][i]
        s[b][i] += 20.0
        s[b][j] = s[b][i]
        pol.set_weights(s)
        mask = np.ones((n, A), dtype=np.uint8)
        mask[n // 2:, i] = 0
        logits, _, _, action = pol.decide(model, gf, mask)
        top = logits[:n // 2]
        np.testing.assert_array_equal(top[:, i].view(np.uint32), top[:, j].view(np.uint32))
        assert (top[:, i] == top.max(1)).all()
        assert (action[:n // 2] == i).all(), (i, j, np.unique(action[:n // 2]))
        assert (action[n // 2:] == j).all(), (i, j, np.unique(action[n // 2:]))
    pol.close()


# ---- the head kernel: categorical draws ----

def test_sampler_draw_for_draw(case):
    n, seed = 50000, 0x5DEECE66D2F1A3B7
    model, gf, mask = batch(case, n, seed=123)
    logits, value, logp, action = case.pol.decide(model, gf, mask, sample=True, seed=seed)
    greedy = case.pol.decide(model, gf, mask)
    np.testing.assert_array_equal(logits, greedy[0])
    np.testing.assert_array_equal(value, greedy[1])
    want, near = expected_draws(logits, seed)
    assert near.mean() < 0.005, near.mean()
    np.testing.assert_array_equal(action[~near], want[~near])
    np.testing.assert_allclose(logp, log_softmax_at(logits, action), rtol=0, atol=1e-5)
    if case.A > 1:
        assert len(np.unique(action)) > 1
    print(f'[policy-err] {case.id:9s} sampler    {int(near.sum())} of {n} rows near a boundary ({100 * near.mean():.3f} %)')


def uniform24(seeds, n):
    """(splitmix64(seed ^ b * 0xD1342543DE82EF95) >> 40) for every seed and row b < n: the 24 bits of each row's uniform"""
    with np.errstate(over='ignore'):
        r = splitmix64(np.asarray(seeds, dtype=np.uint64)[:, None] ^ (np.arange(n, dtype=np.uint64) * np.uint64(ROW_KEY64))[None, :])
    return r >> np.uint64(40)


def all_masked_draw(v, A):
    """The kernel's draw where every logit is -FLT_MAX: every e_i is exactly 1, cum_i = i + 1 and the sum A are exact in fp32, so
    the draw is the first i with i + 1 > fl32(fl32(v 2^-24) A), the greedy action 0 if none"""
    u = (v.astype(np.float32) * np.float32(2.0 ** -24)) * np.float32(A)
    ok = np.arange(1, A + 1, dtype=np.float32) > u[..., None]
    return np.where(ok.any(-1), ok.argmax(-1), 0)


def test_sampler_uses_all_24_bits_of_the_uniform():
    """Rows with every action masked make the kernel's draw exact fp32 arithmetic.  The seeds are searched so that some row's
    draw changes if the uniform's lowest bit is dropped; every row must equal the exact draw."""
    k = _small_case(_cfg(YAML), 17, seed=12)
    n, A = 64, 17
    found = []
    for start in range(0, 1 << 22, 1 << 16):
        seeds = np.arange(start, start + (1 << 16), dtype=np.uint64)
        v = uniform24(seeds, n)
        hit = (all_masked_draw(v, A) != all_masked_draw(v & ~np.uint64(1), A)).any(1)
        found += [int(s) for s in seeds[hit]]
        if len(found) >= 4:
            break
    assert len(found) >= 4
    model = np.arange(n, dtype=np.int32) % k.pol.n_models
    gf = np.random.default_rng(1).standard_normal((n, 17)).astype(np.float32)
    mask = np.zeros((n, A), dtype=np.uint8)
    for seed in found[:4]:
        logits, _, logp, action = k.pol.decide(model, gf, mask, sample=True, seed=seed)
        assert (logits.view(np.uint32) == NEG_FLT_MAX_BITS).all()
        np.testing.assert_array_equal(action, all_masked_draw(uniform24([seed], n)[0], A), err_msg=f'seed {seed}')
        np.testing.assert_allclose(logp, -np.log(A), rtol=0, atol=1e-6)
    k.pol.close()


def _env(B=256, seed=5):
    from ddls_b200 import synth
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    gs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6'),
          synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)]
    env = DeviceRampJobPartitioningEnvironment((4, 4, 2), gs, n_episodes=B, jobs_per_episode=4, max_partitions_per_op=16,
                                               min_op_run_time_quantum=2.0, interarrival=('exponential', 600.0), frac=(0.5, 0.5, 2),
                                               seed=seed)
    return env, gs


def test_act_draws_with_the_call_count_mixed_into_the_seed():
    """act() keys the k-th call (1-based) with seed ^ k * 0x9E3779B97F4A7C15, then draws exactly as decide()."""
    from ddls_b200 import policy as P
    env, gs = _env(B=4096, seed=9)
    pol = P.DeviceGNNPolicy(gs, 17, None, P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=2))
    obs = env.reset()
    live = (obs['model'] >= 0) & ~obs['done']
    assert live.sum() > 1000
    seed = 123456789
    for k in (1, 2):
        pol.act(env, sample=True, seed=seed)
        got = pol.read(env)
        mixed = (seed ^ (GOLDEN_RATIO64 * k)) & (2 ** 64 - 1)
        want, near = expected_draws(got['logits'], mixed)
        assert near[live].mean() < 0.005
        ok = live & ~near
        np.testing.assert_array_equal(got['actions'][ok], want[ok])
        assert (got['actions'][~live] == 0).all()
        np.testing.assert_allclose(got['logp'][live], log_softmax_at(got['logits'], got['actions'])[live], rtol=0, atol=1e-5)
    env.close(); pol.close()


# ---- cached embeddings ----

def _small_case(c, A, seed):
    from ddls_b200 import policy as P
    rng = np.random.default_rng(seed)
    k = Case()
    k.c, k.A = c, A
    k.graphs = [g.features(c, rng) for g in graphs(False)]
    k.sd = P.random_state_dict(c, A, seed=SEED)
    k.pol = raw_policy(c, A, k.graphs, k.sd)
    return k


def _emb64(k):
    from gnn_reference import embed64
    return np.stack([embed64(k.sd, k.c, g.nf, g.ef, g.src, g.dst) for g in k.graphs])


def test_set_weights_invalidates_the_embeddings():
    from ddls_b200 import policy as P
    from gnn_reference import head64
    k = _small_case(_cfg(YAML), 17, seed=1)
    model, gf, mask = batch(k, 256, seed=2)
    k.emb64 = _emb64(k)
    k.pol.embed()
    check_readout(k, model, gf, mask, k.pol.forward(model, gf, mask), 'first weights')
    old = k.emb64
    k.sd = P.random_state_dict(k.c, 17, seed=SEED + 1)
    k.pol.set_weights(k.sd)
    k.emb64 = _emb64(k)
    stale = head64(k.sd, k.c, old[model], gf, mask)[1]
    assert np.abs(stale - head64(k.sd, k.c, k.emb64[model], gf, mask)[1]).max() > 100 * TOL        # stale embeddings would show
    check_readout(k, model, gf, mask, k.pol.forward(model, gf, mask), 'second weights, forward')
    check_readout(k, model, gf, mask, k.pol.decide(model, gf, mask), 'second weights, decide')
    k.pol.close()


def test_set_model_changes_that_model_and_no_other():
    k = _small_case(_cfg(YAML), 17, seed=3)
    model, gf, mask = batch(k, 512, seed=4)
    k.emb64 = _emb64(k)
    before = k.pol.decide(model, gf, mask)
    check_readout(k, model, gf, mask, before, 'before')
    m = 3                                                                                    # multi300 -> a 12-node chain
    k.graphs[m] = Graph('chain12', 12, np.arange(11), np.arange(1, 12)).features(k.c, np.random.default_rng(6))
    g = k.graphs[m]
    k.pol.set_model(m, g.nf, g.ef, g.src, g.dst, g.gs)
    k.emb64 = _emb64(k)
    after = k.pol.decide(model, gf, mask)
    check_readout(k, model, gf, mask, after, 'after')
    other = model != m
    assert (~other).sum() > 50
    for a, b in zip(after, before):
        np.testing.assert_array_equal(a[other], b[other])
    assert np.abs(after[1][~other] - before[1][~other]).max() > 100 * TOL
    emb = k.pol.embed()
    check_close(emb, k.emb64, 'embeddings after set_model')
    k.pol.close()


# ---- forward / decide leave what act left for read ----

def test_forward_and_decide_leave_the_last_act_alone():
    from ddls_b200 import policy as P
    env, gs = _env(B=256, seed=5)
    pol = P.DeviceGNNPolicy(gs, 17, None, P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=4))
    obs = env.reset()
    pol.act(env, sample=True, seed=42)
    first = pol.read(env)
    rng = np.random.default_rng(0)
    for n in (7, 3 * env.B):                                                                 # n > B grows the host-input buffers
        model = rng.integers(0, len(gs), n).astype(np.int32)
        gf = rng.standard_normal((n, 17)).astype(np.float32)
        mask = (rng.random((n, 17)) < 0.5).astype(np.uint8)
        pol.forward(model, gf, mask)
        pol.decide(model, gf, mask, sample=True, seed=1)
    second = pol.read(env)
    for key in first:
        np.testing.assert_array_equal(second[key], first[key], err_msg=key)
    assert (obs['model'] >= 0).any()
    fresh = P.DeviceGNNPolicy(gs, 17, None, P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=4))
    fresh.forward(np.zeros(4 * env.B, dtype=np.int32), np.zeros((4 * env.B, 17), dtype=np.float32), np.ones((4 * env.B, 17)))
    with pytest.raises(Exception, match='nothing to read'):
        fresh.read(env)
    env.close(); pol.close(); fresh.close()


# ---- the binding refuses arrays of the wrong shape before any C call ----

def test_wrong_shapes_raise_value_error():
    k = _small_case(_cfg(YAML), 17, seed=9)
    g = k.graphs[2]
    E = len(g.src)
    for bad in [dict(node_features=g.nf[:, :4]), dict(node_features=g.nf[:, 0]), dict(edge_features=g.ef[:, :1]),
                dict(edge_features=g.ef[:-1]), dict(edges_src=g.src[:-1]), dict(edges_dst=g.dst[:-1]),
                dict(edges_src=np.stack([g.src, g.src])), dict(graph_static=g.gs[:5])]:
        args = dict(node_features=g.nf, edge_features=g.ef, edges_src=g.src, edges_dst=g.dst, graph_static=g.gs)
        args.update(bad)
        with pytest.raises(ValueError):
            k.pol.set_model(2, **args)
    assert E == 39
    model, gf, mask = batch(k, 16, seed=1)
    for bad in [dict(graph_features=gf[:, :16]), dict(graph_features=gf[:-1]), dict(action_mask=mask[:, :16]),
                dict(action_mask=np.concatenate([mask, mask[:1]])), dict(model=model[:, None]), dict(model=model[:-1])]:
        args = dict(model=model, graph_features=gf, action_mask=mask)
        args.update(bad)
        with pytest.raises(ValueError):
            k.pol.forward(**args)
        with pytest.raises(ValueError):
            k.pol.decide(**args, sample=True, seed=1)
    k.emb64 = _emb64(k)
    check_readout(k, model, gf, mask, k.pol.decide(model, gf, mask), 'after the refusals')
    k.pol.close()
