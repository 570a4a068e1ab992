"""-m gpu: every device learner's gradient (PPO, IMPALA, PG: the head-gradient kernel, ramp_gnn_embed_grad_kernel, finish) on
train batches a device environment recorded, against float64 autograd through tests/tie_reference.py's explain().

Synthetic host rows (tests/test_gpu_policy_learn.py) hold the gradient to max(1e-4, 10 e32) per tensor; on recorded batches a
ReLU pre-activation of the bench's graphs or of a row can sit within fp32 rounding of 0, and the kernel may take the other
branch there.  So each tensor of g - g64 must be within that bound once the flips of a small set S of named near-tied units
(margin below tie_reference.TAU) are added to g64; an error no such set explains fails.  Batches are formed as each learner
forms them: PPO's train batch (host_batch, the old logits at the collection weights), IMPALA's fragments (one fragment per
episode, all of them in one batch), PG's train rows (discounted returns).  Environments: config 3 (ResNet-50, 64 workers),
mix128 (ResNet + a GPT-2-like job on 128 workers, |A| = 5) and the three bench job types; 64 episodes of 6 jobs, and 1,300
episodes of 4 jobs (about 5,200 rows); weight seeds 2, 4, 6 and 21.  The PPO learn call that meets a tie at weight seed 4 in
tests/test_gpu_ppo_learn_replay.py ('mixed_types') is traced here minibatch by minibatch.  pytest -s prints, per case, the worst
residual after S, torch fp32's error on that tensor and S."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from test_gpu_policy_learn import _Static, _env, host_batch, tensor_errors
from tie_reference import GNN_MODULES, TAU, deltas, explain, flips, grad64, near_ties

pytestmark = pytest.mark.gpu


def check_explained(pol, tag, grad, model, gf, mask, loss_fn, params=None, graphs=None, max_candidates=None):
    """the kernel's gradient `grad` (blob) of loss_fn(logits, value) over the rows (model, gf, mask) at the policy's weights (or
    `params`, name -> array) against float64 through explain(); returns (S as Flip, residuals, the float64 gradient).  graphs:
    per job type, objects with nf, ef, src, dst (default: the policy's own job types).  Only ReLU / leaky-ReLU sites are
    candidates: tanh has no branch to flip; max_candidates keeps the closest ones (each costs an autograd run)"""
    from ddls_b200 import policy as P
    c, A = pol.config, pol.n_actions
    params = P.unpack_weights(pol.get_weights(), c, A) if params is None else params
    graphs = [_Static(st) for st in pol.static] if graphs is None else graphs
    g64, gl, gv = grad64(params, c, graphs, model, gf, mask, loss_fn)
    g32 = grad64(params, c, graphs, model, gf, mask, loss_fn, dtype=torch.float32)[0]
    e32 = tensor_errors(P.pack_weights(g32, c, A), g64, c, A)
    gk = {k: v.astype(np.float64) for k, v in P.unpack_weights(grad, c, A).items()}
    ties = [t for t in near_ties(params, c, graphs, model, gf, mask, TAU)
            if c['aggregator_activation' if t.site[0] in GNN_MODULES else 'fcnet_activation'] != 'tanh']
    errs = tensor_errors(grad, g64, c, A)
    if all(e <= max(1e-4, 10 * e32[k]) for k, e in errs.items()):
        S, resid = [], errs                                             # nothing to explain: no flip needed
    else:
        ties = ties[:max_candidates]
        bad = {k: f'{e:.2e} (torch fp32 {e32[k]:.2e})' for k, e in errs.items() if e > max(1e-4, 10 * e32[k])}
        print(f'{tag}: explaining {bad} by the closest {len(ties)} near-ties', flush=True)
        cands, ds = flips(ties, deltas(params, c, graphs, model, gf, mask, gl.numpy(), gv.numpy(), ties))
        S, resid = explain(gk, g64, ds, e32, cands)
        S = [cands[i] for i in S]
    assert all(t.margin < TAU for f in S for t in f.ties)
    k = max(resid, key=lambda x: resid[x] / max(1e-4, 10 * e32[x]))
    k0 = max(errs, key=errs.get)
    print(f'{tag}: {len(model)} rows, {len(ties)} candidates below {TAU:g}; before S {errs[k0]:.2e} ({k0}, torch fp32 '
          f'{e32[k0]:.2e}); after S worst {resid[k]:.2e} ({k}, torch fp32 {e32[k]:.2e}); S = '
          + ('[]' if not S else '[' + '; '.join(map(str, S)) + ']'))
    return S, resid, g64


def ppo_loss(b, cfg):
    from ppo_reference import ppo_loss64
    return lambda logits, value: ppo_loss64(logits, value, b['action'], b['old_logits'], b['advantage'], b['value_target'], cfg)[0]


def pg_loss(b):
    from pg_reference import pg_loss64
    return lambda logits, value: pg_loss64(logits, b['action'], b['advantage'])[0]


def impala_rows(b, cfg):
    """the live rows of IMPALA fragments and VTraceLoss as a function of their logits and values"""
    from impala_reference import impala_loss64
    model = np.asarray(b['model']).reshape(-1)
    live = np.flatnonzero(model >= 0)
    idx = torch.as_tensor(live)
    gf = np.asarray(b['graph_features']).reshape(len(model), -1)[live]
    mask = np.asarray(b['action_mask']).reshape(len(model), -1)[live]

    def loss(logits, value):
        full_l = torch.zeros((len(model), logits.shape[1]), dtype=logits.dtype).index_put((idx,), logits)
        full_v = torch.zeros(len(model), dtype=value.dtype).index_put((idx,), value)
        return impala_loss64(full_l, full_v, b, cfg)[0]
    return model[live], gf, mask, loss


def _make_env(kind, B, J):
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    if kind == 'mix128':
        from test_gpu_eval_step_stats import _mix128
        env = _mix128(B=B, J=J, seed=4)
        return env, [m.graph for m in env.models]
    if kind == 'bench':
        graphs = [workload.make_graph(k) for k in ('resnet', 'bert', 'gpt2')]
        return DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=J, seed=7), graphs
    return _env(B=B, J=J, seed=7)


# environment, episodes B, jobs per episode J (the horizon: every episode ends in the segment)
ENVS = {'cfg3': ('cfg3', 64, 6), 'mix128': ('mix128', 64, 6), 'bench_types': ('bench', 64, 6), 'cfg3_1300': ('cfg3', 1300, 4)}


@pytest.mark.parametrize('wseed', [2, 4, 6, 21])
@pytest.mark.parametrize('eid', list(ENVS))
def test_learner_gradients_on_recorded_batches(eid, wseed):
    kind, B, J = ENVS[eid]
    env, graphs = _make_env(kind, B, J)
    learner_gradients_on_a_recorded_batch(env, graphs, J, wseed, f'{eid} seed {wseed}', min_rows=3000 if B > 1000 else 100)


def learner_gradients_on_a_recorded_batch(env, graphs, J, wseed, tag, min_rows):
    """a J-step segment of env recorded by a DeviceGNNPolicy on graphs at weight seed wseed; the PPO, IMPALA and PG gradients on
    the batches each learner forms from it, explained against float64.  Closes env."""
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceIMPALALearner, DevicePGLearner, DevicePPOLearner, IMPALAConfig, PGConfig, PPOConfig
    from impala_reference import fragments
    from pg_reference import train_rows
    A = env.max_partitions_per_op + 1
    pol = P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=wseed))
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=3).items()}
        assert traj['done'][-1].all()
        # PPO: the train batch learn() builds (GAE, standardised advantages), old logits at the collection weights
        cfg = PPOConfig(num_sgd_iter=0)
        probe = DevicePPOLearner(pol, cfg)
        probe.learn(env, J)
        b = host_batch(pol, traj, probe.train_batch(env))
        assert len(b['model']) > min_rows
        _, g = DevicePPOLearner(pol, PPOConfig()).loss_and_grad(b)
        check_explained(pol, f'ppo {tag}', g, b['model'], b['graph_features'], b['action_mask'], ppo_loss(b, PPOConfig()))
        # IMPALA: every fragment of the segment (one per episode) in one batch
        icfg = IMPALAConfig()
        fr = fragments(traj, [st['graph_static'] for st in pol.static], pol.n_models, J)
        _, g, _ = DeviceIMPALALearner(pol, icfg).loss_and_grad(fr)
        model, gf, mask, loss = impala_rows(fr, icfg)
        check_explained(pol, f'impala {tag}', g, model, gf, mask, loss)
        # PG: the train rows with their discounted returns
        pcfg = PGConfig()
        b = train_rows(pol, traj, pcfg.gamma)
        _, g = DevicePGLearner(pol, pcfg).loss_and_grad(b)
        check_explained(pol, f'pg {tag}', g, b['model'], b['graph_features'], b['action_mask'], pg_loss(b))
    finally:
        pol.close(); env.close()


def test_ppo_mixed_types_at_weight_seed_4_minibatch_by_minibatch():
    """test_gpu_ppo_learn_replay's 'mixed_types' call pair at weight seed 4 (the seed it moved away from), on the device learner's
    own parts: every minibatch's loss_and_grad at the current weights explained against float64, then torch's fp32 Adam step"""
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    from ppo_reference import adam_step, shuffle_order
    env, graphs = _make_env('mix128', 64, 6)
    A = env.max_partitions_per_op + 1
    pol = P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=4))
    H = 6
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, H, sample=True, seed=3).items()}
        base = PPOConfig(num_sgd_iter=3, seed=21)
        probe = DevicePPOLearner(pol, dataclasses.replace(base, num_sgd_iter=0))
        probe.learn(env, H)
        n = len(probe.train_batch(env)['advantage'])
        cfg = dataclasses.replace(base, sgd_minibatch_size=-(-n // 4))
        lrn = DevicePPOLearner(pol, cfg)
        lrn.reset()
        n_flips = 0
        for call in range(2):
            c_cfg = dataclasses.replace(cfg, seed=cfg.seed + call, kl_coeff=lrn.config.kl_coeff)
            probe = DevicePPOLearner(pol, dataclasses.replace(c_cfg, num_sgd_iter=0))
            probe.learn(env, H)
            b = host_batch(pol, traj, probe.train_batch(env))
            w0 = w = pol.get_weights()
            m, v, step = lrn.adam_state()
            parts = DevicePPOLearner(pol, c_cfg)
            for p in range(c_cfg.num_sgd_iter):
                order = shuffle_order(c_cfg.seed, p, n)
                for s in range(0, n, c_cfg.sgd_minibatch_size):
                    sub = {k: x[order[s:s + c_cfg.sgd_minibatch_size]] for k, x in b.items()}
                    _, g = parts.loss_and_grad(sub)
                    S, _, _ = check_explained(pol, f'mixed_types seed 4 call {call + 1} pass {p} rows {s}', g, sub['model'],
                                           sub['graph_features'], sub['action_mask'], ppo_loss(sub, c_cfg))
                    n_flips += len(S)
                    w, m, v, _ = adam_step(w, g, m, v, step, c_cfg)
                    step += 1
                    pol.set_weights(w)
            pol.set_weights(w0)
            lrn.learn(env, H)                                           # the call itself, for its weights and kl_coeff
            d = np.abs(pol.get_weights().astype(np.float64) - w).max() / np.abs(w - w0).max()
            assert d <= 1e-4, d
            assert lrn.adam_state()[2] == step
        print(f'mixed_types seed 4: {n_flips} flips over {2 * cfg.num_sgd_iter * math.ceil(n / cfg.sgd_minibatch_size)} minibatches')
    finally:
        pol.close(); env.close()
