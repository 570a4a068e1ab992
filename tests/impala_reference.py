"""TEST INFRASTRUCTURE -- float64 torch restatements for the IMPALA learner (ramp_policy_learn_impala, ramp_impala_loss_grad in
ddls_b200/csrc/ramp_policy.cu and ramp_policy_learn.cuh), on top of tests/ppo_reference.py's policy64 and adam_step.

RLlib is not installed; these restate ray 3.0.0.dev0 (the version the reference pins):

  ray/rllib/algorithms/impala/vtrace_torch.py
    multi_from_logits        target log p(a) = -cross_entropy(target logits, a); with one action component and the behaviour
                             log-probabilities given, those are used as they are: log_rhos = target - behaviour
    from_importance_weights  rhos = exp(log_rhos); clipped_rhos = clamp_max(rhos, clip_rho_threshold); cs = clamp_max(rhos, 1.0);
                             values_t_plus_1 = cat(values[1:], bootstrap_value); deltas = clipped_rhos (rewards + discounts
                             values_t_plus_1 - values); vs_minus_v_xs accumulated backwards: delta_t + discount_t c_t acc;
                             vs = vs_minus_v_xs + values; vs_t_plus_1 = cat(vs[1:], bootstrap_value); pg_advantages =
                             clamp_max(rhos, clip_pg_rho_threshold) (rewards + discounts vs_t_plus_1 - values); both detached
  ray/rllib/algorithms/impala/impala_torch_policy.py
    _make_time_major         [B * T] -> [T, B]; drop_last removes the last time step
    ImpalaTorchPolicy.loss   vtrace_drop_last_ts: every time-major input drop_last, values = values_time_major[:-1],
                             bootstrap_value = values_time_major[-1]; discounts = (1 - dones) gamma
    VTraceLoss               pi_loss = -sum(logp(a) pg_advantages valid); vf_loss = 0.5 sum(((values - vs) valid)^2);
                             entropy = sum(H valid), mean_entropy = entropy / sum(valid);
                             total_loss = pi_loss + vf_loss vf_loss_coeff - entropy entropy_coeff

Line numbers are not cited: RLlib's sources are not available where this project is built, and the restatement follows the
functions named above.

  vtrace64               from_importance_weights on [T, B] tensors in their dtype
  fragments              a recorded [T, B] segment cut into fragments of L rows: fragment f = (time block f // B, episode f % B)
  train_batches          the fragment ranges of the SGD steps
  impala_loss64          VTraceLoss on fragments, given the read-out's logits and values (torch autograd through them)
  impala_learn_replay    ramp_policy_learn_impala from the fragments on: per train batch the read-out at the current weights,
                         V-trace, the loss, its gradient and adam_step
  impala_learn_by_parts  the same loop on the device learner's own parts (loss_and_grad, torch's fp32 Adam step, set_weights)"""
import numpy as np
import torch

from ppo_reference import adam_step, params64, policy64

STAT_KEYS = ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'grad_gnorm', 'mean_rho', 'rows')
FIELDS = ('model', 'graph_features', 'action_mask', 'action', 'behaviour_logp', 'reward', 'done')


def vtrace64(log_rhos, discounts, rewards, values, bootstrap, clip_rho=1.0, clip_pg_rho=1.0):
    """from_importance_weights: [T, B] tensors (bootstrap [B]) -> vs, pg_advantages [T, B], in the inputs' dtype"""
    rhos = torch.exp(log_rhos)
    clipped = torch.clamp_max(rhos, clip_rho)
    cs = torch.clamp_max(rhos, 1.0)
    v1 = torch.cat([values[1:], bootstrap[None]], 0)
    deltas = clipped * (rewards + discounts * v1 - values)
    acc = [torch.zeros_like(bootstrap)]
    for i in reversed(range(len(discounts))):
        acc.append(deltas[i] + discounts[i] * cs[i] * acc[-1])
    vs = torch.flip(torch.stack(acc[1:]), [0]) + values
    vs1 = torch.cat([vs[1:], bootstrap[None]], 0)
    pg = torch.clamp_max(rhos, clip_pg_rho) * (rewards + discounts * vs1 - values)
    return vs.detach(), pg.detach()


def fragments(traj, static, n_models, L):
    """a collect() trajectory ([T, B] arrays) -> the fragments ramp_policy_learn_impala forms, [n_frag, L, ...] (FIELDS): row t of
    fragment f is slot (f // B) L + t of episode f % B.  A row whose episode had finished or had nothing queued has model -1."""
    T, B = traj['model'].shape
    assert T % L == 0
    live = traj['live'] & (traj['model'] < n_models)
    model = np.where(live, traj['model'], -1).astype(np.int32)
    stat = np.stack(static)[np.clip(model, 0, None)]
    dyn = traj['graph_features_dynamic']
    gf = np.concatenate([dyn[..., :9], stat, dyn[..., 9:]], axis=-1).astype(np.float32)
    cols = dict(model=model, graph_features=gf, action_mask=traj['action_mask'].astype(np.uint8), action=traj['action'],
                behaviour_logp=traj['logp'], reward=traj['reward'], done=np.asarray(traj['done'], np.uint8))
    out = {}
    for k, a in cols.items():
        a = np.asarray(a).reshape((T // L, L, B) + np.shape(a)[2:])      # [block, t, b, ...]
        out[k] = np.ascontiguousarray(np.moveaxis(a, 2, 1).reshape((T // L * B, L) + np.shape(a)[3:]))
    return out


def train_batches(n_frag, L, train_batch_size):
    """SGD step k takes fragments [k F, min((k + 1) F, n_frag)), F = train_batch_size // L"""
    F = min(train_batch_size // L, n_frag)
    return [(s, min(s + F, n_frag)) for s in range(0, n_frag, F)]


def impala_loss64(logits, value, batch, cfg):
    """VTraceLoss on n fragments of L rows: logits [n L, A], value [n L] (rows f L + t; any values on rows without decision, which
    are taken as 0); batch: the fragments' FIELDS.  Returns (total loss tensor, statistics, dict(vs, pg_advantages, log_rho) [n, L])."""
    from torch.distributions import Categorical
    dt = logits.dtype
    n, L = np.shape(batch['model'])
    model = torch.as_tensor(np.asarray(batch['model']).reshape(-1))
    dec = model >= 0
    action = torch.as_tensor(np.asarray(batch['action'], np.int64).reshape(-1))
    dist = Categorical(logits=logits)
    logp, ent = dist.log_prob(action), dist.entropy()
    value = torch.where(dec, value, torch.zeros_like(value))
    blogp = torch.as_tensor(np.asarray(batch['behaviour_logp']).reshape(-1), dtype=dt)
    log_rho = torch.where(dec, logp.detach() - blogp, torch.zeros_like(blogp))

    def tm(x):                                                            # _make_time_major: [n L] -> [L, n]
        return x.reshape(n, L).T
    reward = torch.as_tensor(np.asarray(batch['reward']).reshape(-1), dtype=dt)
    done = torch.as_tensor(np.asarray(batch['done']).reshape(-1), dtype=dt)
    v = tm(value)
    vs, pg = vtrace64(tm(log_rho)[:-1], (1.0 - tm(done)[:-1]) * cfg.gamma, tm(reward)[:-1], v[:-1].detach(), v[-1].detach(),
                      cfg.vtrace_clip_rho_threshold, cfg.vtrace_clip_pg_rho_threshold)
    valid = tm(dec.to(dt))[:-1]
    pi = -torch.sum(tm(logp)[:-1] * pg * valid)
    vf = 0.5 * torch.sum(((v[:-1] - vs) * valid) ** 2)
    ent_sum = torch.sum(tm(ent)[:-1] * valid)
    total = pi + vf * cfg.vf_loss_coeff - ent_sum * cfg.entropy_coeff
    rows = int(valid.sum().item())
    rho = torch.exp(tm(log_rho)[:-1])
    stats = dict(total_loss=total.item(), policy_loss=pi.item(), vf_loss=vf.item(), entropy=ent_sum.item() / rows if rows else 0.0,
                 mean_rho=float((rho * valid).sum().item() / rows) if rows else 0.0, rows=rows)
    full_vs = torch.cat([vs, v[-1:].detach()], 0).T
    full_pg = torch.cat([pg, torch.zeros_like(pg[:1])], 0).T
    return total, stats, dict(vs=full_vs.numpy(), pg_advantages=full_pg.numpy(), log_rho=log_rho.reshape(n, L).numpy())


def read_out(p, c, graphs, batch):
    """the read-out of every fragment row at weights p: logits [n L, A], value [n L] (zeros on rows without decision)"""
    model = np.asarray(batch['model']).reshape(-1)
    gf = np.asarray(batch['graph_features']).reshape(len(model), -1)
    mask = np.asarray(batch['action_mask']).reshape(len(model), -1)
    dt = next(iter(p.values())).dtype
    live = np.flatnonzero(model >= 0)
    logits = torch.zeros((len(model), mask.shape[1]), dtype=dt)
    value = torch.zeros(len(model), dtype=dt)
    if len(live):
        lg, v = policy64(p, c, graphs, model[live], gf[live], mask[live])
        idx = torch.as_tensor(live)
        logits = logits.index_put((idx,), lg)
        value = value.index_put((idx,), v)
    return logits, value


def _mean(steps):
    return {k: float(np.mean([s[k] for s in steps])) for k in STAT_KEYS} if steps else {}


def impala_learn_replay(params, c, graphs, batch, cfg, adam_state=None, dtype=torch.float64):
    """ramp_policy_learn_impala restated from its fragments on.  params: the call's starting weights (name -> array, blob order);
    graphs: per job type, objects with nf, ef, src, dst; batch: every fragment's FIELDS ([n_frag, L, ...]); cfg: IMPALAConfig;
    adam_state: (m, v, step) or None.  Per train batch: the read-out at the current weights, impala_loss64, its autograd
    gradient, adam_step.  Returns dict(weights, m, v, step, steps (per SGD step statistics), stats (their means), vtrace (per
    fragment row, as its step computed it))."""
    keys = list(params)
    shapes = [tuple(np.shape(params[k])) for k in keys]
    sizes = [int(np.prod(s)) for s in shapes]
    npdt = np.float64 if dtype == torch.float64 else np.float32

    def unflat(x):
        return dict(zip(keys, (p.reshape(s) for p, s in zip(np.split(x, np.cumsum(sizes)[:-1]), shapes))))
    w = np.concatenate([np.asarray(params[k], dtype=npdt).ravel() for k in keys])
    m, v, step = adam_state if adam_state is not None else (None, None, 0)
    n_frag, L = np.shape(batch['model'])
    steps, vt = [], {k: np.zeros((n_frag, L)) for k in ('vs', 'pg_advantages', 'log_rho')}
    for s, e in train_batches(n_frag, L, cfg.train_batch_size):
        sub = {k: np.asarray(x)[s:e] for k, x in batch.items()}
        pt = params64(unflat(w), dtype=dtype)
        logits, value = read_out(pt, c, graphs, sub)
        total, st, out = impala_loss64(logits, value, sub, cfg)
        gs = torch.autograd.grad(total, list(pt.values()), allow_unused=True)
        g = np.concatenate([(x.numpy() if x is not None else np.zeros(sz, npdt)).ravel() for x, sz in zip(gs, sizes)]).astype(npdt)
        w, m, v, norm = adam_step(w, g, m, v, step, cfg)
        step += 1
        st['grad_gnorm'] = norm
        steps.append(st)
        for k in vt:
            vt[k][s:e] = out[k]
    return dict(weights=unflat(w), m=m, v=v, step=step, steps=steps, stats=_mean(steps), vtrace=vt)


def impala_learn_by_parts(learner, batch, cfg):
    """The loop of one learn call on a DeviceIMPALALearner's own parts: per train batch loss_and_grad at the current weights,
    the fp32 adam_step and policy.set_weights.  Adam starts from the learner's state, which is left as it is; the policy ends with
    the replay's weights.  Returns dict(weights (blob), m, v, step, steps, stats)."""
    from ddls_b200.learn import DeviceIMPALALearner
    pol = learner.policy
    parts = DeviceIMPALALearner(pol, cfg)
    w = pol.get_weights()
    m, v, step = learner.adam_state()
    n_frag, L = np.shape(batch['model'])
    steps = []
    for s, e in train_batches(n_frag, L, cfg.train_batch_size):
        st, g, _ = parts.loss_and_grad({k: np.asarray(x)[s:e] for k, x in batch.items()})
        w, m, v, _ = adam_step(w, g, m, v, step, cfg)
        step += 1
        pol.set_weights(w)
        steps.append(st)
    return dict(weights=w, m=m, v=v, step=step, steps=steps, stats=_mean(steps))
