"""TEST INFRASTRUCTURE -- float64 torch restatements for the PG learner (ramp_policy_learn_pg, ramp_pg_loss_grad in
ddls_b200/csrc/ramp_policy.cu and ramp_policy_learn.cuh), on top of tests/ppo_reference.py's policy64 and adam_step.

RLlib is not installed; these restate ray 3.0.0.dev0 (the version the reference pins):

  ray/rllib/evaluation/postprocessing.py
    compute_advantages       use_gae False, use_critic False: advantages = discount_cumsum(rewards ++ [last_r], gamma)[:-1],
                             cast to float32; no value targets are used
    discount_cumsum          scipy.signal.lfilter([1], [1, -gamma], x[::-1])[::-1], in float64
  ray/rllib/algorithms/pg/utils.py
    post_process_advantages  compute_advantages(batch, last_r 0.0, gamma, use_gae False, use_critic False), per trajectory --
                             last_r is 0 even for a trajectory cut before its episode ends
  ray/rllib/algorithms/pg/pg_torch_policy.py
    pg_torch_loss            -mean(action_dist.logp(actions) * advantages) over the train batch

Line numbers are not cited: RLlib's sources are not available where this project is built, and the restatement follows the
functions named above.

  discounted_returns   post_process_advantages on a recorded [T, B] segment: each episode's alive slots are one trajectory; the
                       train batch's rows (alive, a queued job in range), t-major
  train_rows           a collect() trajectory -> the train batch as host rows (model, graph_features, action_mask, action, logp,
                       advantage)
  pg_loss64            pg_torch_loss with torch.distributions.Categorical, given the read-out's logits
  pg_learn_replay      ramp_policy_learn_pg from the train batch on: the read-out, pg_loss64, its gradient, adam_step
  pg_learn_by_parts    the same step on the device learner's own parts (loss_and_grad, torch's fp32 Adam step, set_weights)"""
import numpy as np
import torch
from scipy.signal import lfilter

from ppo_reference import adam_step, params64, policy64

STAT_KEYS = ('policy_loss', 'entropy', 'grad_gnorm', 'rows')


def discount_cumsum(x, gamma):
    return lfilter([1], [1, float(-gamma)], np.asarray(x, np.float64)[::-1], axis=0)[::-1]


def discounted_returns(reward, done, model, gamma, n_models):
    """[T, B] arrays of a recorded segment -> (advantage of the train batch's rows as float32 [n] t-major, the float64 values,
    rows [T, B] bool).  Episode b's trajectory is its slots up to and including its first done (or the segment's end: last_r 0)."""
    reward = np.asarray(reward, np.float64)
    T, B = reward.shape
    done = np.asarray(done, bool)
    alive = np.concatenate([np.ones((1, B), bool), ~done[:-1]], 0)
    adv = np.zeros((T, B))
    for b in range(B):
        n = int(alive[:, b].sum())                                       # alive slots are a prefix
        adv[:n, b] = discount_cumsum(np.append(reward[:n, b], 0.0), gamma)[:-1]
    rows = alive & (np.asarray(model) >= 0) & (np.asarray(model) < n_models)
    return adv[rows].astype(np.float32), adv[rows], rows


def train_rows(pol, traj, gamma, H=None):
    """the train batch ramp_policy_learn_pg forms from the first H slots of a collect() trajectory, as host rows"""
    tr = {k: np.asarray(v)[:H] for k, v in traj.items()}
    adv, _, rows = discounted_returns(tr['reward'], tr['done'], tr['model'], gamma, pol.n_models)
    model = tr['model'][rows]
    stat = np.stack([st['graph_static'] for st in pol.static])[model]
    dyn = tr['graph_features_dynamic'][rows]
    gf = np.concatenate([dyn[:, :9], stat, dyn[:, 9:]], axis=1).astype(np.float32)
    return dict(model=model.astype(np.int32), graph_features=gf, action_mask=tr['action_mask'][rows].astype(np.uint8),
                action=tr['action'][rows].astype(np.int32), logp=tr['logp'][rows], advantage=adv)


def pg_loss64(logits, action, adv):
    """pg_torch_loss in the dtype of `logits`: (loss tensor, statistics)"""
    from torch.distributions import Categorical
    dist = Categorical(logits=logits)
    logp = dist.log_prob(torch.as_tensor(np.asarray(action, np.int64)))
    loss = -torch.mean(logp * torch.as_tensor(np.asarray(adv), dtype=logits.dtype))
    return loss, dict(policy_loss=loss.item(), entropy=dist.entropy().mean().item(), rows=len(logp))


def pg_learn_replay(params, c, graphs, batch, cfg, adam_state=None, dtype=torch.float64):
    """ramp_policy_learn_pg restated from its train batch on.  params: the call's starting weights (name -> array, blob order);
    graphs: per job type, objects with nf, ef, src, dst; batch: train_rows' arrays; cfg: PGConfig; adam_state: (m, v, step) or
    None.  An empty batch makes no step.  Returns dict(weights, m, v, step, stats)."""
    keys = list(params)
    shapes = [tuple(np.shape(params[k])) for k in keys]
    sizes = [int(np.prod(s)) for s in shapes]
    npdt = np.float64 if dtype == torch.float64 else np.float32
    w = np.concatenate([np.asarray(params[k], dtype=npdt).ravel() for k in keys])
    m, v, step = adam_state if adam_state is not None else (None, None, 0)
    stats = dict(policy_loss=0.0, entropy=0.0, grad_gnorm=0.0, rows=0)
    if len(batch['model']):
        pt = params64(params, dtype=dtype)
        logits, _ = policy64(pt, c, graphs, batch['model'], batch['graph_features'], batch['action_mask'])
        loss, stats = pg_loss64(logits, batch['action'], batch['advantage'])
        gs = torch.autograd.grad(loss, list(pt.values()), allow_unused=True)
        g = np.concatenate([(x.numpy() if x is not None else np.zeros(sz, npdt)).ravel() for x, sz in zip(gs, sizes)]).astype(npdt)
        w, m, v, stats['grad_gnorm'] = adam_step(w, g, m, v, step, cfg)
        step += 1
    ws = dict(zip(keys, (p.reshape(s) for p, s in zip(np.split(w, np.cumsum(sizes)[:-1]), shapes))))
    return dict(weights=ws, m=m, v=v, step=step, stats=stats)


def pg_learn_by_parts(learner, batch, cfg):
    """one learn call on a DevicePGLearner's own parts: loss_and_grad at the current weights, the fp32 adam_step and
    policy.set_weights.  Adam starts from the learner's state, which is left as it is.  Returns dict(weights (blob), m, v, step,
    stats, grad (blob; None for an empty batch))."""
    from ddls_b200.learn import DevicePGLearner
    pol = learner.policy
    w = pol.get_weights()
    m, v, step = learner.adam_state()
    if not len(batch['model']):
        return dict(weights=w, m=m, v=v, step=step, stats=dict(policy_loss=0.0, entropy=0.0, grad_gnorm=0.0, rows=0), grad=None)
    st, g = DevicePGLearner(pol, cfg).loss_and_grad(batch)
    w, m, v, _ = adam_step(w, g, m, v, step, cfg)
    pol.set_weights(w)
    return dict(weights=w, m=m, v=v, step=step + 1, stats=st, grad=g)
