"""TEST INFRASTRUCTURE -- float64 torch restatements for the PPO learner (ddls_b200/csrc/ramp_policy_learn.cuh):

  policy64       GNNPolicy's forward (tests/gnn_reference.py), vectorised (MeanPool's mailbox mean through index_add), as a function of
                 a state_dict of float64 tensors, so torch.autograd gives every weight's gradient on graphs of 20,000 nodes; pinned to
                 the module restatement GNNPolicy run in float64 in tests/test_ppo_model.py; optionally with named ReLU branches
                 forced and every activation site's inputs recorded (tests/tie_reference.py)
  ppo_loss64     PPOTorchPolicy.loss (ray/rllib/algorithms/ppo/ppo_torch_policy.py) with torch.distributions.Categorical
  gae64          RLlib compute_advantages (use_gae) per episode of a recorded segment, and the train batch's rows, t-major
  standardize64  RLlib's standardize_fields: (a - mean) / max(1e-4, std)
  adam_step      torch.optim.Adam + clip_grad_norm_ on one flat parameter (fp32: torch's own step; float64: the same rule by hand)
  update_kl      RLlib's PPO.update_kl
  shuffle_order  shuffle_pos of ramp_policy_learn.cuh: the batch row at each position of a pass
  learn_replay   ramp_policy_learn from the train batch on: every pass, minibatch, gradient and Adam step of one learn call
  learn_by_parts the same loop run on the device learner's own parts (loss_and_grad, torch's fp32 Adam step, set_weights)

The restatements compute in the dtype of their inputs: float64 is the reference, float32 is torch's own fp32 result, which sets
how close an fp32 computation can be expected to come."""
import numpy as np
import torch
import torch.nn.functional as F

F32_MIN = float(np.finfo(np.float32).min)
M64 = (1 << 64) - 1
STAT_KEYS = ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'kl', 'clip_frac', 'grad_gnorm')


def _ln(x, w, b):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + 1e-5) * w + b


def _act(x, kind, forced=None):
    """the activation; forced: {(item, unit): on} -- those units of the [items, units] pre-activation x take the positive branch
    (on) or the other one whatever x's sign, so that their output moves by |x| and their derivative is the forced branch's"""
    if forced:
        if kind == 'tanh':
            raise ValueError('tanh has no branches to force')
        on = x.detach() > 0
        for (i, u), b in forced.items():
            on[i, u] = bool(b)
        return x * torch.where(on, 1.0, 0.0 if kind == 'relu' else 0.01).to(x.dtype)
    if kind == 'relu':
        return torch.relu(x)
    if kind == 'leaky_relu':
        return F.leaky_relu(x, 0.01)
    return torch.tanh(x)


def _sites(forced, module, model, rnd):
    """forced branches {(module, model, round, item, unit): on} of one module instance -> {(item, unit): on}"""
    return {(s[3], s[4]): b for s, b in (forced or {}).items() if s[:3] == (module, model, rnd)}


def params64(sd, requires_grad=True, dtype=torch.float64):
    """the weights as tensors; the restatements below compute in their dtype (float32: what torch's own fp32 autograd gives)"""
    return {k: torch.tensor(np.asarray(v.detach().cpu().numpy() if hasattr(v, 'detach') else v), dtype=dtype,
                            requires_grad=requires_grad) for k, v in sd.items()}


def _dtype(p):
    return next(iter(p.values())).dtype


def embed64(p, c, nf, ef, src, dst, model=0, forced=None, record=None):
    """GNNPolicy.embed of one job type (`model`).  Its activation sites are named (module, model, round, item, unit), module
    'node' (item: node), 'edge' (edge), 'own' (the reduce module on a node's own state; item: node) or 'msg' (on an edge's
    message; item: edge).  forced: {site: on}, branches taken whatever the pre-activation's sign (_act); record(module, model,
    round, pre-activation, Linear input, weight, bias), when given, sees every activation site's inputs."""
    z = torch.as_tensor(np.asarray(nf), dtype=_dtype(p))
    ef = torch.as_tensor(np.asarray(ef), dtype=_dtype(p)).reshape(len(src), c['in_features_edge'])
    src, dst = torch.as_tensor(np.asarray(src, dtype=np.int64)), torch.as_tensor(np.asarray(dst, dtype=np.int64))
    n, a = z.shape[0], c['aggregator_activation']
    deg = torch.bincount(dst, minlength=n).to(_dtype(p))[:, None]
    for r in range(c['num_rounds']):
        pre = f'gnn_module.layers.{r}.'

        def mod(name, site, x):
            x = _ln(x, p[pre + name + '.0.weight'], p[pre + name + '.0.bias'])
            W, b = p[pre + name + '.1.weight'], p[pre + name + '.1.bias']
            y = x @ W.T + b
            if record is not None:
                record(site, model, r, y.detach(), x.detach(), W.detach(), b.detach())
            return _act(y, a, _sites(forced, site, model, r))
        hn, he = mod('node_module', 'node', z), mod('edge_module', 'edge', ef)
        local = mod('reduce_module', 'own', torch.cat([hn, torch.zeros_like(hn)], 1))
        msgs = mod('reduce_module', 'msg', torch.cat([hn[src], he], 1))
        total = local.index_add(0, dst, msgs)
        z = torch.where(deg > 0, total / (deg + 1.0), torch.zeros_like(total))
    return z.mean(0)


def head64(p, c, emb_rows, graph_features, action_mask, forced=None, record=None):
    """the read-out of the rows.  Its activation sites are ('hidden' | 'value', -1, -1, row, unit): the policy's and the value
    branch's hidden units; forced and record as in embed64"""
    mask = torch.as_tensor(np.asarray(action_mask), dtype=_dtype(p))
    x = torch.cat([torch.as_tensor(np.asarray(graph_features), dtype=_dtype(p)), mask], 1)
    g = _ln(x, p['graph_module.0.weight'], p['graph_module.0.bias']) @ p['graph_module.1.weight'].T + p['graph_module.1.bias']
    final = torch.cat([emb_rows, g], 1)

    def fc(name, v):
        return v @ p[f'logit_module.{name}._model.0.weight'].T + p[f'logit_module.{name}._model.0.bias']
    fa = c['fcnet_activation']

    def hidden(name, site):
        y = fc(name, final)
        if record is not None:
            W, b = (p[f'logit_module.{name}._model.0.{k}'].detach() for k in ('weight', 'bias'))
            record(site, -1, -1, y.detach(), final.detach(), W, b)
        return _act(y, fa, _sites(forced, site, -1, -1))
    logits = fc('_logits', hidden('_hidden_layers.0', 'hidden'))
    value = fc('_value_branch', hidden('_value_branch_separate.0', 'value'))[:, 0]
    if c['apply_action_mask']:
        logits = logits + torch.clamp(torch.log(mask), min=F32_MIN)
    return logits, value


def policy64(p, c, graphs, model, graph_features, action_mask, forced=None, record=None):
    """logits, value of the rows (every model must be in range); graphs: objects with nf, ef, src, dst.  forced: {site: on},
    branches taken whatever the pre-activation's sign; record: sees every activation site's inputs (embed64, head64)"""
    model = np.asarray(model)
    used = sorted(set(model.tolist()))
    emb = {m: embed64(p, c, graphs[m].nf, graphs[m].ef, graphs[m].src, graphs[m].dst, m, forced, record) for m in used}
    rows = torch.stack([emb[m] for m in model.tolist()])
    return head64(p, c, rows, graph_features, action_mask, forced, record)


def _as(x, dt):
    return torch.as_tensor(x if isinstance(x, torch.Tensor) else np.asarray(x), dtype=dt)


def ppo_loss64(logits, value, action, old_logits, adv, vt, cfg):
    """PPOTorchPolicy.loss in the dtype of `logits`: (total loss tensor, statistics); the rows are one minibatch,
    reduce_mean_valid is the mean"""
    from torch.distributions import Categorical, kl_divergence
    dt = logits.dtype
    action = torch.as_tensor(np.asarray(action, dtype=np.int64))
    old, adv, vt = _as(old_logits, dt), _as(adv, dt), _as(vt, dt)
    cur, prev = Categorical(logits=logits), Categorical(logits=old)
    ratio = torch.exp(cur.log_prob(action) - prev.log_prob(action))
    clipped = torch.clamp(ratio, 1 - cfg.clip_param, 1 + cfg.clip_param)
    surr = torch.min(adv * ratio, adv * clipped)
    kl, ent = kl_divergence(prev, cur), cur.entropy()
    vf = torch.clamp((value - vt) ** 2, 0, cfg.vf_clip_param)
    total = torch.mean(-surr + cfg.vf_loss_coeff * vf - cfg.entropy_coeff * ent) + cfg.kl_coeff * torch.mean(kl)
    stats = dict(total_loss=total.item(), policy_loss=torch.mean(-surr).item(), vf_loss=torch.mean(vf).item(),
                 entropy=torch.mean(ent).item(), kl=torch.mean(kl).item(),
                 clip_frac=torch.mean((adv * clipped < adv * ratio).to(dt)).item())
    return total, stats


def gae64(reward, value, done, model, boot, gamma, lam, n_models):
    """[T, B] arrays of a recorded segment + boot [B] (value of the state after the last step) -> advantage, value target of the
    train batch's rows (decisions of episodes not finished yet with a queued job in range), t-major"""
    T, B = reward.shape
    done = np.asarray(done, dtype=bool)
    alive = np.concatenate([np.ones((1, B), bool), ~done[:-1]], 0)
    adv = np.zeros((T, B))
    for b in range(B):
        nxt = 0.0
        for t in range(T - 1, -1, -1):
            if not alive[t, b]:
                continue
            nonterm = 0.0 if done[t, b] else 1.0
            vn = float(boot[b]) if t == T - 1 else float(value[t + 1, b])
            delta = float(reward[t, b]) + gamma * vn * nonterm - float(value[t, b])
            nxt = delta + gamma * lam * nonterm * nxt
            adv[t, b] = nxt
    rows = alive & (model >= 0) & (model < n_models)
    return adv[rows], (adv + np.asarray(value, dtype=np.float64))[rows], rows


def standardize64(a):
    a = np.asarray(a, dtype=np.float64)
    return (a - a.mean()) / max(1e-4, a.std())


def adam_step(w, g, m, v, step, cfg):
    """one torch.optim.Adam step after clip_grad_norm_(max_norm=grad_clip) on a flat parameter, in the dtype of `w`; returns
    (w, m, v, norm before clip).  float32: torch's own step on fp32 copies.  float64: the same rule by hand in torch's form
    (exp_avg.lerp_, exp_avg_sq.mul_().addcmul_(), sqrt(v) / sqrt(bias_correction2) + eps).  step: the steps taken so far (0:
    fresh moments, m and v are ignored)"""
    if np.asarray(w).dtype == np.float64:
        return _adam64(w, g, m, v, step, cfg)
    p = torch.nn.Parameter(torch.tensor(w, dtype=torch.float32))
    opt = torch.optim.Adam([p], lr=cfg.lr, betas=(cfg.adam_beta1, cfg.adam_beta2), eps=cfg.adam_eps, foreach=False)
    if step:
        opt.state[p] = {'step': torch.tensor(float(step)), 'exp_avg': torch.tensor(m, dtype=torch.float32),
                        'exp_avg_sq': torch.tensor(v, dtype=torch.float32)}
    p.grad = torch.tensor(g, dtype=torch.float32)
    norm = float(torch.nn.utils.clip_grad_norm_([p], cfg.grad_clip)) if cfg.grad_clip > 0 else float(torch.linalg.vector_norm(p.grad))
    opt.step()
    st = opt.state[p]
    return p.detach().numpy().copy(), st['exp_avg'].numpy().copy(), st['exp_avg_sq'].numpy().copy(), norm


def _adam64(w, g, m, v, step, cfg):
    w, g = np.asarray(w, np.float64), np.asarray(g, np.float64)
    m = np.asarray(m, np.float64) if step else np.zeros_like(w)
    v = np.asarray(v, np.float64) if step else np.zeros_like(w)
    norm = float(np.sqrt(np.dot(g, g)))
    if cfg.grad_clip > 0:
        g = g * min(1.0, cfg.grad_clip / (norm + 1e-6))
    t = step + 1
    m = m + (1.0 - cfg.adam_beta1) * (g - m)
    v = v * cfg.adam_beta2 + (1.0 - cfg.adam_beta2) * g * g
    bc1, bc2 = 1.0 - cfg.adam_beta1 ** t, 1.0 - cfg.adam_beta2 ** t
    w = w - (cfg.lr / bc1) * (m / (np.sqrt(v) / np.sqrt(bc2) + cfg.adam_eps))
    return w, m, v, norm


def update_kl(kl_coeff, kl, kl_target):
    """RLlib's PPO.update_kl: the coefficient x1.5 when the mean KL is above twice the target, x0.5 when below half of it"""
    if kl > 2.0 * kl_target:
        return kl_coeff * 1.5
    if kl < 0.5 * kl_target:
        return kl_coeff * 0.5
    return kl_coeff


def mix64(x):
    """splitmix64's finaliser (the kernels' splitmix64) on a Python int"""
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def _mix64_np(x):
    with np.errstate(over='ignore'):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def shuffle_order(seed, sgd_pass, n):
    """shuffle_pos of ramp_policy_learn.cuh for pass `sgd_pass` of a learn call with `seed`: the batch row of each position.  A
    four-round Feistel network keyed by mix64(seed ^ mix64(pass + 1)) on the smallest even power of two >= n, each position
    walked through it again until it lands in [0, n)."""
    if n <= 1:
        return np.arange(n)
    key = np.uint64(mix64((int(seed) & M64) ^ mix64(sgd_pass + 1)))
    h = np.uint64(((n - 1).bit_length() + 1) // 2)
    mask = (np.uint64(1) << h) - np.uint64(1)
    x = np.arange(n, dtype=np.uint64)
    todo = np.ones(n, dtype=bool)
    while todo.any():
        L, R = x[todo] >> h, x[todo] & mask
        for r in range(4):
            L, R = R, L ^ (_mix64_np(key ^ np.uint64(r << 40) ^ R) & mask)
        x[todo] = (L << h) | R
        todo = x >= np.uint64(n)
    return x.astype(np.int64)


def _last_pass_mean(passes):
    last = passes[-1] if passes else []
    return {k: float(np.mean([s[k] for s in last])) for k in STAT_KEYS} if last else {}


def learn_replay(params, c, graphs, batch, cfg, adam_state=None, dtype=torch.float64):
    """ramp_policy_learn restated from the train batch on, as its kernels document it.

    params: the call's starting weights (name -> array, in blob order); c: the policy configuration; graphs: per job type, objects
    with nf, ef, src, dst; batch: the train batch's rows (model, graph_features, action_mask, action, advantage, value_target);
    cfg: the call's PPOConfig (its seed and kl_coeff as the call uses them); adam_state: (m, v, step) flat in blob order, or None
    (fresh moments).  The old logits are taken once, at the starting weights.  Pass p cuts shuffle_order(cfg.seed, p, n) into
    consecutive slices of sgd_minibatch_size rows -- the last may be short, and its loss is the mean over its own rows -- and
    each slice takes ppo_loss64 at the current weights, its autograd gradient and adam_step.

    Returns dict(weights (name -> array), m, v (flat), step, minibatches ([pass][slice] statistics, with grad_gnorm (before
    clipping) and rows), stats (the mean of the last pass's), kl_coeff (update_kl's new coefficient))."""
    keys = list(params)
    shapes = [tuple(np.shape(params[k])) for k in keys]
    sizes = [int(np.prod(s)) for s in shapes]
    npdt = np.float64 if dtype == torch.float64 else np.float32

    def unflat(x):
        return dict(zip(keys, (p.reshape(s) for p, s in zip(np.split(x, np.cumsum(sizes)[:-1]), shapes))))
    w = np.concatenate([np.asarray(params[k], dtype=npdt).ravel() for k in keys])
    m, v, step = adam_state if adam_state is not None else (None, None, 0)
    model, gf, mask = np.asarray(batch['model']), np.asarray(batch['graph_features']), np.asarray(batch['action_mask'])
    action, adv, vt = np.asarray(batch['action']), np.asarray(batch['advantage']), np.asarray(batch['value_target'])
    n, mb = len(model), cfg.sgd_minibatch_size
    with torch.no_grad():
        old, _ = policy64(params64(params, requires_grad=False, dtype=dtype), c, graphs, model, gf, mask)
    passes = []
    for p in range(cfg.num_sgd_iter):
        order, out = shuffle_order(cfg.seed, p, n), []
        for s in range(0, n, mb):
            idx = order[s:s + mb]
            pt = params64(unflat(w), dtype=dtype)
            logits, value = policy64(pt, c, graphs, model[idx], gf[idx], mask[idx])
            total, st = ppo_loss64(logits, value, action[idx], old[torch.as_tensor(idx)], adv[idx], vt[idx], cfg)
            gs = torch.autograd.grad(total, list(pt.values()), allow_unused=True)
            g = np.concatenate([(x.numpy() if x is not None else np.zeros(sz, npdt)).ravel() for x, sz in zip(gs, sizes)]).astype(npdt)
            w, m, v, norm = adam_step(w, g, m, v, step, cfg)
            step += 1
            st.update(grad_gnorm=norm, rows=len(idx))
            out.append(st)
        passes.append(out)
    stats = _last_pass_mean(passes)
    kl_coeff = update_kl(cfg.kl_coeff, stats['kl'], cfg.kl_target) if stats else cfg.kl_coeff
    return dict(weights=unflat(w), m=m, v=v, step=step, minibatches=passes, stats=stats, kl_coeff=kl_coeff)


def learn_by_parts(learner, batch, cfg):
    """The loop of one learn call run on a DevicePPOLearner's own parts: for every pass the slices learn_replay takes, each
    DevicePPOLearner.loss_and_grad at the current weights, the fp32 adam_step and policy.set_weights.  batch: the train batch
    with old_logits (the policy's logits at the call's starting weights); cfg: the call's PPOConfig.  Adam starts from the
    learner's state, which is left as it is; the policy ends with the replay's weights.  Returns learn_replay's dict, without
    kl_coeff and with the weights as a blob."""
    from ddls_b200.learn import DevicePPOLearner
    pol = learner.policy
    parts = DevicePPOLearner(pol, cfg)
    w = pol.get_weights()
    m, v, step = learner.adam_state()
    n, mb = len(batch['model']), cfg.sgd_minibatch_size
    passes = []
    for p in range(cfg.num_sgd_iter):
        order, out = shuffle_order(cfg.seed, p, n), []
        for s in range(0, n, mb):
            idx = order[s:s + mb]
            st, g = parts.loss_and_grad({k: x[idx] for k, x in batch.items()})
            w, m, v, _ = adam_step(w, g, m, v, step, cfg)
            step += 1
            pol.set_weights(w)
            out.append(st)
        passes.append(out)
    return dict(weights=w, m=m, v=v, step=step, minibatches=passes, stats=_last_pass_mean(passes))
