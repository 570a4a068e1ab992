"""TEST INFRASTRUCTURE -- float64 torch restatements for the PPO learner (ddls_b200/csrc/ramp_policy_learn.cuh):

  policy64       GNNPolicy's forward (tests/gnn_reference.py), vectorised (MeanPool's mailbox mean through index_add), as a function of
                 a state_dict of float64 tensors, so torch.autograd gives every weight's gradient on graphs of 20,000 nodes; pinned to
                 the module restatement GNNPolicy run in float64 in tests/test_ppo_model.py
  ppo_loss64     PPOTorchPolicy.loss (ray/rllib/algorithms/ppo/ppo_torch_policy.py) with torch.distributions.Categorical
  gae64          RLlib compute_advantages (use_gae) per episode of a recorded segment, and the train batch's rows, t-major
  standardize64  RLlib's standardize_fields: (a - mean) / max(1e-4, std)
  adam_step      torch.optim.Adam + clip_grad_norm_ on one flat fp32 parameter"""
import numpy as np
import torch
import torch.nn.functional as F

F32_MIN = float(np.finfo(np.float32).min)


def _ln(x, w, b):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + 1e-5) * w + b


def _act(x, kind):
    if kind == 'relu':
        return torch.relu(x)
    if kind == 'leaky_relu':
        return F.leaky_relu(x, 0.01)
    return torch.tanh(x)


def params64(sd, requires_grad=True, dtype=torch.float64):
    """the weights as tensors; the restatements below compute in their dtype (float32: what torch's own fp32 autograd gives)"""
    return {k: torch.tensor(np.asarray(v.detach().cpu().numpy() if hasattr(v, 'detach') else v), dtype=dtype,
                            requires_grad=requires_grad) for k, v in sd.items()}


def _dtype(p):
    return next(iter(p.values())).dtype


def embed64(p, c, nf, ef, src, dst):
    z = torch.as_tensor(np.asarray(nf), dtype=_dtype(p))
    ef = torch.as_tensor(np.asarray(ef), dtype=_dtype(p)).reshape(len(src), c['in_features_edge'])
    src, dst = torch.as_tensor(np.asarray(src, dtype=np.int64)), torch.as_tensor(np.asarray(dst, dtype=np.int64))
    n, a = z.shape[0], c['aggregator_activation']
    deg = torch.bincount(dst, minlength=n).to(_dtype(p))[:, None]
    for r in range(c['num_rounds']):
        pre = f'gnn_module.layers.{r}.'

        def mod(name, x):
            x = _ln(x, p[pre + name + '.0.weight'], p[pre + name + '.0.bias'])
            return _act(x @ p[pre + name + '.1.weight'].T + p[pre + name + '.1.bias'], a)
        hn, he = mod('node_module', z), mod('edge_module', ef)
        local = mod('reduce_module', torch.cat([hn, torch.zeros_like(hn)], 1))
        msgs = mod('reduce_module', torch.cat([hn[src], he], 1))
        total = local.index_add(0, dst, msgs)
        z = torch.where(deg > 0, total / (deg + 1.0), torch.zeros_like(total))
    return z.mean(0)


def head64(p, c, emb_rows, graph_features, action_mask):
    mask = torch.as_tensor(np.asarray(action_mask), dtype=_dtype(p))
    x = torch.cat([torch.as_tensor(np.asarray(graph_features), dtype=_dtype(p)), mask], 1)
    g = _ln(x, p['graph_module.0.weight'], p['graph_module.0.bias']) @ p['graph_module.1.weight'].T + p['graph_module.1.bias']
    final = torch.cat([emb_rows, g], 1)

    def fc(name, v):
        return v @ p[f'logit_module.{name}._model.0.weight'].T + p[f'logit_module.{name}._model.0.bias']
    fa = c['fcnet_activation']
    logits = fc('_logits', _act(fc('_hidden_layers.0', final), fa))
    value = fc('_value_branch', _act(fc('_value_branch_separate.0', final), fa))[:, 0]
    if c['apply_action_mask']:
        logits = logits + torch.clamp(torch.log(mask), min=F32_MIN)
    return logits, value


def policy64(p, c, graphs, model, graph_features, action_mask):
    """logits, value of the rows (every model must be in range); graphs: objects with nf, ef, src, dst"""
    model = np.asarray(model)
    used = sorted(set(model.tolist()))
    emb = {m: embed64(p, c, graphs[m].nf, graphs[m].ef, graphs[m].src, graphs[m].dst) for m in used}
    rows = torch.stack([emb[m] for m in model.tolist()])
    return head64(p, c, rows, graph_features, action_mask)


def ppo_loss64(logits, value, action, old_logits, adv, vt, cfg):
    """PPOTorchPolicy.loss: (total loss tensor, statistics); the rows are one minibatch, reduce_mean_valid is the mean"""
    from torch.distributions import Categorical, kl_divergence
    action = torch.as_tensor(np.asarray(action, dtype=np.int64))
    old = torch.as_tensor(np.asarray(old_logits), dtype=torch.float64)
    adv = torch.as_tensor(np.asarray(adv), dtype=torch.float64)
    vt = torch.as_tensor(np.asarray(vt), dtype=torch.float64)
    cur, prev = Categorical(logits=logits), Categorical(logits=old)
    ratio = torch.exp(cur.log_prob(action) - prev.log_prob(action))
    clipped = torch.clamp(ratio, 1 - cfg.clip_param, 1 + cfg.clip_param)
    surr = torch.min(adv * ratio, adv * clipped)
    kl, ent = kl_divergence(prev, cur), cur.entropy()
    vf = torch.clamp((value - vt) ** 2, 0, cfg.vf_clip_param)
    total = torch.mean(-surr + cfg.vf_loss_coeff * vf - cfg.entropy_coeff * ent) + cfg.kl_coeff * torch.mean(kl)
    stats = dict(total_loss=total.item(), policy_loss=torch.mean(-surr).item(), vf_loss=torch.mean(vf).item(),
                 entropy=torch.mean(ent).item(), kl=torch.mean(kl).item(),
                 clip_frac=torch.mean((adv * clipped < adv * ratio).double()).item())
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
    """one torch.optim.Adam step after clip_grad_norm_(max_norm=grad_clip) on fp32 copies; returns (w, m, v, norm before clip)"""
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
