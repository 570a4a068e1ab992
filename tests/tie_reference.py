"""TEST INFRASTRUCTURE -- ReLU near-ties of the float64 restatement (tests/ppo_reference.py's policy64), and an account of a
kernel's gradient error in terms of them.

An fp32 computation of the policy rounds every pre-activation; one whose float64 value lies within that rounding of 0 may come
out with the other sign, and then takes the other branch of its ReLU.  The forward moves by the pre-activation itself (tiny),
but the backward mask flips: a whole unit's gradient appears or vanishes for one item.  Such a flip is not an error of the
kernel, but it can move a weight tensor's gradient far more than fp32 rounding does.  So a gradient error above the usual bound
is accepted only when it is explained by flips of named near-tied units:

  sites      every ReLU / leaky-ReLU pre-activation a with its margin |a| / (sum_k |w_k y_k| + |b|), y the Linear's input: the
             node, edge, reduce-own and reduce-message items of every round, the read-out's hidden and value-branch units per row
  near_ties  the sites whose margin is below tau, closest first
  deltas     per candidate i, D_i: the float64 gradient with candidate i's branch flipped minus the unflipped one, one autograd run
             each.  The upstream gradient (d loss / d logits, d value) is taken at the unflipped forward: a flip moves the forward
             only by about its margin
  flips      the candidates grouped: ties of the same unit at the same float64 pre-activation (identical rows) flip together
  explain    a small set S of candidates, chosen greedily, such that every tensor of g_kernel - (g64 + sum_{i in S} D_i) is within
             max(1e-4, 10 e32) of ||g64|| (e32: torch fp32's own relative error on the tensor); otherwise an AssertionError that
             names the tensors left unexplained

A site is (module, model, round, item, unit): module 'node' (item: node), 'edge' (edge), 'own' (a node's own state through the
reduce module), 'msg' (an edge's message through the reduce module) with the job type and round, or 'hidden' / 'value' with
model and round -1 and the row as the item."""
import dataclasses

import numpy as np
import torch

from ppo_reference import embed64, head64, params64, policy64

TAU = 1e-4
REL = 1e-4
FP32_FACTOR = 10
MAX_SET = 12
GNN_MODULES = ('node', 'edge', 'own', 'msg')


@dataclasses.dataclass(frozen=True)
class Tie:
    site: tuple            # (module, model, round, item, unit)
    pre: float             # the float64 pre-activation
    margin: float

    def flipped(self):
        """the forced branch that flips this site: the one its float64 pre-activation does not take"""
        return {self.site: not self.pre > 0}

    def __str__(self):
        mod, m, r, i, u = self.site
        where = f'row {i}' if m < 0 else f'model {m} round {r} {"node" if mod in ("node", "own") else "edge"} {i}'
        return f'{mod} {where} unit {u} (pre-activation {self.pre:+.2e}, margin {self.margin:.1e})'


def sites(params, c, graphs, model, graph_features, action_mask):
    """every activation site of the rows' forward in float64: a list of (module, model, round, pre-activation [items, units],
    margin [items, units]).  A zero-in-degree node's own item is left out: its output is the constant 0"""
    out = []

    def record(mod, m, r, pre, y, W, b):
        scale = y.abs() @ W.abs().T + b.abs()
        margin = torch.where(scale > 0, pre.abs() / scale, torch.full_like(pre, np.inf))
        if mod == 'own':
            deg = np.bincount(np.asarray(graphs[m].dst, np.int64), minlength=len(pre))
            margin[torch.as_tensor(deg == 0)] = np.inf
        out.append((mod, m, r, pre.numpy(), margin.numpy()))
    with torch.no_grad():
        policy64(params64(params, requires_grad=False), c, graphs, model, graph_features, action_mask, record=record)
    return out


def near_ties(params, c, graphs, model, graph_features, action_mask, tau=TAU):
    """the sites with margin below tau, closest first (Tie)"""
    ties = []
    for mod, m, r, pre, margin in sites(params, c, graphs, model, graph_features, action_mask):
        for i, u in zip(*np.nonzero(margin < tau)):
            ties.append(Tie((mod, int(m), int(r), int(i), int(u)), float(pre[i, u]), float(margin[i, u])))
    return sorted(ties, key=lambda t: t.margin)


def _grads(out, p, retain=False):
    gs = torch.autograd.grad(out, list(p.values()), allow_unused=True, retain_graph=retain)
    return {k: (g.numpy() if g is not None else np.zeros(tuple(v.shape))) for (k, v), g in zip(p.items(), gs)}


def grad64(params, c, graphs, model, graph_features, action_mask, loss_fn, dtype=torch.float64, forced=None):
    """the gradient of loss_fn(logits, value) at params, in dtype, with the forced branches: (name -> array, d logits, d value)"""
    p = params64(params, dtype=dtype)
    logits, value = policy64(p, c, graphs, model, graph_features, action_mask, forced=forced)
    loss = loss_fn(logits, value)
    gs = torch.autograd.grad(loss, [logits, value] + list(p.values()), allow_unused=True)
    up = [g.detach() if g is not None else torch.zeros_like(x) for g, x in zip(gs[:2], (logits, value))]
    return {k: (g.numpy() if g is not None else np.zeros(tuple(v.shape))) for (k, v), g in zip(p.items(), gs[2:])}, up[0], up[1]


def deltas(params, c, graphs, model, graph_features, action_mask, d_logits, d_value, ties):
    """D_i per tie (name -> array): the float64 gradient of sum(d_logits logits + d_value value) with the tie's branch flipped,
    minus the unflipped one.  A GNN tie moves only its job type's embedding, so it is run through d emb of that job type.  A
    read-out tie moves only its row: the read-out of that row alone is run, and what it changes of d emb is taken through the
    job type's embedding Jacobian (computed once per job type)"""
    model = np.asarray(model)
    gf, mask = np.asarray(graph_features), np.asarray(action_mask)
    gl, gv = torch.as_tensor(d_logits, dtype=torch.float64), torch.as_tensor(d_value, dtype=torch.float64)
    p0 = params64(params, requires_grad=False)
    with torch.no_grad():
        emb = {m: embed64(p0, c, graphs[m].nf, graphs[m].ef, graphs[m].src, graphs[m].dst, m) for m in sorted(set(model.tolist()))}
    need = sorted({t.site[1] for t in ties if t.site[0] in GNN_MODULES})
    d_emb = {}
    if need:
        leaves = {m: e.clone().requires_grad_() for m, e in emb.items()}
        lg, v = head64(p0, c, torch.stack([leaves[m] for m in model.tolist()]), gf, mask)
        gs = torch.autograd.grad((gl * lg).sum() + (gv * v).sum(), [leaves[m] for m in need])
        d_emb = dict(zip(need, gs))
    jac = {}

    def jacobian(m):                                                     # d emb[m] / d params: name -> [out_features_node, ...]
        if m not in jac:
            p, g = params64(params), graphs[m]
            e = embed64(p, c, g.nf, g.ef, g.src, g.dst, m)
            rows_ = [_grads(e[o], p, True) for o in range(len(e))]
            jac[m] = {k: np.stack([r[k] for r in rows_]) for k in p}
        return jac[m]

    def gnn(m, forced):
        p, g = params64(params), graphs[m]
        return _grads((d_emb[m] * embed64(p, c, g.nf, g.ef, g.src, g.dst, m, forced)).sum(), p)

    def row(j, forced):
        p = params64(params)
        leaf = emb[int(model[j])].clone().requires_grad_()
        lg, v = head64(p, c, leaf[None], gf[j:j + 1], mask[j:j + 1], forced)
        gs = torch.autograd.grad((gl[j:j + 1] * lg).sum() + (gv[j:j + 1] * v).sum(), [leaf] + list(p.values()), allow_unused=True)
        out = {k: (g.numpy() if g is not None else np.zeros(tuple(x.shape))) for (k, x), g in zip(p.items(), gs[1:])}
        out['d emb'] = gs[0].numpy()
        return out
    base, out = {}, []
    for t in ties:
        mod, m, r, i, u = t.site
        if mod in GNN_MODULES:
            if ('gnn', m) not in base:
                base['gnn', m] = gnn(m, None)
            flip = gnn(m, t.flipped())
            out.append({k: flip[k] - base['gnn', m][k] for k in flip})
            continue
        b, flip = row(i, None), row(i, {(mod, m, r, 0, u): not t.pre > 0})
        J = jacobian(int(model[i]))
        dd = flip.pop('d emb') - b.pop('d emb')
        out.append({k: flip[k] - b[k] + np.tensordot(dd, J[k], 1) for k in flip})
    return out


@dataclasses.dataclass(frozen=True)
class Flip:
    """ties that flip together: the same unit at the same float64 pre-activation (identical rows, which the kernels compute
    bit for bit alike, so that they take one branch)"""
    ties: tuple

    @property
    def margin(self):
        return self.ties[0].margin

    def __str__(self):
        if len(self.ties) == 1:
            return str(self.ties[0])
        mod, m, r, _, u = self.ties[0].site
        what = 'rows' if m < 0 else ('nodes' if mod in ('node', 'own') else 'edges')
        return (f'{mod} {what} {", ".join(str(t.site[3]) for t in self.ties)}{"" if m < 0 else f" of model {m} round {r}"} unit {u} '
                f'(pre-activation {self.ties[0].pre:+.2e}, margin {self.margin:.1e})')


def flips(ties, deltas_):
    """the candidates of explain(): ties grouped into Flip (same module, job type, round, unit and float64 pre-activation), each
    with the sum of its members' D_i"""
    groups = {}
    for t, d in zip(ties, deltas_):
        mod, m, r, _, u = t.site
        groups.setdefault((mod, m, r, u, t.pre), []).append((t, d))
    out = sorted(groups.values(), key=lambda g: g[0][0].margin)
    return [Flip(tuple(t for t, _ in g)) for g in out], [{k: sum(d[k] for _, d in g) for k in g[0][1]} for g in out]


def bounds(e32):
    """the per tensor bound on ||g - g64|| / ||g64||: max(1e-4, 10 e32)"""
    return {k: max(REL, FP32_FACTOR * e) for k, e in e32.items()}


def _ratios(resid, g64, bound):
    out = {}
    for k, r in resid.items():
        nrm = np.linalg.norm(g64[k])
        out[k] = (np.linalg.norm(r) / nrm if nrm > 0 else np.linalg.norm(r)) / bound[k]
    return out


def explain(g_kernel, g64, deltas_, e32, ties=None, max_set=MAX_SET):
    """a set S of candidates (indices into deltas_, in the order chosen) such that every tensor of g_kernel - (g64 + sum_S D_i)
    is within bounds(e32) relative to ||g64||; returns (S, per tensor relative residuals).  Greedy: while a tensor is outside
    its bound, add the candidate that most lowers sum_k (residual_k / bound_k)^2; an AssertionError when none lowers it or S
    would exceed max_set.  g_kernel, g64, e32: name -> array / relative error; ties: the candidates' Tie, for the message."""
    bound = bounds(e32)
    resid = {k: np.asarray(g_kernel[k], np.float64) - g64[k] for k in g64}
    S = []

    def score(r):
        q = _ratios(r, g64, bound)
        return sum(x * x for x in q.values()), max(q.values())
    cur, worst = score(resid)
    while worst > 1.0:
        best, best_i = None, None
        if len(S) < max_set:
            for i, d in enumerate(deltas_):
                if i in S:
                    continue
                s = score({k: resid[k] - d[k] for k in resid})
                if s[0] < cur and (best is None or s[0] < best[0]):
                    best, best_i = s, i
        if best is None:
            q = _ratios(resid, g64, bound)
            bad = {k: f'{x * bound[k]:.2e} (bound {bound[k]:.1e})' for k, x in q.items() if x > 1.0}
            named = [str(ties[i]) if ties else i for i in S]
            raise AssertionError(f'gradient error not explained by {len(deltas_)} near-tie candidates (chosen: {named}): {bad}')
        S.append(best_i)
        resid = {k: resid[k] - deltas_[best_i][k] for k in resid}
        cur, worst = best
    norms = {k: np.linalg.norm(g64[k]) for k in g64}
    return S, {k: np.linalg.norm(r) / norms[k] if norms[k] > 0 else np.linalg.norm(r) for k, r in resid.items()}
