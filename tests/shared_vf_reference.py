"""TEST INFRASTRUCTURE -- the reference's read-out under RLlib's vf_share_layers (impala / pg / es.yaml leave MODEL_DEFAULTS' True):
FullyConnectedNetwork has no _value_branch_separate, and _value_branch reads the policy's hidden layer.

The separate-branch restatements (tests/gnn_reference.py, tests/ppo_reference.py, tests/tie_reference.py) are used unchanged:
the shared read-out is the separate one with the value hidden layer tied to the policy's (expand).  In float64 that computes the
same value from the same hidden activations; through torch the two uses of one tensor sum their gradients, and a gradient taken
with the value hidden layer as its own tensor is folded back onto the policy's (fold).

  GNNPolicy        the module restatement with RLlib's shared-layer FullyConnectedNetwork (state_dict: RLlib's key set)
  head64           gnn_reference.head64 (numpy float64) under either key set
  policy64         ppo_reference.policy64 (torch) under either key set
  check_explained  test_gpu_learn_grad_recorded.check_explained for a policy with shared value layers: the kernel's gradient
                   against float64, with named near-ties flipped through tie_reference.explain()"""
import numpy as np
import torch
from torch import nn

import gnn_reference
import ppo_reference

HID = 'logit_module._hidden_layers.0._model.0.'
SEP = 'logit_module._value_branch_separate.0._model.0.'


def shared(c):
    return bool(c.get('vf_share_layers', False))


def separate_config(c):
    return dict(c, vf_share_layers=False)


def expand(params):
    """the separate-branch key set with the value hidden layer tied to the policy's (the same arrays / tensors)"""
    out = dict(params)
    out[SEP + 'weight'], out[SEP + 'bias'] = params[HID + 'weight'], params[HID + 'bias']
    return out


def fold(grads):
    """a separate-branch gradient of tied weights back onto the shared key set: the policy hidden layer's plus the value's"""
    out = {k: v for k, v in grads.items() if not k.startswith(SEP)}
    for k in ('weight', 'bias'):
        out[HID + k] = grads[HID + k] + grads[SEP + k]
    return out


class _SharedFCN(nn.Module):
    """ray.rllib.models.torch.fcnet.FullyConnectedNetwork with vf_share_layers True: hidden SlimFCs, a logits SlimFC and a value
    SlimFC, both on the last hidden layer"""

    def __init__(self, i, hiddens, n_out, act):
        super().__init__()
        dims = [i] + list(hiddens)
        self._hidden_layers = nn.Sequential(*[gnn_reference.SlimFC(dims[k], dims[k + 1], act) for k in range(len(hiddens))])
        self._logits = gnn_reference.SlimFC(dims[-1], n_out)
        self._value_branch = gnn_reference.SlimFC(dims[-1], 1)

    def forward(self, x):
        h = self._hidden_layers(x)
        return self._logits(h), self._value_branch(h).squeeze(-1)


class GNNPolicy(gnn_reference.GNNPolicy):
    def __init__(self, c, n_actions):
        super().__init__(c, n_actions)
        if shared(c):
            self.logit_module = _SharedFCN(c['out_features_graph'] + c['out_features_node'], c['fcnet_hiddens'], n_actions,
                                           c['fcnet_activation'])


def head64(sd, c, emb_rows, graph_features, action_mask):
    if not shared(c):
        return gnn_reference.head64(sd, c, emb_rows, graph_features, action_mask)
    return gnn_reference.head64(expand(sd), separate_config(c), emb_rows, graph_features, action_mask)


def policy64(p, c, graphs, model, graph_features, action_mask):
    if not shared(c):
        return ppo_reference.policy64(p, c, graphs, model, graph_features, action_mask)
    return ppo_reference.policy64(expand(p), separate_config(c), graphs, model, graph_features, action_mask)


def _pair_value_ties(ties, ds):
    """read-out ties of the separate-branch form: a 'value' site is the same unit of the same row as a 'hidden' one (the same
    pre-activation), and the kernel's shared unit takes one branch for both -- each 'hidden' tie with its 'value' twin's D added"""
    value = {(t.site[3], t.site[4]): d for t, d in zip(ties, ds) if t.site[0] == 'value'}
    out_t, out_d = [], []
    for t, d in zip(ties, ds):
        if t.site[0] == 'value':
            continue
        if t.site[0] == 'hidden':
            twin = value.get((t.site[3], t.site[4]))
            if twin is not None:
                d = {k: d[k] + twin[k] for k in d}
        out_t.append(t)
        out_d.append(d)
    return out_t, out_d


def check_explained(pol, tag, grad, model, gf, mask, loss_fn):
    """the kernel's gradient `grad` (blob, shared key set) of loss_fn(logits, value) over the rows against float64 through
    tie_reference.explain(); returns (S, residuals, the float64 gradient)"""
    from ddls_b200 import policy as P
    from test_gpu_policy_learn import _Static, tensor_errors
    from tie_reference import TAU, deltas, explain, flips, grad64, near_ties
    c, A = pol.config, pol.n_actions
    assert shared(c)
    cx = separate_config(c)
    params = expand(P.unpack_weights(pol.get_weights(), c, A))
    graphs = [_Static(st) for st in pol.static]
    g64x, gl, gv = grad64(params, cx, graphs, model, gf, mask, loss_fn)
    g64 = fold(g64x)
    g32 = fold(grad64(params, cx, graphs, model, gf, mask, loss_fn, dtype=torch.float32)[0])
    e32 = tensor_errors(P.pack_weights(g32, c, A), g64, c, A)
    gk = {k: v.astype(np.float64) for k, v in P.unpack_weights(grad, c, A).items()}
    ties = near_ties(params, cx, graphs, model, gf, mask, TAU)
    errs = tensor_errors(grad, g64, c, A)
    if all(e <= max(1e-4, 10 * e32[k]) for k, e in errs.items()):
        S, resid = [], errs
    else:
        ts, ds = _pair_value_ties(ties, deltas(params, cx, graphs, model, gf, mask, gl.numpy(), gv.numpy(), ties))
        cands, ds = flips(ts, [fold(d) for d in ds])
        S, resid = explain(gk, g64, ds, e32, cands)
        S = [cands[i] for i in S]
    assert all(t.margin < TAU for f in S for t in f.ties)
    k = max(resid, key=lambda x: resid[x] / max(1e-4, 10 * e32[x]))
    print(f'{tag}: {len(model)} rows, {len(ties)} candidates below {TAU:g}; worst {resid[k]:.2e} ({k}, torch fp32 {e32[k]:.2e}); '
          f'S = ' + ('[]' if not S else '[' + '; '.join(map(str, S)) + ']'))
    return S, resid, g64
