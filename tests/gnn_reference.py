"""TEST INFRASTRUCTURE -- a plain PyTorch fp32 restatement of the reference's GNN policy, module for module, with the reference's
parameter names so that its state_dict is what a GNNPolicy checkpoint holds:

  MeanPool   ml_models/models/mean_pool.py:38-150 (node / edge / reduce modules; per destination node the mean of reduce_module over
             [own (node | zeros) state, mailbox]); DGL is not installed here, so update_all is spelled out per node -- a node with no
             incoming edge gets zeros, which is what dgl fills in for nodes its reduce function is never called on
  GNN        ml_models/models/gnn.py:36-92
  GNNPolicy  ml_models/policies/gnn_policy.py:56-296 (graph module, RLlib FullyConnectedNetwork read-out with a separate value
             branch, log-mask on the logits)

The CUDA path (ddls_b200/csrc/ramp_policy.cu) is compared with this in tests/test_gpu_policy.py, and with the float64 numpy
restatement at the end of this file (embed64 / head64) in tests/test_gpu_policy_kernels.py."""
import numpy as np
import torch
from torch import nn

ACT = {'relu': nn.ReLU, 'leaky_relu': nn.LeakyReLU, 'tanh': nn.Tanh}


class MeanPool(nn.Module):
    def __init__(self, in_node, in_edge, msg, out, act):
        super().__init__()
        self.node_module = nn.Sequential(nn.LayerNorm(in_node), nn.Linear(in_node, msg // 2), ACT[act]())
        self.edge_module = nn.Sequential(nn.LayerNorm(in_edge), nn.Linear(in_edge, msg // 2), ACT[act]())
        self.reduce_module = nn.Sequential(nn.LayerNorm(msg), nn.Linear(msg, out), ACT[act]())
        self.msg = msg

    def forward(self, z, ef, src, dst):
        n = z.shape[0]
        m = torch.cat((self.node_module(z[src]), self.edge_module(ef)), -1)              # mp_func, one message per edge
        local = torch.cat((self.node_module(z), z.new_zeros(n, self.msg // 2)), -1)      # reduce_func's own state
        out = []
        for v in range(n):
            inbox = m[dst == v]
            if inbox.shape[0] == 0:
                out.append(z.new_zeros(self.reduce_module[1].out_features))
                continue
            states = torch.cat((local[v:v + 1], inbox), 0)
            out.append(torch.mean(self.reduce_module(states), dim=0))
        return torch.stack(out)


class GNN(nn.Module):
    def __init__(self, c):
        super().__init__()
        dims = [c['in_features_node']] + [c['out_features_hidden']] * (c['num_rounds'] - 1) + [c['out_features_node']]
        self.layers = nn.ModuleList([MeanPool(dims[r], c['in_features_edge'], c['out_features_msg'], dims[r + 1], c['aggregator_activation'])
                                     for r in range(c['num_rounds'])])

    def forward(self, z, ef, src, dst):
        for layer in self.layers:
            z = layer(z, ef, src, dst)
        return z


class SlimFC(nn.Module):
    def __init__(self, i, o, act=None):
        super().__init__()
        self._model = nn.Sequential(*([nn.Linear(i, o)] + ([ACT[act]()] if act else [])))

    def forward(self, x):
        return self._model(x)


class FullyConnectedNetwork(nn.Module):
    """ray.rllib.models.torch.fcnet.FullyConnectedNetwork with vf_share_layers False: hidden SlimFCs, a logits SlimFC, and the
    same stack again for the value."""

    def __init__(self, i, hiddens, n_out, act):
        super().__init__()
        dims = [i] + list(hiddens)
        self._hidden_layers = nn.Sequential(*[SlimFC(dims[k], dims[k + 1], act) for k in range(len(hiddens))])
        self._logits = SlimFC(dims[-1], n_out)
        self._value_branch_separate = nn.Sequential(*[SlimFC(dims[k], dims[k + 1], act) for k in range(len(hiddens))])
        self._value_branch = SlimFC(dims[-1], 1)

    def forward(self, x):
        return self._logits(self._hidden_layers(x)), self._value_branch(self._value_branch_separate(x)).squeeze(-1)


class GNNPolicy(nn.Module):
    def __init__(self, c, n_actions):
        super().__init__()
        self.c = c
        self.gnn_module = GNN(c)
        gin = c['in_features_graph'] + n_actions
        self.graph_module = nn.Sequential(nn.LayerNorm(gin), nn.Linear(gin, c['out_features_graph']))
        self.logit_module = FullyConnectedNetwork(c['out_features_graph'] + c['out_features_node'], c['fcnet_hiddens'], n_actions,
                                                  c['fcnet_activation'])

    def embed(self, node_features, edge_features, src, dst):
        return torch.mean(self.gnn_module(node_features, edge_features, src, dst), 0)

    def forward(self, emb_nodes, graph_features_and_mask, action_mask):
        """emb_nodes [n, out_node] (the node mean of each observation's job), graph_features_and_mask [n, in_graph + |A|] (the
        observation's 'graph_features'), action_mask [n, |A|]"""
        final = torch.cat((emb_nodes, self.graph_module(graph_features_and_mask)), dim=1)
        logits, value = self.logit_module(final)
        if self.c['apply_action_mask']:
            logits = logits + torch.maximum(torch.log(action_mask), torch.tensor(torch.finfo(torch.float32).min))
        return logits, value


# ---- the same forward in numpy float64, vectorised (a 20,000-node graph takes seconds), for the CUDA kernels' tolerance tests
# (tests/test_gpu_policy_kernels.py).  It follows the module restatement above rule for rule and is pinned to it, run in float64,
# in tests/test_policy_weights.py.

F32_MIN = float(np.finfo(np.float32).min)


def _act64(x, kind):
    if kind == 'relu':
        return np.maximum(x, 0.0)
    if kind == 'leaky_relu':
        return np.where(x > 0, x, 0.01 * x)
    return np.tanh(x)


def _ln64(x, w, b, eps=1e-5):
    mean = x.mean(-1, keepdims=True)
    var = ((x - mean) ** 2).mean(-1, keepdims=True)            # biased, like torch.nn.LayerNorm
    return (x - mean) / np.sqrt(var + eps) * w + b


def _f64(sd):
    return {k: np.asarray(v.detach().cpu().numpy() if hasattr(v, 'detach') else v, dtype=np.float64) for k, v in sd.items()}


def embed64(sd, c, node_features, edge_features, src, dst):
    """GNNPolicy.embed in float64: num_rounds MeanPool rounds, then the mean over the nodes -> [out_features_node]"""
    w = _f64(sd)
    z = np.asarray(node_features, dtype=np.float64)
    ef = np.asarray(edge_features, dtype=np.float64).reshape(len(src), c['in_features_edge'])
    src, dst = np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)
    n, a = len(z), c['aggregator_activation']
    deg = np.bincount(dst, minlength=n)
    for r in range(c['num_rounds']):
        p = f'gnn_module.layers.{r}.'

        def mod(name, x):
            x = _ln64(x, w[p + name + '.0.weight'], w[p + name + '.0.bias'])
            return _act64(x @ w[p + name + '.1.weight'].T + w[p + name + '.1.bias'], a)
        hn, he = mod('node_module', z), mod('edge_module', ef)
        local = mod('reduce_module', np.concatenate([hn, np.zeros_like(hn)], 1))                  # own (node | zeros) state
        msgs = mod('reduce_module', np.concatenate([hn[src], he], 1))                            # one message per edge
        total = local.copy()
        np.add.at(total, dst, msgs)
        z = np.where(deg[:, None] > 0, total / (deg[:, None] + 1.0), 0.0)                        # zero in-degree -> zeros
    return z.mean(0)


def head64(sd, c, emb_rows, graph_features, action_mask):
    """GNNPolicy.forward in float64 for a batch: emb_rows [n, out_features_node], graph_features [n, in_features_graph] (without
    the mask), action_mask [n, |A|] -> logits [n, |A|], value [n]"""
    w = _f64(sd)
    mask = np.asarray(action_mask, dtype=np.float64)
    x = np.concatenate([np.asarray(graph_features, dtype=np.float64), mask], 1)
    g = _ln64(x, w['graph_module.0.weight'], w['graph_module.0.bias']) @ w['graph_module.1.weight'].T + w['graph_module.1.bias']
    final = np.concatenate([np.asarray(emb_rows, dtype=np.float64), g], 1)

    def fc(name, v):
        return v @ w[f'logit_module.{name}._model.0.weight'].T + w[f'logit_module.{name}._model.0.bias']
    fa = c['fcnet_activation']
    logits = fc('_logits', _act64(fc('_hidden_layers.0', final), fa))
    value = fc('_value_branch', _act64(fc('_value_branch_separate.0', final), fa))[:, 0]
    if c['apply_action_mask']:
        with np.errstate(divide='ignore'):
            logits = logits + np.maximum(np.log(mask), F32_MIN)
    return logits, value
