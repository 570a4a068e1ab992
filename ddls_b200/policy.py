"""The reference's GNN policy on the device (SURVEY.md 8f-3): ``GNNPolicy.forward`` (ml_models/policies/gnn_policy.py:137-296) behind
``ramp_policy_*`` of include/ramp_b200.h.

``DeviceGNNPolicy`` holds one weight set (a flat fp32 blob packed from a ``GNNPolicy`` state_dict, reference key names) and the
static observation of every job type; ``embed()`` runs the MeanPool rounds once per weight set, ``forward()`` evaluates the
read-out on host inputs (what the parity test compares with a plain torch fp32 restatement), ``act(env)`` decides for every episode
of a ``DeviceRampJobPartitioningEnvironment`` without any host transfer: it reads the environment's device buffers and writes its
action buffer, so ``env.step(None)`` after it is one RampJobPartitioningEnvironment.step per episode driven by the policy.

There is no CPU fallback: the CUDA library is required."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import numpy as np

from . import engine as _engine
from .observation import static_observation

ACTIVATIONS = {'relu': 0, 'leaky_relu': 1, 'tanh': 2}

# scripts/ramp_job_partitioning_configs/model/gnn.yaml
DEFAULT_CONFIG = dict(in_features_node=5, in_features_edge=2, in_features_graph=17, out_features_msg=32, out_features_hidden=64,
                      out_features_node=16, out_features_graph=8, num_rounds=2, aggregator_activation='relu', fcnet_hiddens=(256,),
                      fcnet_activation='relu', apply_action_mask=True)


class _Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('in_features_node', 'in_features_edge', 'in_features_graph', 'n_actions', 'out_features_msg',
                                          'out_features_hidden', 'out_features_node', 'out_features_graph', 'num_rounds', 'fcnet_hidden',
                                          'aggregator_activation', 'fcnet_activation', 'apply_action_mask', 'n_models')]


def c_config(config: Dict, n_actions: int, n_models: int) -> _Config:
    """ramp_policy_config_t of a gnn.yaml-style configuration (one read-out hidden layer)"""
    c = config
    return _Config(c['in_features_node'], c['in_features_edge'], c['in_features_graph'], int(n_actions), c['out_features_msg'],
                   c['out_features_hidden'], c['out_features_node'], c['out_features_graph'], c['num_rounds'],
                   tuple(c['fcnet_hiddens'])[0], ACTIVATIONS[c['aggregator_activation']], ACTIVATIONS[c['fcnet_activation']],
                   1 if c['apply_action_mask'] else 0, int(n_models))


def _shaped(name, a, shape):
    """a, refusing any other shape: the library reads exactly that many elements through the raw pointer"""
    if a.shape != tuple(shape):
        raise ValueError(f'{name}: shape {a.shape}, expected {tuple(shape)}')
    return a


def _bind(L):
    if getattr(L, '_policy_bound', False):
        return
    L.ramp_policy_weight_count.restype = C.c_int64
    L.ramp_policy_weight_count.argtypes = [C.POINTER(_Config)]
    L.ramp_policy_create.restype = C.c_int
    L.ramp_policy_create.argtypes = [C.c_int, C.POINTER(_Config), C.POINTER(C.c_void_p)]
    L.ramp_policy_destroy.restype = None
    L.ramp_policy_destroy.argtypes = [C.c_void_p]
    L.ramp_policy_set_weights.restype = C.c_int
    L.ramp_policy_set_weights.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.ramp_policy_set_model.restype = C.c_int
    L.ramp_policy_set_model.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 5
    L.ramp_policy_embed.restype = C.c_int
    L.ramp_policy_embed.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_policy_forward.restype = C.c_int
    L.ramp_policy_forward.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 5
    L.ramp_policy_decide.restype = C.c_int
    L.ramp_policy_decide.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 3 + [C.c_int32, C.c_uint64] + [C.c_void_p] * 4
    L.ramp_policy_act.restype = C.c_int
    L.ramp_policy_act.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_uint64]
    L.ramp_policy_read.restype = C.c_int
    L.ramp_policy_read.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 4
    L.ramp_pinned_alloc.restype = C.c_void_p
    L.ramp_pinned_alloc.argtypes = [C.c_size_t]
    L.ramp_pinned_free.restype = None
    L.ramp_pinned_free.argtypes = [C.c_void_p]
    L.ramp_policy_trajectory_begin.restype = C.c_int
    L.ramp_policy_trajectory_begin.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.ramp_policy_trajectory_record.restype = C.c_int
    L.ramp_policy_trajectory_record.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]
    L.ramp_policy_trajectory_read.restype = C.c_int
    L.ramp_policy_trajectory_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int32] + [C.c_void_p] * 8
    L.ramp_policy_get_weights.restype = C.c_int
    L.ramp_policy_get_weights.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_policy_backward.restype = C.c_int
    L.ramp_policy_backward.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 6
    L._policy_bound = True


def weight_keys(config: Dict) -> Sequence[str]:
    """state_dict keys of the reference's GNNPolicy in blob order (weights then biases per module): gnn_module.layers.{r}.
    {node,edge,reduce}_module.{0: LayerNorm, 1: Linear}; graph_module.{0,1}; the RLlib FullyConnectedNetwork read-out
    (logit_module._hidden_layers.0, ._logits, ._value_branch_separate.0, ._value_branch; each a SlimFC whose Linear is ._model.0)."""
    keys = []
    for r in range(config['num_rounds']):
        for mod in ('node_module', 'edge_module', 'reduce_module'):
            for layer in (0, 1):
                keys += [f'gnn_module.layers.{r}.{mod}.{layer}.weight', f'gnn_module.layers.{r}.{mod}.{layer}.bias']
    keys += ['graph_module.0.weight', 'graph_module.0.bias', 'graph_module.1.weight', 'graph_module.1.bias']
    for name in ('logit_module._hidden_layers.0', 'logit_module._logits', 'logit_module._value_branch_separate.0', 'logit_module._value_branch'):
        keys += [f'{name}._model.0.weight', f'{name}._model.0.bias']
    return keys


def weight_shapes(config: Dict, n_actions: int) -> Dict[str, tuple]:
    c = config
    half, msg = c['out_features_msg'] // 2, c['out_features_msg']
    (H,) = tuple(c['fcnet_hiddens'])
    shapes = {}
    for r in range(c['num_rounds']):
        i = c['in_features_node'] if r == 0 else c['out_features_hidden']
        o = c['out_features_node'] if r == c['num_rounds'] - 1 else c['out_features_hidden']
        p = f'gnn_module.layers.{r}.'
        shapes.update({p + 'node_module.0.weight': (i,), p + 'node_module.0.bias': (i,), p + 'node_module.1.weight': (half, i),
                       p + 'node_module.1.bias': (half,), p + 'edge_module.0.weight': (c['in_features_edge'],),
                       p + 'edge_module.0.bias': (c['in_features_edge'],), p + 'edge_module.1.weight': (half, c['in_features_edge']),
                       p + 'edge_module.1.bias': (half,), p + 'reduce_module.0.weight': (msg,), p + 'reduce_module.0.bias': (msg,),
                       p + 'reduce_module.1.weight': (o, msg), p + 'reduce_module.1.bias': (o,)})
    gin, fin = c['in_features_graph'] + n_actions, c['out_features_node'] + c['out_features_graph']
    shapes.update({'graph_module.0.weight': (gin,), 'graph_module.0.bias': (gin,), 'graph_module.1.weight': (c['out_features_graph'], gin),
                   'graph_module.1.bias': (c['out_features_graph'],)})
    for name, (o, i) in (('logit_module._hidden_layers.0', (H, fin)), ('logit_module._logits', (n_actions, H)),
                         ('logit_module._value_branch_separate.0', (H, fin)), ('logit_module._value_branch', (1, H))):
        shapes[f'{name}._model.0.weight'] = (o, i)
        shapes[f'{name}._model.0.bias'] = (o,)
    return shapes


def pack_weights(state_dict: Dict, config: Dict, n_actions: int) -> np.ndarray:
    """Flat fp32 blob from a GNNPolicy state_dict (torch tensors or arrays); shapes are checked against the configuration."""
    shapes = weight_shapes(config, n_actions)
    parts = []
    for k in weight_keys(config):
        if k not in state_dict:
            raise KeyError(f'state_dict has no {k!r}')
        v = state_dict[k]
        v = v.detach().cpu().numpy() if hasattr(v, 'detach') else np.asarray(v)
        if tuple(v.shape) != shapes[k]:
            raise ValueError(f'{k}: shape {tuple(v.shape)}, the configuration needs {shapes[k]}')
        parts.append(np.ascontiguousarray(v, dtype=np.float32).ravel())
    return np.concatenate(parts)


def unpack_weights(blob, config: Dict, n_actions: int) -> Dict[str, np.ndarray]:
    """The state_dict of a flat blob, reference key names and shapes (pack_weights' inverse)."""
    blob = np.asarray(blob, dtype=np.float32)
    shapes = weight_shapes(config, n_actions)
    out, at = {}, 0
    for k in weight_keys(config):
        n = int(np.prod(shapes[k]))
        out[k] = blob[at:at + n].reshape(shapes[k]).copy()
        at += n
    if at != len(blob):
        raise ValueError(f'blob has {len(blob)} weights, the configuration {at}')
    return out


def random_state_dict(config: Dict, n_actions: int, seed: int = 0) -> Dict[str, np.ndarray]:
    """A random weight set of the right shapes (uniform +-1/sqrt(fan_in) like torch.nn.Linear; LayerNorm gains around 1)."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, shp in weight_shapes(config, n_actions).items():
        if len(shp) == 2:
            out[k] = rng.uniform(-1, 1, shp).astype(np.float32) / np.float32(np.sqrt(shp[1]))
        elif '.0.weight' in k and '_model' not in k:
            out[k] = (1.0 + 0.1 * rng.standard_normal(shp)).astype(np.float32)
        else:
            out[k] = (0.1 * rng.standard_normal(shp)).astype(np.float32)
    return out


class DeviceGNNPolicy:
    def __init__(self, graphs, n_actions: int, config: Optional[Dict] = None, state_dict: Optional[Dict] = None, device: int = 0, seed: int = 0):
        """graphs: the job types (``synth.ForwardGraph``) in the environment's model order; config: gnn.yaml's custom_model_config
        (+ fcnet_hiddens / fcnet_activation); state_dict: a GNNPolicy checkpoint (random weights when omitted)."""
        self.config = dict(DEFAULT_CONFIG)
        self.config.update(config or {})
        if len(tuple(self.config['fcnet_hiddens'])) != 1:
            raise ValueError('the device read-out has one hidden layer (gnn.yaml: fcnet_hiddens [256])')
        if self.config.get('module_depth', 1) != 1:
            raise ValueError('module_depth must be 1 (gnn.yaml)')
        self.n_actions, self.n_models = int(n_actions), len(graphs)
        L = _engine.load_library()
        _bind(L)
        self._L = L
        self._cfg = c_config(self.config, self.n_actions, self.n_models)
        self._h = C.c_void_p()
        _engine._check(L.ramp_policy_create(device, C.byref(self._cfg), C.byref(self._h)))
        self.static = [static_observation(g) for g in graphs]
        for m, st in enumerate(self.static):
            self.set_model(m, st['node_features'], st['edge_features'], st['edges_src'], st['edges_dst'], st['graph_static'])
        self.set_weights(state_dict if state_dict is not None else random_state_dict(self.config, self.n_actions, seed))

    def close(self):
        if getattr(self, '_h', None):
            self._free_trajectory_buffers()
            self._L.ramp_policy_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_model(self, m, node_features, edge_features, edges_src, edges_dst, graph_static):
        c = self.config
        nf = np.ascontiguousarray(node_features, dtype=np.float32)
        src = np.ascontiguousarray(edges_src, dtype=np.int32)
        N, E = (len(nf) if nf.ndim == 2 else -1), (len(src) if src.ndim == 1 else -1)
        _shaped('node_features', nf, (N, c['in_features_node']))
        _shaped('edges_src', src, (E,))
        dst = _shaped('edges_dst', np.ascontiguousarray(edges_dst, dtype=np.int32), (E,))
        ef = _shaped('edge_features', np.ascontiguousarray(edge_features, dtype=np.float32), (E, c['in_features_edge']))
        gs = _shaped('graph_static', np.ascontiguousarray(graph_static, dtype=np.float32), (6,))
        _engine._check(self._L.ramp_policy_set_model(self._h, int(m), len(nf), len(ef), nf.ctypes.data, ef.ctypes.data, src.ctypes.data,
                                                     dst.ctypes.data, gs.ctypes.data))

    def set_weights(self, state_dict):
        blob = state_dict if isinstance(state_dict, np.ndarray) else pack_weights(state_dict, self.config, self.n_actions)
        blob = np.ascontiguousarray(blob, dtype=np.float32)
        _engine._check(self._L.ramp_policy_set_weights(self._h, blob.ctypes.data, len(blob)))

    def get_weights(self) -> np.ndarray:
        """the current weight blob (after a learner step: the updated weights)"""
        out = np.zeros(self._L.ramp_policy_weight_count(C.byref(self._cfg)), dtype=np.float32)
        _engine._check(self._L.ramp_policy_get_weights(self._h, out.ctypes.data))
        return out

    def state_dict(self) -> Dict[str, np.ndarray]:
        """the current weights under the reference's GNNPolicy key names and shapes (loadable into its checkpoint)"""
        return unpack_weights(self.get_weights(), self.config, self.n_actions)

    def backward(self, model, graph_features, action_mask, grad_logits, grad_value) -> np.ndarray:
        """gradient of sum(grad_logits * logits) + sum(grad_value * value) with respect to every weight (blob order) for forward()'s
        inputs: grad_logits [n, |A|], grad_value [n]"""
        model, gf, mask = self._host_inputs(model, graph_features, action_mask)
        n = len(model)
        gl = _shaped('grad_logits', np.ascontiguousarray(grad_logits, dtype=np.float32), (n, self.n_actions))
        gv = _shaped('grad_value', np.ascontiguousarray(grad_value, dtype=np.float32), (n,))
        out = np.zeros(self._L.ramp_policy_weight_count(C.byref(self._cfg)), dtype=np.float32)
        _engine._check(self._L.ramp_policy_backward(self._h, n, model.ctypes.data, gf.ctypes.data, mask.ctypes.data, gl.ctypes.data,
                                                    gv.ctypes.data, out.ctypes.data))
        return out

    def embed(self):
        out = np.zeros((self.n_models, self.config['out_features_node']), dtype=np.float32)
        _engine._check(self._L.ramp_policy_embed(self._h, out.ctypes.data))
        return out

    def forward(self, model, graph_features, action_mask):
        """logits [n, |A|], value [n] for host inputs: model [n], graph_features [n, in_features_graph] (the observation's
        graph_features without the mask), action_mask [n, |A|]."""
        model, gf, mask = self._host_inputs(model, graph_features, action_mask)
        n = len(model)
        logits = np.zeros((n, self.n_actions), dtype=np.float32)
        value = np.zeros(n, dtype=np.float32)
        _engine._check(self._L.ramp_policy_forward(self._h, n, model.ctypes.data, gf.ctypes.data, mask.ctypes.data, logits.ctypes.data,
                                                   value.ctypes.data))
        return logits, value

    def decide(self, model, graph_features, action_mask, sample: bool = False, seed: int = 0):
        """forward() plus act()'s action selection on host inputs: logits [n, |A|], value [n], logp [n] (of the chosen action),
        action [n].  Row b draws with the key (seed, b), the seed used as given.  Rows whose model is outside [0, n_models) get
        zeros and action 0."""
        model, gf, mask = self._host_inputs(model, graph_features, action_mask)
        n = len(model)
        logits = np.zeros((n, self.n_actions), dtype=np.float32)
        value, logp, action = np.zeros(n, dtype=np.float32), np.zeros(n, dtype=np.float32), np.zeros(n, dtype=np.int32)
        _engine._check(self._L.ramp_policy_decide(self._h, n, model.ctypes.data, gf.ctypes.data, mask.ctypes.data, 1 if sample else 0,
                                                  C.c_uint64(seed & (2 ** 64 - 1)), logits.ctypes.data, value.ctypes.data,
                                                  logp.ctypes.data, action.ctypes.data))
        return logits, value, logp, action

    def _host_inputs(self, model, graph_features, action_mask):
        model = np.ascontiguousarray(model, dtype=np.int32)
        n = len(model) if model.ndim == 1 else -1
        _shaped('model', model, (n,))
        gf = _shaped('graph_features', np.ascontiguousarray(graph_features, dtype=np.float32), (n, self.config['in_features_graph']))
        mask = _shaped('action_mask', np.ascontiguousarray(action_mask, dtype=np.uint8), (n, self.n_actions))
        return model, gf, mask

    def act(self, env, sample: bool = False, seed: int = 0):
        """One decision per episode of a DeviceRampJobPartitioningEnvironment, written into its device action buffer; follow with
        ``env.step(None)``.  Nothing is copied to the host."""
        _engine._check(self._L.ramp_policy_act(self._h, env.eng._h, 1 if sample else 0, C.c_uint64(seed & (2 ** 64 - 1))))

    def read(self, env):
        B = env.B
        logits = np.zeros((B, self.n_actions), dtype=np.float32)
        value, logp, actions = np.zeros(B, dtype=np.float32), np.zeros(B, dtype=np.float32), np.zeros(B, dtype=np.int32)
        _engine._check(self._L.ramp_policy_read(self._h, env.eng._h, logits.ctypes.data, value.ctypes.data, logp.ctypes.data, actions.ctypes.data))
        return {'logits': logits, 'value': value, 'logp': logp, 'actions': actions}

    def _trajectory_buffers(self, horizon, B, A):
        """Page-locked host arrays the trajectory is read into (allocated once per shape, re-used by every collect())."""
        key = (horizon, B, A)
        if getattr(self, '_traj_key', None) != key:
            self._free_trajectory_buffers()
            spec = {'graph_features_dynamic': ((horizon, B, 11), C.c_float), 'model': ((horizon, B), C.c_int32),
                    'action_mask': ((horizon, B, A), C.c_uint8), 'action': ((horizon, B), C.c_int32), 'logp': ((horizon, B), C.c_float),
                    'value': ((horizon, B), C.c_float), 'reward': ((horizon, B), C.c_double), 'done': ((horizon, B), C.c_uint8)}
            self._traj_ptrs, self._traj_buf = [], {}
            for k, (shape, ct) in spec.items():
                n = int(np.prod(shape))
                ptr = self._L.ramp_pinned_alloc(n * C.sizeof(ct))
                if not ptr:
                    raise Exception(self._L.ramp_last_error().decode('utf-8', 'replace'))
                self._traj_ptrs.append(ptr)
                self._traj_buf[k] = np.ctypeslib.as_array((ct * n).from_address(ptr)).reshape(shape)
            self._traj_key = key
        return self._traj_buf

    def _free_trajectory_buffers(self):
        for ptr in getattr(self, '_traj_ptrs', []):
            self._L.ramp_pinned_free(ptr)
        self._traj_ptrs, self._traj_buf, self._traj_key = [], {}, None

    def collect(self, env, horizon: int, sample: bool = True, seed: int = 0, reset: bool = True):
        """One rollout segment entirely on the device: ``horizon`` decisions of this policy for every episode of a
        DeviceRampJobPartitioningEnvironment, recorded on the device, read back ONCE.  Returns arrays [horizon, B, ...]:
        what the policy saw (``model`` of the queued job, ``graph_features_dynamic``, ``action_mask``), what it did (``action``,
        ``logp``, ``value``) and what came back (``reward``, ``done`` after the step); ``live`` marks the decisions of episodes that
        were not finished yet.  The arrays are views of page-locked buffers owned by the policy: valid until the next ``collect()`` /
        ``close()`` -- copy what must outlive that."""
        L, h = self._L, self._h
        if reset:
            env.reset()
        _engine._check(L.ramp_policy_trajectory_begin(h, env.eng._h, int(horizon)))
        for t in range(horizon):
            self.act(env, sample=sample, seed=seed + t)
            _engine._check(L.ramp_policy_trajectory_record(h, env.eng._h, t, 0))
            env.step_device()
            _engine._check(L.ramp_policy_trajectory_record(h, env.eng._h, t, 1))
        B, A = env.B, self.n_actions
        buf = self._trajectory_buffers(horizon, B, A)
        _engine._check(L.ramp_policy_trajectory_read(h, env.eng._h, int(horizon), *[buf[k].ctypes.data for k in (
            'graph_features_dynamic', 'model', 'action_mask', 'action', 'logp', 'value', 'reward', 'done')]))
        env.read()                                         # raises what a step would have raised (invalid action, simulation errors)
        out = dict(buf)                                    # views of page-locked arrays: valid until the next collect()
        out['done'] = buf['done'].astype(bool)
        out['live'] = np.concatenate([np.ones((1, B), dtype=bool), ~out['done'][:-1]], axis=0) & (out['model'] >= 0)
        return out
