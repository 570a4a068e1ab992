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

ALGOS = ('ppo', 'impala', 'pg', 'es')


def algo_model_config(algo: str, n_actions: int) -> Dict:
    """gnn.yaml with the model overrides of scripts/ramp_job_partitioning_configs/algo/{algo}.yaml: fcnet_hiddens [n_actions]
    ("must == action_space.n"); ppo.yaml sets vf_share_layers False, impala / pg / es.yaml leave RLlib's MODEL_DEFAULTS value, True
    (the value layer reads the policy's hidden layer).  DQN / Ape-X keep gnn.yaml's [256] and are not device learners."""
    if algo not in ALGOS:
        raise ValueError(f'no device learner for algorithm {algo!r} (one of {ALGOS})')
    return dict(DEFAULT_CONFIG, fcnet_hiddens=(int(n_actions),), vf_share_layers=algo != 'ppo')


def _shared(config: Dict) -> bool:
    """RLlib's vf_share_layers: absent means gnn.yaml's model, a separate value branch"""
    return bool(config.get('vf_share_layers', False))


class _Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('in_features_node', 'in_features_edge', 'in_features_graph', 'n_actions', 'out_features_msg',
                                          'out_features_hidden', 'out_features_node', 'out_features_graph', 'num_rounds', 'fcnet_hidden',
                                          'aggregator_activation', 'fcnet_activation', 'apply_action_mask', 'n_models',
                                          'vf_share_layers')]


def c_config(config: Dict, n_actions: int, n_models: int) -> _Config:
    """ramp_policy_config_t of a gnn.yaml-style configuration (one read-out hidden layer)"""
    c = config
    return _Config(c['in_features_node'], c['in_features_edge'], c['in_features_graph'], int(n_actions), c['out_features_msg'],
                   c['out_features_hidden'], c['out_features_node'], c['out_features_graph'], c['num_rounds'],
                   tuple(c['fcnet_hiddens'])[0], ACTIVATIONS[c['aggregator_activation']], ACTIVATIONS[c['fcnet_activation']],
                   1 if c['apply_action_mask'] else 0, int(n_models), 1 if _shared(c) else 0)


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
    L.ramp_policy_get_act_count.restype = C.c_int
    L.ramp_policy_get_act_count.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_policy_set_act_count.restype = C.c_int
    L.ramp_policy_set_act_count.argtypes = [C.c_void_p, C.c_uint64]
    L._policy_bound = True


def _readout(config: Dict) -> Sequence[str]:
    names = ['logit_module._hidden_layers.0', 'logit_module._logits', 'logit_module._value_branch_separate.0', 'logit_module._value_branch']
    return [n for n in names if not (_shared(config) and '_separate' in n)]


def weight_keys(config: Dict) -> Sequence[str]:
    """state_dict keys of the reference's GNNPolicy in blob order (weights then biases per module): gnn_module.layers.{r}.
    {node,edge,reduce}_module.{0: LayerNorm, 1: Linear}; graph_module.{0,1}; the RLlib FullyConnectedNetwork read-out
    (logit_module._hidden_layers.0, ._logits, ._value_branch_separate.0, ._value_branch; each a SlimFC whose Linear is ._model.0).
    Under vf_share_layers there is no ._value_branch_separate: ._value_branch reads ._hidden_layers.0's output."""
    keys = []
    for r in range(config['num_rounds']):
        for mod in ('node_module', 'edge_module', 'reduce_module'):
            for layer in (0, 1):
                keys += [f'gnn_module.layers.{r}.{mod}.{layer}.weight', f'gnn_module.layers.{r}.{mod}.{layer}.bias']
    keys += ['graph_module.0.weight', 'graph_module.0.bias', 'graph_module.1.weight', 'graph_module.1.bias']
    for name in _readout(config):
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
    dims = {'logit_module._hidden_layers.0': (H, fin), 'logit_module._logits': (n_actions, H),
            'logit_module._value_branch_separate.0': (H, fin), 'logit_module._value_branch': (1, H)}
    for name in _readout(config):
        o, i = dims[name]
        shapes[f'{name}._model.0.weight'] = (o, i)
        shapes[f'{name}._model.0.bias'] = (o,)
    return shapes


def weight_count(config: Dict, n_actions: int) -> int:
    """the weights of a configuration (ramp_policy_weight_count)"""
    return sum(int(np.prod(v)) for v in weight_shapes(config, n_actions).values())


def pack_weights(state_dict: Dict, config: Dict, n_actions: int) -> np.ndarray:
    """Flat fp32 blob from a GNNPolicy state_dict (torch tensors or arrays); shapes are checked against the configuration, and a
    value branch the configuration's vf_share_layers does not have is refused."""
    shapes = weight_shapes(config, n_actions)
    for k in state_dict:
        if k.startswith('logit_module._value_branch_separate.') and _shared(config):
            raise KeyError(f'state_dict has {k!r}: a separate value branch, but the configuration shares the value layers '
                           '(vf_share_layers)')
    parts = []
    for k in weight_keys(config):
        if k not in state_dict:
            hint = ' (a checkpoint with vf_share_layers?)' if '_value_branch_separate' in k else ''
            raise KeyError(f'state_dict has no {k!r}{hint}')
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

    def act_count(self) -> int:
        """act calls so far, which the draws mix in (act_draw_key's `calls`)"""
        n = C.c_uint64()
        _engine._check(self._L.ramp_policy_get_act_count(self._h, C.byref(n)))
        return n.value

    def set_act_count(self, n: int):
        """resume the draws after n act calls"""
        _engine._check(self._L.ramp_policy_set_act_count(self._h, int(n) & _M64))

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
        return self._collect(env, horizon, lambda t: self.act(env, sample=sample, seed=seed + t), reset)

    def _collect(self, env, horizon: int, act, reset: bool):
        """collect() with act(t) deciding env-step t (this policy's act, or a population's that writes this policy's act outputs)"""
        L, h = self._L, self._h
        if reset:
            env.reset()
        _engine._check(L.ramp_policy_trajectory_begin(h, env.eng._h, int(horizon)))
        for t in range(horizon):
            act(t)
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


GOLDEN = 0x9E3779B97F4A7C15            # ramp_policy_act mixes seed ^ GOLDEN * (its call count)
ROW_MIX = 0xD1342543DE82EF95           # ... then the episode index: splitmix64(seed ^ ROW_MIX * b)
_M64 = 2 ** 64 - 1


def splitmix64(x: int) -> int:
    x = (x + GOLDEN) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def act_draw_key(seed: int, calls: int, b: int) -> int:
    """the 64-bit draw of episode b in a policy's act call number `calls` (from 1) made with `seed` (ramp_policy_head_kernel)"""
    return splitmix64((seed ^ (GOLDEN * calls)) & _M64 ^ ((b * ROW_MIX) & _M64))


def population_draw(seeds: Sequence[int], calls: int, b: int, group_size: int):
    """(group k, local index i, draw) of episode b of a population's act call number `calls`: group k's seed, the population's call
    count and i = b - k group_size -- the draw of episode i of a single policy whose act got seeds[k] on a group_size-episode twin"""
    k = b // group_size
    i = b - k * group_size
    return k, i, act_draw_key(int(seeds[k]) & _M64, calls, i)


def _bind_population(L):
    if getattr(L, '_population_bound', False):
        return
    for name, args in (('ramp_population_create', [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]),
                       ('ramp_population_create_configs', [C.c_void_p, C.c_int32, C.POINTER(_Config), C.POINTER(C.c_void_p)]),
                       ('ramp_population_set_weights', [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]),
                       ('ramp_population_get_weights', [C.c_void_p, C.c_int32, C.c_void_p]),
                       ('ramp_population_act', [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
                       ('ramp_population_embed_ctas', [C.c_void_p, C.c_void_p]),
                       ('ramp_population_copy_sets', [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
                       ('ramp_population_get_act_count', [C.c_void_p, C.c_void_p]),
                       ('ramp_population_set_act_count', [C.c_void_p, C.c_uint64])):
        getattr(L, name).restype = C.c_int
        getattr(L, name).argtypes = args
    L.ramp_population_destroy.restype = None
    L.ramp_population_destroy.argtypes = [C.c_void_p]
    L._population_bound = True


# the ramp_policy_config_t fields the environment and its job types fix: every set of a population shares them
ENV_FIELDS = ('in_features_node', 'in_features_edge', 'in_features_graph', 'n_actions', 'n_models')


class DeviceGNNPolicyPopulation:
    """K weight sets acting on one DeviceRampJobPartitioningEnvironment: its B = K b episodes are K contiguous groups of b, group k
    decided by set k.  Group k's decisions are, bit for bit, those a DeviceGNNPolicy holding set k's weights makes on a b-episode
    environment with the same episode streams (include/ramp_b200.h: ramp_population_*).  The sets may differ in shape: each has
    its own configuration (widths, rounds, read-out, activations), all of them in the same launches.
    DevicePopulationPPOLearner, DevicePopulationIMPALALearner and DevicePopulationPGLearner train the K sets."""

    def __init__(self, graphs, n_actions: int, config=None, state_dicts: Sequence = (), device: int = 0):
        """graphs, n_actions: as DeviceGNNPolicy's; config: one configuration for every set (a dict, as DeviceGNNPolicy's), or a
        sequence of K, set k's completed from DEFAULT_CONFIG; state_dicts: one GNNPolicy state_dict (or blob) per set, of its
        set's shape, K = their number."""
        state_dicts = list(state_dicts)
        if not state_dicts:
            raise ValueError('a population needs at least one state_dict')
        K, n_actions, n_models = len(state_dicts), int(n_actions), len(graphs)
        per_set = config is not None and not isinstance(config, dict)
        configs = list(config) if per_set else [config] * K
        if len(configs) != K:
            raise ValueError(f'{len(configs)} configs for {K} state_dicts')
        configs = [dict(DEFAULT_CONFIG, **(c or {})) for c in configs]
        ccfgs = []
        for k, c in enumerate(configs):               # every set's configuration and shapes are checked before anything is allocated
            if len(tuple(c['fcnet_hiddens'])) != 1:
                raise ValueError(f'configs[{k}]: the device read-out has one hidden layer (gnn.yaml: fcnet_hiddens [256])')
            if c.get('module_depth', 1) != 1:
                raise ValueError(f'configs[{k}]: module_depth must be 1 (gnn.yaml)')
            ccfgs.append(c_config(c, n_actions, n_models))
            for f in ENV_FIELDS:
                if getattr(ccfgs[k], f) != getattr(ccfgs[0], f):
                    raise ValueError(f'configs[{k}]: {f} = {getattr(ccfgs[k], f)}, set 0 has {getattr(ccfgs[0], f)} '
                                     '(the environment fixes it for every set)')
        blobs = []
        for k, sd in enumerate(state_dicts):
            try:
                blob = sd if isinstance(sd, np.ndarray) else pack_weights(sd, configs[k], n_actions)
            except (KeyError, ValueError) as e:
                raise ValueError(f'state_dicts[{k}]: {e}') from None
            blob = np.ascontiguousarray(blob, dtype=np.float32)
            n = weight_count(configs[k], n_actions)
            if blob.shape != (n,):
                raise ValueError(f'state_dicts[{k}]: a blob of shape {blob.shape}, set {k}\'s configuration has {n} weights')
            blobs.append(blob)
        self.K, self.graphs, self.device = K, list(graphs), device
        self.configs = configs
        self.template = DeviceGNNPolicy(graphs, n_actions, configs[0], state_dict=blobs[0], device=device)
        self.config, self.n_actions, self.n_models = self.template.config, self.template.n_actions, self.template.n_models
        self._ccfgs = ccfgs
        self._L = self.template._L
        _bind_population(self._L)
        self._h = C.c_void_p()
        if per_set:
            arr = (_Config * K)(*ccfgs)
            _engine._check(self._L.ramp_population_create_configs(self.template._h, K, arr, C.byref(self._h)))
            first = 0
        else:
            _engine._check(self._L.ramp_population_create(self.template._h, K, C.byref(self._h)))
            first = 1                                   # set 0 holds the template's weights
        for k in range(first, K):
            self.set_weights(k, blobs[k])

    def close(self):
        if getattr(self, '_h', None):
            self._L.ramp_population_destroy(self._h)
            self._h = None
        if getattr(self, 'template', None) is not None:
            self.template.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _set(self, k) -> int:
        k = int(k)
        if not 0 <= k < self.K:
            raise IndexError(f'set {k} outside [0, {self.K})')
        return k

    def weight_count(self, k: int) -> int:
        """the weights of set k's configuration"""
        return int(self._L.ramp_policy_weight_count(C.byref(self._ccfgs[self._set(k)])))

    def set_weights(self, k: int, state_dict):
        """set k's weights: a state_dict of its configuration's shapes, or a blob"""
        k = self._set(k)
        blob = state_dict if isinstance(state_dict, np.ndarray) else pack_weights(state_dict, self.configs[k], self.n_actions)
        blob = np.ascontiguousarray(blob, dtype=np.float32)
        _engine._check(self._L.ramp_population_set_weights(self._h, k, blob.ctypes.data, len(blob)))

    def get_weights(self, k: int) -> np.ndarray:
        out = np.zeros(self.weight_count(k), dtype=np.float32)
        _engine._check(self._L.ramp_population_get_weights(self._h, int(k), out.ctypes.data))
        return out

    def gnn_state_dict(self, k: int) -> Dict[str, np.ndarray]:
        """set k's weights under the reference's GNNPolicy key names and its configuration's shapes"""
        return unpack_weights(self.get_weights(k), self.configs[self._set(k)], self.n_actions)

    def policy(self, k: int) -> DeviceGNNPolicy:
        """a standalone DeviceGNNPolicy with set k's configuration and current weights (e.g. for agents.evaluate)"""
        return DeviceGNNPolicy(self.graphs, self.n_actions, self.configs[self._set(k)], state_dict=self.get_weights(k), device=self.device)

    def group_size(self, env) -> int:
        """b, the episodes of one group; ValueError unless K divides the environment's B"""
        if env.B % self.K:
            raise ValueError(f'{env.B} episodes do not split into {self.K} groups of equal size')
        return env.B // self.K

    def _seeds(self, seed) -> np.ndarray:
        seeds = [seed] * self.K if np.isscalar(seed) else list(seed)
        if len(seeds) != self.K:
            raise ValueError(f'{len(seeds)} seeds for {self.K} sets')
        return np.array([int(s) & _M64 for s in seeds], dtype=np.uint64)

    def act(self, env, sample: bool = False, seed=0):
        """one decision per episode, group k by set k; seed: group k's act seed, one for all or a sequence of K"""
        self.group_size(env)
        seeds = self._seeds(seed)
        _engine._check(self._L.ramp_population_act(self._h, env.eng._h, 1 if sample else 0, seeds.ctypes.data))

    def collect(self, env, horizon: int, sample: bool = True, seed=0, reset: bool = True):
        """DeviceGNNPolicy.collect for every group at once: env-step t acts with seeds seed_k + t; arrays [horizon, B, ...], group k
        in columns k b .. (k + 1) b - 1"""
        self.group_size(env)
        seeds = self._seeds(seed)
        return self.template._collect(env, horizon, lambda t: self.act(env, sample=sample, seed=[int(s) + t for s in seeds]), reset)

    def read(self, env):
        return self.template.read(env)

    def copy_sets(self, dst: Sequence[int], src: Sequence[int]):
        """set src[i]'s weights and torch-Adam state (DevicePopulation{PPO,IMPALA,PG}Learner's) onto set dst[i], every pair in one
        device launch with no host synchronisation; the destinations' embeddings are recomputed by the next act or learn call.
        Refused, naming the pair: a set outside [0, K), two sets of different configurations, a set that is the destination of two
        pairs, a set that is both a source and a destination."""
        d = np.ascontiguousarray(dst, dtype=np.int32).ravel()
        s = np.ascontiguousarray(src, dtype=np.int32).ravel()
        if len(d) != len(s):
            raise ValueError(f'{len(d)} destinations for {len(s)} sources')
        _engine._check(self._L.ramp_population_copy_sets(self._h, len(d), d.ctypes.data, s.ctypes.data))

    def act_count(self) -> int:
        """act calls so far, one count for every group (DeviceGNNPolicy.act_count)"""
        n = C.c_uint64()
        _engine._check(self._L.ramp_population_get_act_count(self._h, C.byref(n)))
        return n.value

    def set_act_count(self, n: int):
        _engine._check(self._L.ramp_population_set_act_count(self._h, int(n) & _M64))

    def embed_ctas(self) -> int:
        """CTAs of the MeanPool launches; each runs the (set, job type) items c, c + ctas, ..."""
        n = C.c_int32()
        _engine._check(self._L.ramp_population_embed_ctas(self._h, C.byref(n)))
        return n.value
