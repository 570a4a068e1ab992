"""The device GNN policy as a ``torch.nn.Module``: forward and backward on CUDA tensors, ordered on the caller's stream.

``TorchGNNPolicy`` runs the device policy's kernels (include/ramp_b200.h: ramp_policy_forward_device / _backward_device) on
``torch.cuda.current_stream()`` with no host synchronisation, so a training loop written in torch -- any loss, optimiser or
algorithm -- trains the same model the fused learners train, at the kernels' speed.  It owns one flat fp32 ``nn.Parameter``
``weight`` in blob order (``policy.weight_keys``): what ``torch.optim`` and ``clip_grad_norm_`` see, and what the kernels read.
Checkpoints in the reference's GNNPolicy key set go through ``gnn_state_dict()`` / ``load_gnn_state_dict()``.

The weights are copied to the library on the device when ``(weight.data_ptr(), weight._version)`` changes, which re-embeds the
job types; forwards at fixed weights (a rollout under ``torch.no_grad()``) run the read-out kernel alone.  A row whose model is
outside [0, n_models) -- a finished episode's -1 -- gets logits 0 and value 0 and passes no gradient, as the head kernel rules.
With ``torch_env`` this is one of the two modules of the package that import torch.

A forward under ``torch.no_grad()`` can be captured with ``torch.cuda.graph`` (DESIGN.md §7 g): the graph gathers the rows and runs
the read-out, reading the embeddings from a buffer the module holds for its whole life.  A replay runs no host code, so it cannot
see a weight change: after an optimiser step (or any change to ``weight``), call ``refresh()`` -- or any eager forward -- before the
next replay.  A capture refuses, before anything is enqueued, a forward that would upload weights or re-embed inside the graph,
or that has more rows than an eager forward has staged; backward is not capturable.  A replay is ordered only by the stream it
runs on: replay on the stream the module's eager calls use (torch's current stream).  Staging that a later, larger eager forward
outgrows is kept, not freed, until ``close()``, so a captured forward's buffers stay valid for the graph's life."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import engine as _engine
from . import policy as _policy
from .observation import static_observation

MODEL_INT32, MODEL_INT64 = 0, 1               # include/ramp_b200.h RAMP_MODEL_*


def _bind(L):
    _policy._bind(L)
    for name in ('ramp_policy_set_weights_device', 'ramp_policy_forward_device', 'ramp_policy_backward_device',
                 'ramp_policy_refresh_device'):
        getattr(L, name).restype = C.c_int
    L.ramp_policy_set_weights_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.ramp_policy_refresh_device.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_policy_forward_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64,
                                             C.c_void_p, C.c_void_p, C.c_void_p]
    L.ramp_policy_backward_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]


def gnn_state_dict_of(flat, config: Dict, n_actions: int) -> Dict[str, torch.Tensor]:
    """The reference's GNNPolicy state_dict (CPU fp32 tensors) of a flat weight vector in blob order."""
    flat = flat.detach().cpu().numpy() if isinstance(flat, torch.Tensor) else np.asarray(flat)
    return {k: torch.from_numpy(v) for k, v in _policy.unpack_weights(flat, config, n_actions).items()}


def flat_weights_of(state_dict: Dict, config: Dict, n_actions: int) -> torch.Tensor:
    """The flat fp32 weight vector (CPU) of a GNNPolicy state_dict of numpy arrays or torch tensors (``policy.pack_weights``)."""
    return torch.from_numpy(_policy.pack_weights(state_dict, config, n_actions))


def _config(config: Optional[Dict]) -> Dict:
    out = dict(_policy.DEFAULT_CONFIG)
    out.update(config or {})
    if len(tuple(out['fcnet_hiddens'])) != 1:
        raise ValueError('the device read-out has one hidden layer (gnn.yaml: fcnet_hiddens [256])')
    if out.get('module_depth', 1) != 1:
        raise ValueError('module_depth must be 1 (gnn.yaml)')
    return out


class _PolicyFunction(torch.autograd.Function):
    """(logits, value) of the rows; backward: the weight gradient by ramp_policy_backward_device.  The weight is saved, so an
    in-place change between forward and backward raises torch's version error."""

    @staticmethod
    def forward(ctx, weight, model, gf, mask, module):
        logits, value = module._forward_rows(model, gf, mask)
        ctx.module = module
        ctx.save_for_backward(weight, model, gf, mask)
        return logits, value

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_logits, grad_value):
        weight, model, gf, mask = ctx.saved_tensors
        return ctx.module._backward_rows(weight, model, gf, mask, grad_logits, grad_value), None, None, None, None


class TorchGNNPolicy(torch.nn.Module):
    def __init__(self, graphs, n_actions: int, config: Optional[Dict] = None, state_dict: Optional[Dict] = None, device: int = 0,
                 seed: int = 0):
        """The arguments of ``DeviceGNNPolicy``: graphs (the job types in the environment's model order: ``synth`` graphs, or dicts
        of node_features, edge_features, edges_src, edges_dst and graph_static such as ``TorchRampJobPartitioningEnvironment.static``
        holds), config (gnn.yaml's, or ``policy.algo_model_config``'s), state_dict (a GNNPolicy checkpoint; random weights when
        omitted).  The module owns its own device policy and never touches an engine.  A failed construction frees what it
        allocated."""
        super().__init__()
        self.config = _config(config)
        self.n_actions, self.n_models = int(n_actions), len(graphs)
        self.device = torch.device('cuda', int(device))
        self._h = None
        L = _engine.load_library()
        _bind(L)
        self._L = L
        self._cfg = _policy.c_config(self.config, self.n_actions, self.n_models)
        h = C.c_void_p()
        _engine._check(L.ramp_policy_create(int(device), C.byref(self._cfg), C.byref(h)))
        self._h = h
        try:
            for m, g in enumerate(graphs):
                st = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in g.items()} if isinstance(g, dict) \
                    else static_observation(g)
                nf = np.ascontiguousarray(st['node_features'], dtype=np.float32)
                ef = np.ascontiguousarray(st['edge_features'], dtype=np.float32)
                src = np.ascontiguousarray(st['edges_src'], dtype=np.int32)
                dst = np.ascontiguousarray(st['edges_dst'], dtype=np.int32)
                gs = np.ascontiguousarray(st['graph_static'], dtype=np.float32)
                _engine._check(L.ramp_policy_set_model(h, m, len(nf), len(ef), nf.ctypes.data, ef.ctypes.data, src.ctypes.data,
                                                       dst.ctypes.data, gs.ctypes.data))
            sd = state_dict if state_dict is not None else _policy.random_state_dict(self.config, self.n_actions, seed)
            self.weight = torch.nn.Parameter(flat_weights_of(sd, self.config, self.n_actions).to(self.device))
        except BaseException:
            self.close()
            raise
        self._key = None                               # (data_ptr, _version) of the weights the library holds

    # ---- lifetime ------------------------------------------------------------------------------------------------------
    def close(self):
        """Frees the device policy (waits for its queued work)."""
        if getattr(self, '_h', None):
            self._L.ramp_policy_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- checkpoints ---------------------------------------------------------------------------------------------------
    def gnn_state_dict(self) -> Dict[str, torch.Tensor]:
        """The weights under the reference's GNNPolicy key names and shapes (CPU tensors; ``DeviceGNNPolicy(state_dict=...)`` loads it)."""
        return gnn_state_dict_of(self.weight, self.config, self.n_actions)

    def load_gnn_state_dict(self, state_dict: Dict):
        """Copies a GNNPolicy state_dict (numpy arrays or torch tensors) into ``weight`` in place."""
        flat = flat_weights_of(state_dict, self.config, self.n_actions)
        with torch.no_grad():
            self.weight.copy_(flat.to(self.device))

    # ---- the model -----------------------------------------------------------------------------------------------------
    def forward(self, obs):
        """obs: the torch environment's observation dict -- ``model`` int32 / int64 [..., ], ``graph_features`` float32
        [..., in_features_graph (+ n_actions)] (only the first in_features_graph columns are read, in place when each row's columns
        are contiguous), ``action_mask`` bool [..., n_actions] -- with any leading dimensions.  Returns (logits [..., n_actions],
        value [...]): GNNPolicy's, with + max(log mask, finfo.min) under apply_action_mask.  A row whose model is outside
        [0, n_models) (a finished episode) gets logits 0 and value 0 and passes no gradient."""
        if not isinstance(obs, dict):
            raise TypeError(f'obs must be a dict with model, graph_features and action_mask, not {type(obs).__name__}')
        missing = [k for k in ('model', 'graph_features', 'action_mask') if k not in obs]
        if missing:
            raise ValueError(f'obs has no {missing}')
        model, gf, mask = obs['model'], obs['graph_features'], obs['action_mask']
        for k, t in (('model', model), ('graph_features', gf), ('action_mask', mask)):
            if not isinstance(t, torch.Tensor):
                raise TypeError(f'{k} must be a torch.Tensor, not {type(t).__name__}')
            if t.device != self.device:
                raise ValueError(f'{k} is on {t.device}, the policy on {self.device}')
        if model.dtype not in (torch.int32, torch.int64):
            raise TypeError(f'model must be int32 or int64, not {model.dtype}')
        if gf.dtype != torch.float32:
            raise TypeError(f'graph_features must be float32, not {gf.dtype}')
        if mask.dtype not in (torch.bool, torch.uint8):
            raise TypeError(f'action_mask must be bool (or uint8), not {mask.dtype}')
        lead, G, A = tuple(model.shape), self.config['in_features_graph'], self.n_actions
        if tuple(gf.shape[:-1]) != lead or gf.dim() != len(lead) + 1 or gf.shape[-1] not in (G, G + A):
            raise ValueError(f'graph_features have shape {tuple(gf.shape)}, expected {lead + (G,)} or {lead + (G + A,)}')
        if tuple(mask.shape) != lead + (A,):
            raise ValueError(f'action_mask has shape {tuple(mask.shape)}, expected {lead + (A,)}')
        model = model.reshape(-1).contiguous()
        gf = gf.reshape(-1, gf.shape[-1])
        if gf.stride(-1) != 1 or (gf.shape[0] > 1 and gf.stride(0) < G):
            gf = gf.contiguous()
        mask = mask.reshape(-1, A).contiguous()
        logits, value = _PolicyFunction.apply(self.weight, model, gf, mask, self)
        return logits.reshape(lead + (A,)), value.reshape(lead)

    def refresh(self):
        """Eagerly, on the current stream: uploads ``weight`` and re-embeds the job types, into the buffer a captured forward reads,
        when the weights changed since the last upload; otherwise does nothing.  Call it after an optimiser step and before the next
        replay of a graph that captured the forward (an eager forward does the same)."""
        if not self._h:
            raise RuntimeError('the policy is closed')
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('TorchGNNPolicy.refresh() runs eagerly, before a replay; it cannot be captured')
        stream = self._stream()
        self._upload(self.weight, stream)
        _engine._check(self._L.ramp_policy_refresh_device(self._h, stream))

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _upload(self, weight, stream):
        """the library's weights := `weight` when they are not already (re-embeds on the next call)"""
        key = (weight.data_ptr(), weight._version)
        if key != self._key:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError('CUDA-graph capture refused: the weights changed since they were last uploaded (or never were), '
                                   'so the forward would upload and re-embed inside the graph; call refresh() or an eager forward '
                                   'before capturing')
            w = weight.detach()
            if not w.is_contiguous() or w.dtype != torch.float32 or w.device != self.device:
                raise ValueError(f'weight must be a contiguous float32 tensor on {self.device}')
            _engine._check(self._L.ramp_policy_set_weights_device(self._h, w.data_ptr(), w.numel(), stream))
            self._key = key

    def _rows(self, model, gf, mask):
        dtype = MODEL_INT64 if model.dtype == torch.int64 else MODEL_INT32
        stride = gf.stride(0) if gf.shape[0] > 1 else gf.shape[-1]
        return [model.data_ptr(), dtype, gf.data_ptr(), stride, mask.data_ptr()]

    def _forward_rows(self, model, gf, mask):
        if not self._h:
            raise RuntimeError('the policy is closed')
        n, A = model.shape[0], self.n_actions
        logits = torch.empty((n, A), dtype=torch.float32, device=self.device)
        value = torch.empty((n,), dtype=torch.float32, device=self.device)
        if n:
            stream = self._stream()
            self._upload(self.weight, stream)
            _engine._check(self._L.ramp_policy_forward_device(self._h, stream, n, *self._rows(model, gf, mask), logits.data_ptr(),
                                                              value.data_ptr()))
        return logits, value

    def _backward_rows(self, weight, model, gf, mask, grad_logits, grad_value):
        if not self._h:
            raise RuntimeError('the policy is closed')
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('CUDA-graph capture refused: the backward of TorchGNNPolicy is not capturable')
        n, A = model.shape[0], self.n_actions
        grad = torch.empty(weight.shape, dtype=torch.float32, device=self.device)
        if not n:
            return grad.zero_()
        gl = torch.zeros((n, A), dtype=torch.float32, device=self.device) if grad_logits is None else \
            grad_logits.to(torch.float32).reshape(n, A).contiguous()
        gv = torch.zeros((n,), dtype=torch.float32, device=self.device) if grad_value is None else \
            grad_value.to(torch.float32).reshape(n).contiguous()
        stream = self._stream()
        self._upload(weight, stream)                   # another forward may have run at other weights in between
        _engine._check(self._L.ramp_policy_backward_device(self._h, stream, n, *self._rows(model, gf, mask), gl.data_ptr(),
                                                           gv.data_ptr(), grad.data_ptr()))
        return grad
