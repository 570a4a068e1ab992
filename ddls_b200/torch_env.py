"""The device environment with PyTorch CUDA tensors in and out, ordered on the caller's stream.

``TorchRampJobPartitioningEnvironment`` wraps a ``DeviceRampJobPartitioningEnvironment``: ``step(actions)`` takes an int32 or int64
CUDA tensor [B] and returns the reference's observation (``model`` [B] int64, ``graph_features`` [B, 17 + |A|] float32 in
RampJobPartitioningObservation's layout, ``action_mask`` [B, |A|] bool), ``reward`` [B] float64 and ``done`` [B] bool as CUDA tensors.
Every kernel that touches a tensor runs on ``torch.cuda.current_stream()`` (include/ramp_b200.h: ramp_env_ingest / ramp_env_export),
so a torch policy feeds the environment and reads it back at device speed, and the caching allocator never needs ``record_stream``.
What the policy observes of a job type whatever the cluster holds -- node and edge features, edge endpoints, the six per-graph
statistics -- is ``static``, uploaded once per job type.  With ``torch_policy`` it is one of the two modules of the package that
import torch.

``step`` can be captured with ``torch.cuda.graph`` and replayed (DESIGN.md §7 g): a replay gives the bits an eager step gives.  Each
replayed step reads its actions from the tensor captured (copy the next actions into it before ``g.replay()``) and writes the
outputs captured (``out=`` tensors, or the graph pool's tensors the captured call returned).  A capture needs the device tables to
decide every placement (``prewarm=True``, no model that splits its ops unevenly), every template on the thread kernel, and an
eager step since the last template was registered; otherwise ``step`` refuses it before anything is enqueued.  ``reset()`` and
``record_steps()`` stay eager, and a graph replays correctly after any number of resets.  Replay on the stream the environment's
other calls then run on (torch's current stream): those calls order the engine behind it."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import engine as _engine
from .batched import DeviceRampJobPartitioningEnvironment
from .observation import static_observation

ACTIONS_INT32, ACTIONS_INT64 = 0, 1           # include/ramp_b200.h RAMP_ACTIONS_*
N_GRAPH_FEATURES = 17                          # graph_features columns before the action mask
OUTPUTS = ('model', 'graph_features', 'action_mask', 'reward', 'done')


class _Export(C.Structure):
    _fields_ = [('model', C.c_void_p), ('graph_features', C.c_void_p), ('action_mask', C.c_void_p), ('reward', C.c_void_p),
                ('done', C.c_void_p)]


def _bind(L):
    for name in ('ramp_env_set_graph_static', 'ramp_env_ingest', 'ramp_env_export'):
        getattr(L, name).restype = C.c_int
    L.ramp_env_set_graph_static.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_env_ingest.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    L.ramp_env_export.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(_Export)]
    L.ramp_env_join.restype = C.c_int
    L.ramp_env_join.argtypes = [C.c_void_p, C.c_void_p]


def static_tensors(graphs, device='cpu'):
    """Per job type: ``node_features`` [N, 5], ``edge_features`` [E, 2] float32, ``edges_src`` / ``edges_dst`` [E] int64 and
    ``graph_static`` [6] float32 -- ``observation.static_observation`` as tensors on `device`, what GNNPolicy embeds."""
    out = []
    for g in graphs:
        st = static_observation(g)
        out.append({'node_features': torch.from_numpy(st['node_features']).to(device),
                    'edge_features': torch.from_numpy(st['edge_features']).to(device),
                    'edges_src': torch.from_numpy(st['edges_src'].astype(np.int64)).to(device),
                    'edges_dst': torch.from_numpy(st['edges_dst'].astype(np.int64)).to(device),
                    'graph_static': torch.from_numpy(st['graph_static']).to(device)})
    return out


class TorchRampJobPartitioningEnvironment:
    def __init__(self, *args, prewarm: bool = False, place_on_device: bool = False, **kw):
        """The arguments of ``DeviceRampJobPartitioningEnvironment`` (``device`` picks cuda:<device>; ``place_on_device`` places
        jobs whose ops split unevenly on the device).  A failed construction frees what it allocated."""
        env = DeviceRampJobPartitioningEnvironment.__new__(DeviceRampJobPartitioningEnvironment)
        try:
            env.__init__(*args, prewarm=prewarm, place_on_device=place_on_device, **kw)
            self.env = env
            self.device = torch.device('cuda', int(kw.get('device', 0)))
            self.B, self.n_actions = env.B, env.max_partitions_per_op + 1
            self._L, self._h = env.eng._L, env.eng._h
            _bind(self._L)
            self.static = static_tensors([m.graph for m in env.models], self.device)
            table = np.ascontiguousarray(np.stack([st['graph_static'].cpu().numpy() for st in self.static]), dtype=np.float32)
            _engine._check(self._L.ramp_env_set_graph_static(self._h, table.ctypes.data))
        except BaseException:
            eng = getattr(env, 'eng', None)
            if eng is not None:
                eng.close()
            raise

    # ---- pass-throughs (each first orders the engine stream behind the caller's, so it sees replayed steps) ------------------
    def episode_stats(self):
        self._join()
        return self.env.episode_stats()

    def decisions(self):
        """[B] env-steps every episode has taken since reset(): the device's count, replayed steps included."""
        self._join()
        return self.env.decisions()

    def record_steps(self, horizon: int):
        """Eager only.  Once a step has been captured, the record keeps its buffers: only its own horizon is accepted (the record
        is cleared), as captured steps write it at its address."""
        self._join()
        self.env.record_steps(horizon)

    def recorded_steps(self):
        self._join()
        return self.env.recorded_steps()

    def close(self):
        env = getattr(self, 'env', None)
        if env is not None:
            try:
                self._join()                           # a replay still queued on the caller's stream ends before the free
            finally:
                self.env = None
                env.close()

    def _join(self):
        _engine._check(self._L.ramp_env_join(self._h, torch.cuda.current_stream(self.device).cuda_stream))

    # ---- the environment -----------------------------------------------------------------------------------------------
    def check(self):
        """Synchronises and raises what the steps since the last check deferred: an action outside the action set, an action
        the mask forbids (apply_action_mask=True), a simulation error -- replayed steps' included, with an eager step's episode and
        message.  Inside a capture it does nothing: call it after the replays."""
        if torch.cuda.is_current_stream_capturing():
            return
        self._join()
        _engine._check(self._L.ramp_env_read(self._h, None, None, None, None, None))

    def reset(self):
        """RampJobPartitioningEnvironment.reset for every episode; the first observation: {model, graph_features, action_mask}.
        Eager only: it draws the arrival streams on the host."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('CUDA-graph capture refused: reset() draws the arrival streams on the host and stays eager')
        self._join()
        self.env.reset()
        obs = self._export(None)
        return {k: obs[k] for k in ('model', 'graph_features', 'action_mask')}

    def step(self, actions: torch.Tensor, out=None):
        """One RampJobPartitioningEnvironment.step per episode.  actions: int32 / int64 [B] on this environment's device.  Returns
        (obs, reward, done, info): fresh tensors, or the tensors of ``out`` (a dict keyed by 'model', 'graph_features',
        'action_mask', 'reward', 'done'; any subset) written in place.  Does not synchronise when the device tables decide every
        placement (``prewarm=True``, no model splits its ops unevenly); errors then surface at ``check()`` or the next synchronising
        call.  Otherwise the host's placer decides the rest, as ``step_device()`` does.

        Inside ``torch.cuda.graph`` the call is captured; see the module's docstring for what a capture needs.  ``step_counter`` is
        a host counter: it counts the captured call once and replays do not advance it (``decisions()`` is the device's count)."""
        if not isinstance(actions, torch.Tensor):
            raise TypeError(f'actions must be a torch.Tensor, not {type(actions).__name__}')
        if actions.dtype not in (torch.int32, torch.int64):
            raise TypeError(f'actions must be int32 or int64, not {actions.dtype}')
        if actions.device != self.device:
            raise ValueError(f'actions are on {actions.device}, the environment on {self.device}')
        if tuple(actions.shape) != (self.B,):
            raise ValueError(f'actions have shape {tuple(actions.shape)}, expected ({self.B},)')
        if torch.cuda.is_current_stream_capturing() and not self.env._device_decides_everything:
            raise RuntimeError('CUDA-graph capture refused: the device tables do not decide every placement (the environment is '
                               "not prewarmed, or a model splits its ops unevenly), so a step may need the host's placer")
        actions = actions.contiguous()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        dtype = ACTIONS_INT64 if actions.dtype == torch.int64 else ACTIONS_INT32
        _engine._check(self._L.ramp_env_ingest(self._h, actions.data_ptr(), dtype, stream))
        self.env.step_device()                         # decides and steps on the actions the ingest kernel wrote
        res = self._export(out)
        obs = {k: res[k] for k in ('model', 'graph_features', 'action_mask')}
        return obs, res['reward'], res['done'], {}

    def _export(self, out):
        B, A = self.B, self.n_actions
        spec = {'model': ((B,), torch.int64), 'graph_features': ((B, N_GRAPH_FEATURES + A), torch.float32),
                'action_mask': ((B, A), torch.bool), 'reward': ((B,), torch.float64), 'done': ((B,), torch.bool)}
        out = dict(out or {})
        unknown = set(out) - set(OUTPUTS)
        if unknown:
            raise ValueError(f'unknown outputs {sorted(unknown)}; expected a subset of {list(OUTPUTS)}')
        res = {}
        for k, (shape, dtype) in spec.items():
            t = out.get(k)
            if t is None:
                t = torch.empty(shape, dtype=dtype, device=self.device)
            elif t.dtype != dtype or tuple(t.shape) != shape or t.device != self.device or not t.is_contiguous():
                raise ValueError(f"out['{k}'] must be a contiguous {dtype} tensor of shape {shape} on {self.device}, "
                                 f'not {t.dtype} {tuple(t.shape)} on {t.device}')
            res[k] = t
        ex = _Export(*[res[k].data_ptr() for k in OUTPUTS])
        _engine._check(self._L.ramp_env_export(self._h, torch.cuda.current_stream(self.device).cuda_stream, C.byref(ex)))
        return res
