"""Eager against CUDA-graph rollouts through TorchRampJobPartitioningEnvironment: segments of 8 decisions per episode, an eager
reset before each, at three sizes (every block geometry prewarmed):

  cfg1  one episode, the 2x2x2 RAMP cluster, chain jobs
  cfg2  256 episodes, the 4x4x2 cluster, ResNet-50-like jobs
  cfg3  4,096 episodes, the 4x4x4 cluster, ResNet-50-like jobs

and two policies: the masked-uniform torch policy of scripts/torch_env_rollouts.py (torch.multinomial over the mask) and
TorchGNNPolicy under no_grad with a Categorical draw.  The graphed arm captures the segment's 8 decisions once (policy + step,
observations into static tensors) and per segment copies the reset's observation in and replays.  Eager and graphed segments
alternate, three repeats each.  Env-steps are the decisions of episodes that were not done (decisions() after each segment,
outside the timed region); `seconds` covers the reset and the steps, `step_seconds` the steps alone (from the reset's return to
the synchronisation after the last step).

In the same run, for each size, a twin pair of environments (apply_action_mask=False) takes one segment of fixed actions, one
eagerly and one replaying a graph: every output of every step, the episode statistics and the decision counts must be the same
bytes.  Writes one JSON line per run to --out, with the GPU's name, power limit and maximum SM clock.

  python scripts/graph_rollouts.py --out profiles/h100_graph_rollouts.jsonl
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

SIZES = {'cfg1': ((2, 2, 2), 'chain', 1), 'cfg2': ((4, 4, 2), 'resnet', 256), 'cfg3': ((4, 4, 4), 'resnet', 4096)}
OBS_KEYS = ('model', 'graph_features', 'action_mask')
OUT_KEYS = OBS_KEYS + ('reward', 'done')


def make_env(size, L, **kw):
    from ddls_b200 import synth
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    shape, kind, B = SIZES[size]
    g = synth.chain_graph() if kind == 'chain' else synth.resnet_like_graph()
    env = TorchRampJobPartitioningEnvironment(shape, [g], n_episodes=B, jobs_per_episode=L, prewarm=True, **kw)
    assert env.env._device_decides_everything
    return env


def static_outs(env):
    import torch
    B, A = env.B, env.n_actions
    spec = {'model': ((B,), torch.int64), 'graph_features': ((B, 17 + A), torch.float32), 'action_mask': ((B, A), torch.bool),
            'reward': ((B,), torch.float64), 'done': ((B,), torch.bool)}
    return {k: torch.empty(s, dtype=d, device=env.device) for k, (s, d) in spec.items()}


def same_bytes(a, b):
    """a and b (arrays, or dicts / lists of them) hold the same bytes"""
    import numpy as np
    if isinstance(a, dict):
        return isinstance(b, dict) and sorted(a) == sorted(b) and all(same_bytes(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same_bytes(x, y) for x, y in zip(a, b))
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def bytes_check(size, L):
    """twin environments, one segment of fixed actions: eager steps against one graph replay, compared byte for byte"""
    import torch
    env, twin = make_env(size, L, seed=11, apply_action_mask=False), make_env(size, L, seed=11, apply_action_mask=False)
    gen = torch.Generator(device=env.device).manual_seed(5)
    acts = [torch.randint(0, env.n_actions, (env.B,), generator=gen, device=env.device) for _ in range(L + 1)]
    env.reset(); twin.reset()
    env.step(acts[0]); twin.step(acts[0])                     # the eager step a capture needs
    static = [torch.zeros_like(a) for a in acts[1:]]
    outs = [static_outs(env) for _ in range(L)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for a, o in zip(static, outs):
            env.step(a, out=o)
    for s, a in zip(static, acts[1:]):
        s.copy_(a)
    g.replay()
    same = True
    for t in range(L):
        obs, reward, done, _ = twin.step(acts[1 + t])
        want = dict(obs, reward=reward, done=done)
        same &= same_bytes({k: outs[t][k].cpu().numpy() for k in OUT_KEYS}, {k: want[k].cpu().numpy() for k in OUT_KEYS})
    env.check(); twin.check()
    same &= same_bytes(env.decisions(), twin.decisions()) and same_bytes(env.episode_stats(), twin.episode_stats())
    del g
    env.close(); twin.close()
    return bool(same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='cfg1,cfg2,cfg3')
    ap.add_argument('--segment', type=int, default=8)
    ap.add_argument('--segments', type=int, default=16, help='timed segments per run')
    ap.add_argument('--warmup', type=int, default=2, help='untimed segments per run')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch_env_rollouts import gpu_info
    from ddls_b200.torch_policy import TorchGNNPolicy
    if not torch.cuda.is_available():
        raise SystemExit('this measurement needs a GPU')
    L = args.segment
    meta = dict(gpu_info(), segment=L, segments=args.segments, torch=torch.__version__)
    lines = []

    def emit(x):
        lines.append(x)
        print(json.dumps(x), flush=True)

    for size in args.sizes.split(','):
        emit(dict(meta, size=size, run='bytes_check', eager_equals_graph=bytes_check(size, L)))
        torch.manual_seed(0)
        env = make_env(size, L, seed=0)
        mod = TorchGNNPolicy(env.static, env.n_actions, seed=0)
        policies = {
            'masked_uniform': lambda obs: torch.multinomial(obs['action_mask'].to(torch.float32), 1).reshape(-1),
            'gnn_categorical': lambda obs: torch.distributions.Categorical(logits=mod(obs)[0], validate_args=False).sample(),
        }
        for pname, act in policies.items():
            obs = env.reset()
            with torch.no_grad():
                obs = env.step(act(obs))[0]                       # eager: sizes the buffers, uploads and embeds the weights
            env.check()
            obs0 = {k: torch.empty_like(v) for k, v in obs.items()}
            outs = [static_outs(env) for _ in range(L)]
            g = torch.cuda.CUDAGraph()
            with torch.no_grad(), torch.cuda.graph(g):
                o = obs0
                for t in range(L):
                    env.step(act(o), out=outs[t])
                    o = {k: outs[t][k] for k in OBS_KEYS}

            def seg_eager():
                obs = env.reset()
                t1 = time.perf_counter()
                with torch.no_grad():
                    for _ in range(L):
                        obs = env.step(act(obs))[0]
                env.check()
                return t1

            def seg_graph():
                obs = env.reset()
                t1 = time.perf_counter()
                for k in OBS_KEYS:
                    obs0[k].copy_(obs[k])
                g.replay()
                env.check()
                return t1

            for rep in range(args.repeats):
                for arm, seg in (('eager', seg_eager), ('graph', seg_graph)):
                    for _ in range(args.warmup):
                        seg()
                    torch.cuda.synchronize()
                    n_steps, wall, step_wall = 0, 0.0, 0.0
                    for _ in range(args.segments):
                        t0 = time.perf_counter()
                        t1 = seg()
                        torch.cuda.synchronize()
                        t2 = time.perf_counter()
                        wall += t2 - t0
                        step_wall += t2 - t1
                        n_steps += int(env.decisions().sum())
                    emit(dict(meta, size=size, episodes=env.B, policy=pname, arm=arm, repeat=rep, env_steps=n_steps, seconds=wall,
                              step_seconds=step_wall, env_steps_per_s=n_steps / wall, step_env_steps_per_s=n_steps / step_wall,
                              us_per_step=step_wall / (args.segments * L) * 1e6))
            for arm in ('eager', 'graph'):
                v = [x['env_steps_per_s'] for x in lines if x.get('size') == size and x.get('policy') == pname and x.get('arm') == arm]
                w = [x['us_per_step'] for x in lines if x.get('size') == size and x.get('policy') == pname and x.get('arm') == arm]
                emit(dict(meta, size=size, policy=pname, arm=arm, summary='median over repeats', env_steps_per_s_median=float(np.median(v)),
                          us_per_step_median=float(np.median(w)), values=v))
            del g
        mod.close()
        env.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for x in lines:
                f.write(json.dumps(x) + '\n')


if __name__ == '__main__':
    main()
