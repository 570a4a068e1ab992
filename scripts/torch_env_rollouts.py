"""Env-steps per second of config 3 (4,096 episodes, the 64-worker RAMP cluster, ResNet-50 jobs, every block geometry prewarmed)
through three ways of driving the device environment, each over whole segments of 8 decisions per episode with a reset before each:

  torch_env      a masked-uniform torch policy (torch.multinomial on the device) through TorchRampJobPartitioningEnvironment.step:
                 CUDA tensors in and out, no synchronisation inside a segment
  host_step      the same policy through DeviceRampJobPartitioningEnvironment.step(actions.cpu().numpy()), the mask copied back
                 to the device for the next draw: two PCIe round trips and a host synchronisation per step
  device_policy  DeviceGNNPolicy.act + step_device() (the policy kernels write the action buffer), for reference

Env-steps are the decisions of episodes that were not done (decisions() at the end of each segment).  Also timed: one
ramp_env_ingest + ramp_env_export pair alone (both kernels and their four fences), over many calls.  Writes one JSON line per run to
--out, with the GPU's name and power limit.

  python scripts/torch_env_rollouts.py --repeats 3 --out profiles/h100_torch_env_rollouts.jsonl
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    import torch
    info = {'gpu': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        info['power_limit'], info['max_sm_clock'] = [x.strip() for x in q[0].split(',')]
    except Exception as ex:          # the record still names the GPU
        info['power_limit'] = f'unknown ({ex!r})'
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--episodes', type=int, default=4096)
    ap.add_argument('--segment', type=int, default=8, help='decisions per episode between resets (bench.py --segment)')
    ap.add_argument('--segments', type=int, default=16, help='timed segments per run')
    ap.add_argument('--warmup', type=int, default=2, help='untimed segments per run')
    ap.add_argument('--repeats', type=int, default=3, help='the three runs, alternated, this many times')
    ap.add_argument('--io-calls', type=int, default=2000)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from ddls_b200 import engine, synth
    from ddls_b200 import policy as P
    from ddls_b200.torch_env import ACTIONS_INT64, TorchRampJobPartitioningEnvironment, _Export
    if not torch.cuda.is_available():
        raise SystemExit('this measurement needs a GPU')
    dev = torch.device('cuda', 0)
    B, L = args.episodes, args.segment
    graphs = [synth.resnet_like_graph()]
    env = TorchRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=L, seed=0, prewarm=True)
    assert env.env._device_decides_everything
    base = env.env                                   # the wrapped DeviceRampJobPartitioningEnvironment: runs 2 and 3 drive it directly
    pol = P.DeviceGNNPolicy(graphs, env.n_actions, seed=0)
    pol.embed()
    gen = torch.Generator(device=dev).manual_seed(0)

    def draw(mask):
        return torch.multinomial(mask.to(torch.float32), 1, generator=gen).reshape(-1)

    def seg_torch_env(s):
        obs = env.reset()
        for _ in range(L):
            obs = env.step(draw(obs['action_mask']))[0]
        env.check()

    def seg_host_step(s):
        obs = base.reset()
        for _ in range(L):
            mask = torch.from_numpy(obs['action_mask']).to(dev)
            obs = base.step(draw(mask).cpu().numpy())[0]

    def seg_device_policy(s):
        base.reset()
        for t in range(L):
            pol.act(base, sample=True, seed=1000 * s + t)
            base.step_device()
        base.read()

    runs = {'torch_env': seg_torch_env, 'host_step': seg_host_step, 'device_policy': seg_device_policy}
    meta = dict(gpu_info(), workload='cfg3-resnet50-64w', episodes=B, segment=L, segments=args.segments, torch=torch.__version__)
    lines = []
    for rep in range(args.repeats):
        for name, seg in runs.items():
            for s in range(args.warmup):
                seg(s)
            torch.cuda.synchronize()
            n_steps, wall = 0, 0.0
            for s in range(args.segments):
                t0 = time.perf_counter()
                seg(args.warmup + s)
                torch.cuda.synchronize()
                wall += time.perf_counter() - t0
                n_steps += int(base.decisions().sum())        # outside the timed region
            lines.append(dict(meta, run=name, repeat=rep, env_steps=n_steps, seconds=wall, env_steps_per_s=n_steps / wall,
                              ms_per_step=wall / (args.segments * L) * 1e3))
            print(json.dumps(lines[-1]), flush=True)

    # one ingest + export pair alone: the two kernels and the four event fences of a torch step, without the step between them
    L_ = env._L
    a = torch.zeros(B, dtype=torch.int64, device=dev)
    outs = {'model': torch.empty(B, dtype=torch.int64, device=dev), 'graph_features': torch.empty((B, 17 + env.n_actions), device=dev),
            'action_mask': torch.empty((B, env.n_actions), dtype=torch.bool, device=dev),
            'reward': torch.empty(B, dtype=torch.float64, device=dev), 'done': torch.empty(B, dtype=torch.bool, device=dev)}
    ex = _Export(*[outs[k].data_ptr() for k in ('model', 'graph_features', 'action_mask', 'reward', 'done')])
    env.reset()
    stream = torch.cuda.current_stream(dev).cuda_stream
    for n in (100, args.io_calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            engine._check(L_.ramp_env_ingest(env._h, a.data_ptr(), ACTIONS_INT64, stream))
            engine._check(L_.ramp_env_export(env._h, stream, C.byref(ex)))
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    env.check()
    lines.append(dict(meta, run='ingest_export_pair', calls=args.io_calls, us_per_pair=dt / args.io_calls * 1e6))
    print(json.dumps(lines[-1]), flush=True)
    for name in runs:
        v = [x['env_steps_per_s'] for x in lines if x.get('run') == name]
        summary = dict(meta, run=name, summary='median over repeats', env_steps_per_s_median=float(np.median(v)), values=v)
        lines.append(summary)
        print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for x in lines:
                f.write(json.dumps(x) + '\n')
    pol.close()
    env.close()


if __name__ == '__main__':
    main()
