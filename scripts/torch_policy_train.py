"""PPO written in plain torch on the device environment and the device GNN policy: TorchRampJobPartitioningEnvironment +
TorchGNNPolicy + torch.optim.Adam, at ppo.yaml's settings (ddls_b200.learn.PPOConfig) -- the worked example of a learner the library
has no fused kernel for.  Each iteration collects one segment (a torch.no_grad() forward, torch.distributions.Categorical, env.step),
computes GAE, and takes num_sgd_iter shuffled passes of minibatch steps on the clipped loss of tests/ppo_reference.py in fp32 with
clip_grad_norm_.  Everything stays on the device; the iteration reads one number back, the live-row count that sizes the minibatch
loop, and synchronises at the end of its collect and of its learn for the timing.  The distributions are built with
validate_args=False: torch's argument checks read a flag back from the device on every construction and log_prob.  CUDA events
between the phases of each minibatch step (forward, loss, backward, clip + Adam) give the step's breakdown in stream time.

The same iteration is then run through DevicePPOLearner (DeviceGNNPolicy.collect + learn) on a twin environment, alternated in the
same process, and both are written per iteration as JSON lines to --out with the card's name and power limit:

    python scripts/torch_policy_train.py --iters 5 --out profiles/h100_torch_policy_train.jsonl

--rollouts measures the rollout rate instead, at scripts/torch_env_rollouts.py's settings (config 3: 4,096 episodes, segments of 8
decisions from a reset), three runs alternated: the torch module (torch.no_grad() forward + Categorical sample + env.step), a
masked-uniform torch policy through env.step, and DeviceGNNPolicy.act + step_device():

    python scripts/torch_policy_train.py --rollouts --out profiles/h100_torch_policy_rollouts.jsonl"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    import torch
    info = {'gpu': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=20).stdout.strip().splitlines()
        info['power_limit'] = q[0].strip()
    except Exception as ex:          # the record still names the GPU
        info['power_limit'] = f'unknown ({ex!r})'
    return info


def collect(env, mod, T):
    """one segment of T steps from a fresh reset: per step the observation, the collection logits, action, log p, value, and
    the reward and done that came back; the value of the state after the last step"""
    import torch
    from torch.distributions import Categorical
    obs = env.reset()
    seg = {k: [] for k in ('model', 'graph_features', 'action_mask', 'logits', 'action', 'value', 'reward', 'done')}
    with torch.no_grad():
        for _ in range(T):
            logits, value = mod(obs)
            action = Categorical(logits=logits, validate_args=False).sample()
            for k in ('model', 'graph_features', 'action_mask'):
                seg[k].append(obs[k])
            seg['logits'].append(logits); seg['action'].append(action); seg['value'].append(value)
            obs, reward, done, _ = env.step(action)
            seg['reward'].append(reward); seg['done'].append(done)
        _, boot = mod(obs)
    return {k: torch.stack(v) for k, v in seg.items()}, boot


def gae(seg, boot, gamma, lam):
    """RLlib's compute_advantages (use_gae) per episode, [T, B], in float64; live: decisions of episodes not finished yet with a
    job queued"""
    import torch
    T, B = seg['reward'].shape
    done = seg['done']
    alive = torch.cat([torch.ones((1, B), dtype=torch.bool, device=done.device), ~done[:-1]], 0)
    value = seg['value'].double()
    adv = torch.zeros((T, B), dtype=torch.float64, device=done.device)
    nxt = torch.zeros(B, dtype=torch.float64, device=done.device)
    for t in range(T - 1, -1, -1):
        nonterm = (~done[t]).double()
        vn = boot.double() if t == T - 1 else value[t + 1]
        a = seg['reward'][t] + gamma * vn * nonterm - value[t] + gamma * lam * nonterm * nxt
        adv[t] = torch.where(alive[t], a, 0.0)
        nxt = torch.where(alive[t], a, nxt)
    live = alive & (seg['model'] >= 0)
    return adv, adv + value, live


def ppo_loss(logits, value, action, old_logits, adv, vt, cfg, kl_coeff):
    """PPOTorchPolicy.loss as tests/ppo_reference.py states it, in fp32"""
    import torch
    from torch.distributions import Categorical, kl_divergence
    cur, prev = Categorical(logits=logits, validate_args=False), Categorical(logits=old_logits, validate_args=False)
    ratio = torch.exp(cur.log_prob(action) - prev.log_prob(action))
    surr = torch.min(adv * ratio, adv * torch.clamp(ratio, 1 - cfg.clip_param, 1 + cfg.clip_param))
    vf = torch.clamp((value - vt) ** 2, 0, cfg.vf_clip_param)
    kl = kl_divergence(prev, cur)
    total = torch.mean(-surr + cfg.vf_loss_coeff * vf - cfg.entropy_coeff * cur.entropy()) + kl_coeff * torch.mean(kl)
    return total, torch.mean(kl)


def torch_iteration(env, mod, opt, cfg, T, kl_coeff, gen):
    """one collect + learn; returns (collect seconds, learn seconds, minibatch steps, the new kl coefficient, ms per step of each
    phase in stream time)"""
    import torch
    dev = mod.device
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    seg, boot = collect(env, mod, T)
    torch.cuda.synchronize(dev)
    t1 = time.perf_counter()
    adv, vt, live = gae(seg, boot, cfg.gamma, cfg.lambda_)
    flat = {k: v.reshape((-1,) + tuple(v.shape[2:])) for k, v in seg.items()}
    live, adv, vt = live.reshape(-1), adv.reshape(-1), vt.reshape(-1)
    n = int(live.sum())                                            # the iteration's one read-back: the train batch's size
    rows = torch.argsort((~live).to(torch.int32), stable=True)[:n]   # the live rows, t-major
    batch = {k: v[rows] for k, v in flat.items()}
    adv, vt = adv[rows], vt[rows]
    if cfg.standardize_advantages:
        adv = (adv - adv.mean()) / torch.clamp(adv.std(unbiased=False), min=1e-4)
    adv, vt = adv.float(), vt.float()
    mb, steps, kl_last, marks = cfg.sgd_minibatch_size, 0, [], []
    for _ in range(cfg.num_sgd_iter):
        order = torch.randperm(n, device=dev, generator=gen)
        kl_last = []
        for s in range(0, n, mb):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            idx = order[s:s + mb]
            ev[0].record()
            logits, value = mod({k: batch[k][idx] for k in ('model', 'graph_features', 'action_mask')})
            ev[1].record()
            loss, kl = ppo_loss(logits, value, batch['action'][idx], batch['logits'][idx], adv[idx], vt[idx], cfg, kl_coeff)
            ev[2].record()
            opt.zero_grad(set_to_none=True)
            loss.backward()
            ev[3].record()
            torch.nn.utils.clip_grad_norm_(mod.parameters(), cfg.grad_clip)
            opt.step()
            ev[4].record()
            marks.append(ev)
            kl_last.append(kl.detach())
            steps += 1
    if kl_last:                                                    # RLlib's update_kl on the last pass's mean KL, on the device
        kl = torch.stack(kl_last).mean()
        kl_coeff = torch.where(kl > 2 * cfg.kl_target, kl_coeff * 1.5, torch.where(kl < 0.5 * cfg.kl_target, kl_coeff * 0.5, kl_coeff))
    torch.cuda.synchronize(dev)
    t2 = time.perf_counter()
    phases = ('forward', 'loss', 'backward', 'clip_adam')
    breakdown = {ph: sum(ev[i].elapsed_time(ev[i + 1]) for ev in marks) / max(1, steps) for i, ph in enumerate(phases)}
    return t1 - t0, t2 - t1, steps, kl_coeff, breakdown


def rollouts(args):
    """rollout rates at scripts/torch_env_rollouts.py's settings, three runs alternated --repeats times"""
    import numpy as np
    import torch
    from torch.distributions import Categorical
    from ddls_b200 import synth
    from ddls_b200.policy import DeviceGNNPolicy
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    from ddls_b200.torch_policy import TorchGNNPolicy
    B, L, dev = 4096, 8, torch.device('cuda', 0)
    graphs = [synth.resnet_like_graph()]
    env = TorchRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=L, seed=0, prewarm=True)
    base = env.env
    mod = TorchGNNPolicy(env.static, env.n_actions, seed=0)
    pol = DeviceGNNPolicy(graphs, env.n_actions, state_dict=mod.gnn_state_dict())
    gen = torch.Generator(device=dev).manual_seed(0)

    def seg_torch_policy(s):
        obs = env.reset()
        with torch.no_grad():
            for _ in range(L):
                logits, _ = mod(obs)
                obs = env.step(Categorical(logits=logits, validate_args=False).sample())[0]
        env.check()

    def seg_torch_env(s):
        obs = env.reset()
        for _ in range(L):
            obs = env.step(torch.multinomial(obs['action_mask'].to(torch.float32), 1, generator=gen).reshape(-1))[0]
        env.check()

    def seg_device_policy(s):
        base.reset()
        for t in range(L):
            pol.act(base, sample=True, seed=1000 * s + t)
            base.step_device()
        base.read()

    runs = {'torch_policy': seg_torch_policy, 'torch_env': seg_torch_env, 'device_policy': seg_device_policy}
    meta = dict(gpu_info(), workload='cfg3-resnet50-64w', episodes=B, segment=L, segments=16, torch=torch.__version__)
    lines = []
    for rep in range(args.repeats):
        for name, seg in runs.items():
            for s in range(2):
                seg(s)
            torch.cuda.synchronize()
            n_steps, wall = 0, 0.0
            for s in range(16):
                t0 = time.perf_counter()
                seg(2 + s)
                torch.cuda.synchronize()
                wall += time.perf_counter() - t0
                n_steps += int(base.decisions().sum())        # outside the timed region
            lines.append(dict(meta, run=name, repeat=rep, env_steps=n_steps, seconds=wall, env_steps_per_s=n_steps / wall))
            print(json.dumps(lines[-1]), flush=True)
    for name in runs:
        v = [x['env_steps_per_s'] for x in lines if x.get('run') == name]
        lines.append(dict(meta, run=name, summary='median over repeats', env_steps_per_s_median=float(np.median(v)), values=v))
        print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            for x in lines:
                f.write(json.dumps(x) + '\n')
    mod.close(); pol.close(); env.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--episodes', type=int, default=1024)
    ap.add_argument('--jobs', type=int, default=16, help='jobs per episode = the segment horizon (whole episodes)')
    ap.add_argument('--num-sgd-iter', type=int, default=None, help="override ppo.yaml's 50 passes")
    ap.add_argument('--model', choices=('gnn', 'algo'), default='gnn',
                    help="gnn: gnn.yaml's read-out ([256], separate value branch); algo: algo/ppo.yaml's (policy.algo_model_config)")
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    ap.add_argument('--rollouts', action='store_true', help='measure the rollout rates instead of training')
    ap.add_argument('--repeats', type=int, default=3, help='--rollouts: the three runs, alternated, this many times')
    args = ap.parse_args()
    if args.rollouts:
        return rollouts(args)
    import torch
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    from ddls_b200.policy import DeviceGNNPolicy, algo_model_config
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    from ddls_b200.torch_policy import TorchGNNPolicy

    graphs = [workload.make_graph('resnet')]
    kw = dict(n_episodes=args.episodes, jobs_per_episode=args.jobs, seed=args.seed, prewarm=True)
    env = TorchRampJobPartitioningEnvironment((4, 4, 4), graphs, **kw)
    twin = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, **kw)
    A = env.n_actions
    model = algo_model_config('ppo', A) if args.model == 'algo' else None
    cfg = PPOConfig(seed=args.seed)
    if args.num_sgd_iter is not None:
        cfg.num_sgd_iter = args.num_sgd_iter
    mod = TorchGNNPolicy(env.static, A, config=model, seed=args.seed)
    pol = DeviceGNNPolicy(graphs, A, config=model, state_dict=mod.gnn_state_dict())
    lrn = DevicePPOLearner(pol, dataclasses.replace(cfg))
    opt = torch.optim.Adam(mod.parameters(), lr=cfg.lr, betas=(cfg.adam_beta1, cfg.adam_beta2), eps=cfg.adam_eps)
    gen = torch.Generator(device=mod.device).manual_seed(args.seed)
    torch.manual_seed(args.seed)
    kl_coeff = torch.tensor(cfg.kl_coeff, device=mod.device)
    meta = dict(gpu_info(), episodes=args.episodes, jobs=args.jobs, model=args.model, num_sgd_iter=cfg.num_sgd_iter,
                sgd_minibatch_size=cfg.sgd_minibatch_size, weights=int(mod.weight.numel()))
    out = open(args.out, 'w') if args.out else None
    for it in range(args.iters):
        c_s, l_s, steps, kl_coeff, breakdown = torch_iteration(env, mod, opt, cfg, args.jobs, kl_coeff, gen)
        env.check()
        t0 = time.perf_counter()
        pol.collect(twin, args.jobs, sample=True, seed=args.seed + 1000 * it)
        t1 = time.perf_counter()
        stats = lrn.learn(twin, args.jobs)
        t2 = time.perf_counter()
        f_steps = cfg.num_sgd_iter * -(-int(stats['rows']) // cfg.sgd_minibatch_size)
        env_steps = args.episodes * args.jobs
        row = dict(meta, iter=it,
                   torch=dict(collect_s=c_s, collect_env_steps_per_s=env_steps / c_s, learn_s=l_s, minibatch_steps=steps,
                              ms_per_minibatch_step=1e3 * l_s / max(1, steps), stream_ms_per_step=breakdown),
                   fused=dict(collect_s=t1 - t0, collect_env_steps_per_s=env_steps / (t1 - t0), learn_s=t2 - t1,
                              minibatch_steps=f_steps, ms_per_minibatch_step=1e3 * (t2 - t1) / max(1, f_steps)))
        print(json.dumps(row), flush=True)
        if out:
            out.write(json.dumps(row) + '\n')
            out.flush()
    mod.close(); pol.close(); env.close(); twin.close()


if __name__ == '__main__':
    main()
