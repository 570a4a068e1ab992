"""-m gpu: the GNN policy's forward and MeanPool backward (ramp_gnn_embed_kernel, embed_grad_body in ramp_policy_learn.cuh) on the
graph shapes where a per-node loop turns on degree: hubs of thousands of out-edges (the backward gathers d node-module output
over a node's out-edge row, serially), a node with large in- and out-degree at once, 1,000 parallel copies of one edge,
self-loops, no edges at all, a 2-cycle, a chain deeper than any round count, K64,64, and in- and out-degrees around a warp's 32.

- raw graphs (topologies() below), each its own job type of one RawPolicy next to the one-node graph, at every configuration
  of tests/test_gpu_policy_kernels.py: embeddings, logits and values against float64 (gnn_reference: embed64 / head64) within
  its TOL; pol.backward on rows of each topology against float64 autograd (ppo_reference.policy64), every weight tensor within
  max(1e-4, 10 e32) once tie_reference has accounted for named near-ties (test_gpu_learn_grad_recorded.check_explained);
- fan job types through the device environment (fan_graphs(): one op feeding 512 that join again, a 32-wide diamond around a
  K32,32 core), next to ResNet-50: the PPO / IMPALA / PG gradients on recorded batches against float64, PPO's first pass
  recomputing the collected log-probabilities bit for bit, a mixed-shape population (the smallest shape next to the largest,
  shared and separate value branches; a 256-wide fan) against its twins bit for bit, and TorchGNNPolicy's gradients against float64.

pytest -s prints, per configuration and topology, the worst forward error and the backward's worst tensor error next to torch
fp32's, the named ties used, and the largest in- and out-degree among the graphs."""
import numpy as np
import pytest
import torch

from test_gpu_learn_grad_recorded import check_explained
from test_gpu_policy_kernels import CONFIGS, SEED, Graph, _cfg, batch, check_close, check_readout, raw_policy
from test_gpu_policy_learn import rows

pytestmark = pytest.mark.gpu

MAX_CANDIDATES = 32            # near-ties offered to explain() per backward case, closest first: each costs a float64 autograd run


def topologies():
    """the raw graphs (Graph without features), the one-node graph first"""
    hub_in, hub_out = np.arange(1, 2049), np.arange(2049, 4097)
    leaves = np.arange(6, 39)                           # degree hubs: out-hubs 0, 1, 2 and in-hubs 3, 4, 5 over 31, 32, 33 leaves
    deg_src = np.concatenate([np.full(d, h) for h, d in zip((0, 1, 2), (31, 32, 33))] + [leaves[:d] for d in (31, 32, 33)])
    deg_dst = np.concatenate([leaves[:d] for d in (31, 32, 33)] + [np.full(d, h) for h, d in zip((3, 4, 5), (31, 32, 33))])
    k = np.arange(64)
    return [
        Graph('single', 1, [], []),
        Graph('out_star', 4097, np.zeros(4096), np.arange(1, 4097)),
        Graph('bi_hub', 4097, np.concatenate([hub_in, np.zeros(2048)]), np.concatenate([np.zeros(2048), hub_out])),
        Graph('parallel', 8, np.concatenate([np.zeros(1000), [1, 2, 3, 4, 5, 6, 3]]),
              np.concatenate([np.ones(1000), [2, 3, 4, 5, 6, 7, 1]])),
        Graph('self_loops', 16, np.arange(16), np.arange(16)),
        Graph('hub_loop', 301, np.concatenate([[0], np.arange(1, 151), np.zeros(150)]),
              np.concatenate([[0], np.zeros(150), np.arange(151, 301)])),
        Graph('edgeless', 64, [], []),
        Graph('two_cycle', 2, [0, 1], [1, 0]),
        Graph('chain2000', 2000, np.arange(1999), np.arange(1, 2000)),
        Graph('k64_64', 128, np.repeat(k, 64), np.tile(k + 64, 64)),
        Graph('deg31_32_33', 39, deg_src, deg_dst),
    ]


def degrees(g):
    return np.bincount(g.src, minlength=g.n), np.bincount(g.dst, minlength=g.n)


class Case:
    pass


@pytest.fixture(scope='module', params=list(CONFIGS))
def case(request):
    """one policy per configuration, every topology registered as its own job type, and the float64 embeddings of each"""
    from ddls_b200 import policy as P
    from gnn_reference import embed64
    over, A, _, _ = CONFIGS[request.param]
    k = Case()
    k.id, k.c, k.A = request.param, _cfg(over), A
    rng = np.random.default_rng(23)
    k.graphs = [g.features(k.c, rng) for g in topologies()]
    k.sd = P.random_state_dict(k.c, A, seed=SEED)
    k.emb64 = np.stack([embed64(k.sd, k.c, g.nf, g.ef, g.src, g.dst) for g in k.graphs])
    k.pol = raw_policy(k.c, A, k.graphs, k.sd)
    yield k
    k.pol.close()


def test_the_graphs_reach_hub_degrees():
    out_deg = max(int(degrees(g)[0].max(initial=0)) for g in topologies())
    in_deg = max(int(degrees(g)[1].max(initial=0)) for g in topologies())
    print(f'[topology] largest out-degree {out_deg}, largest in-degree {in_deg}')
    assert out_deg >= 4096 and in_deg >= 2048


def test_forward_matches_float64(case):
    """embeddings per job type, then logits and values of rows of every job type (decide)"""
    emb = case.pol.embed()
    model, gf, mask = batch(case, 2113, seed=31)
    logits, value, _, _ = case.pol.decide(model, gf, mask)
    for m, g in enumerate(case.graphs):
        ee = check_close(emb[m], case.emb64[m], f'{case.id} {g.name} embedding')
        mine = model == m
        assert mine.sum() > 50
        el, ev = check_readout(case, model[mine], gf[mine], mask[mine], (logits[mine], value[mine]), f'{case.id} {g.name}')
        print(f'[topology] {case.id:9s} {g.name:12s} forward max |err|: embedding {ee:.2e} (max |ref| '
              f'{np.abs(case.emb64[m]).max():.2e}), logits {el:.2e}, value {ev:.2e}')
    edgeless = [m for m, g in enumerate(case.graphs) if g.name == 'edgeless']
    assert not emb[edgeless].any()                                  # every node has zero in-degree: every round ends at zeros


def linear_loss(gl, gv):
    return lambda logits, value: (torch.as_tensor(gl, dtype=logits.dtype) * logits).sum() + \
        (torch.as_tensor(gv, dtype=value.dtype) * value).sum()


def test_backward_matches_float64_autograd(case):
    """per topology, 48 rows: its own job type, every eighth row the one-node graph's, two rows with model -1; random upstream
    gradients and masks.  The other job types have no rows, so their CTAs take the zero-gradient exit"""
    for m, g in enumerate(case.graphs[1:], start=1):
        model, gf, mask = rows(len(case.graphs), case.A, case.c, 48, seed=100 + m)
        model = np.where(model >= 0, np.where(np.arange(48) % 8 == 0, 0, m), -1)
        rng = np.random.default_rng(200 + m)
        gl = rng.standard_normal((48, case.A)).astype(np.float32)
        gv = rng.standard_normal(48).astype(np.float32)
        got = case.pol.backward(model, gf, mask, gl, gv)
        live = model >= 0
        check_explained(case.pol, f'[topology] {case.id:9s} {g.name:12s} backward', got, model[live], gf[live], mask[live],
                        linear_loss(gl[live], gv[live]), graphs=case.graphs, max_candidates=MAX_CANDIDATES)
        np.testing.assert_array_equal(case.pol.backward(model, gf, mask, gl, gv), got)


# ---- fan job types through the device environment ----

def fan_graphs(width=512):
    """synth.ForwardGraph job types whose mirrored graphs have hubs: one op feeding `width` ops that join again (out- and
    in-degree `width`), and a diamond whose 32-wide middle is a complete K32,32 (nodes of in- and out-degree 32)"""
    from ddls_b200 import synth
    rng = np.random.default_rng(41)

    def op(g, kind):
        return g.add(kind, round(float(rng.uniform(0.2, 4.0)), 6), round(float(rng.uniform(0.4, 8.0)), 6),
                     float(rng.integers(1, 40) * 100352), float(rng.integers(1, 100) * 4096))
    fan = synth.ForwardGraph(name=f'fan{width}')
    src = op(fan, 'Conv2d')
    mid = [op(fan, ['Conv2d', 'BatchNorm2d', 'ReLU'][i % 3]) for i in range(width)]
    join = op(fan, 'Add')
    fan.edges = sorted([(src, v) for v in mid] + [(v, join) for v in mid])
    dia = synth.ForwardGraph(name='diamond32')
    src = op(dia, 'Conv2d')
    left = [op(dia, 'Conv2d') for _ in range(32)]
    right = [op(dia, 'ReLU') for _ in range(32)]
    join = op(dia, 'Add')
    dia.edges = sorted([(src, u) for u in left] + [(u, v) for u in left for v in right] + [(v, join) for v in right])
    return [fan, dia]


def _fan_env(B=64, J=6, seed=7):
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    graphs = [workload.make_graph('resnet')] + fan_graphs()
    return DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=J, seed=seed), graphs


def test_fan_job_types_mirror_into_hubs():
    from ddls_b200 import policy as P
    env, graphs = _fan_env(B=4)
    pol = P.DeviceGNNPolicy(graphs, env.max_partitions_per_op + 1)
    try:
        for st, want in zip(pol.static[1:], (512, 32)):
            src, dst = np.asarray(st['edges_src']), np.asarray(st['edges_dst'])
            n = len(st['node_features'])
            print(f'[topology] mirrored {n} nodes, {len(src)} edges: out-degree {np.bincount(src, minlength=n).max()}, '
                  f'in-degree {np.bincount(dst, minlength=n).max()}')
            assert np.bincount(src, minlength=n).max() >= want and np.bincount(dst, minlength=n).max() >= want
    finally:
        pol.close(); env.close()


@pytest.mark.parametrize('wseed', [2, 4])
def test_learner_gradients_on_fan_job_types(wseed):
    from test_gpu_learn_grad_recorded import learner_gradients_on_a_recorded_batch
    env, graphs = _fan_env()
    learner_gradients_on_a_recorded_batch(env, graphs, 6, wseed, f'fan seed {wseed}', min_rows=100)


def test_first_pass_recomputes_the_collected_log_probabilities_on_fan_job_types():
    from ddls_b200 import policy as P
    from test_gpu_policy_learn import first_pass_recomputes_the_collected_log_probabilities
    J = 6
    env, graphs = _fan_env(J=J, seed=9)
    A = env.max_partitions_per_op + 1
    pol = P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=4))
    first_pass_recomputes_the_collected_log_probabilities(env, pol, J)


def test_population_on_fan_job_types_matches_its_twins():
    """K = 4: the smallest shape next to the largest, twice, the smallest with a separate value branch and then a shared one, the
    largest shared; PPO, IMPALA and PG in turn.  Each (set, job type) item's scratch spans a 516-node fan next to the 132-node
    diamond.  Twins of the first two sets (separate and shared): each twin environment keeps its own lookahead scratch for the
    fan's templates, and three environments with the 512-wide fan's do not fit in 80 GB"""
    from test_gpu_population_shapes import LARGEST, SMALLEST, _twin_run
    from ddls_b200 import workload
    cfgs = [SMALLEST, LARGEST, dict(SMALLEST, vf_share_layers=True), LARGEST]
    _twin_run(['ppo', 'impala', 'pg'], cfgs, graphs=[workload.make_graph('resnet')] + fan_graphs(256), compare=[0, 1])


def test_module_gradients_on_fan_job_types():
    from test_gpu_torch_policy import module_gradients_on_a_recorded_batch
    env, graphs = _fan_env(seed=11)
    module_gradients_on_a_recorded_batch(env, graphs, 6, 2, 'module fan seed 2')
