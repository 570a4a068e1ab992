"""CPU: the float64 references tests/test_gpu_graph_topologies.py holds the GPU policy to, on that file's raw graphs (hubs of 4,096
out-edges, a node of 2,048 in- and 2,048 out-edges, 1,000 parallel edges, self-loops, no edges, a 2-cycle, a 2,000-node chain,
K64,64, degrees 31 / 32 / 33), pinned to the module restatement GNNPolicy (tests/gnn_reference.py) run in float64:

- gnn_reference.embed64 (numpy) equals GNNPolicy.embed to 1e-12;
- ppo_reference.policy64's autograd gradient of sum(gl logits) + sum(gv value) equals autograd through GNNPolicy to 1e-12 of each
  tensor's largest element."""
import numpy as np
import pytest
import torch

from ddls_b200 import policy as P
from test_gpu_graph_topologies import degrees, topologies
from test_gpu_policy_kernels import CONFIGS, SEED, _cfg


def test_the_graphs_reach_hub_degrees():
    gs = topologies()
    assert max(int(degrees(g)[0].max(initial=0)) for g in gs) >= 4096
    assert max(int(degrees(g)[1].max(initial=0)) for g in gs) >= 2048
    hub = {g.name: g for g in gs}['bi_hub']
    out_deg, in_deg = degrees(hub)
    assert out_deg[0] == in_deg[0] == 2048


@pytest.mark.parametrize('cid', ['yaml', 'odd'])
def test_references_equal_the_module_restatement_in_float64(cid):
    from gnn_reference import GNNPolicy, embed64
    from ppo_reference import params64, policy64
    over, A, _, _ = CONFIGS[cid]
    c = _cfg(over)
    sd = P.random_state_dict(c, A, seed=SEED)
    ref = GNNPolicy(c, A).double()
    ref.load_state_dict({k: torch.from_numpy(v.astype(np.float64)) for k, v in sd.items()}, strict=True)
    rng = np.random.default_rng(29)
    gs = [g.features(c, rng) for g in topologies()]
    for m, g in enumerate(gs):
        src, dst = torch.from_numpy(g.src.astype(np.int64)), torch.from_numpy(g.dst.astype(np.int64))
        nf, ef = torch.from_numpy(g.nf.astype(np.float64)), torch.from_numpy(g.ef.astype(np.float64))
        with torch.no_grad():
            want = ref.embed(nf, ef, src, dst).numpy()
        np.testing.assert_allclose(embed64(sd, c, g.nf, g.ef, g.src, g.dst), want, rtol=1e-12, atol=1e-12, err_msg=g.name)
        if m == 0:
            continue
        # rows of this graph and of the one-node graph, the backward of a linear function of the read-out
        n = 12
        model = np.where(np.arange(n) % 4 == 0, 0, m)
        gf = rng.standard_normal((n, c['in_features_graph']))
        mask = (rng.random((n, A)) < 0.6).astype(np.float64)
        mask[:, 0] = 1
        gl, gv = torch.from_numpy(rng.standard_normal((n, A))), torch.from_numpy(rng.standard_normal(n))
        p = params64(sd)
        logits, value = policy64(p, c, gs, model, gf, mask)
        grads = torch.autograd.grad((gl * logits).sum() + (gv * value).sum(), list(p.values()), allow_unused=True)
        embs = {u: ref.embed(*(torch.from_numpy(np.asarray(x, dtype=np.float64)) for x in (gs[u].nf, gs[u].ef)),
                             torch.from_numpy(gs[u].src.astype(np.int64)), torch.from_numpy(gs[u].dst.astype(np.int64)))
                for u in (0, m)}
        l2, v2 = ref(torch.stack([embs[u] for u in model]), torch.from_numpy(np.concatenate([gf, mask], 1)), torch.from_numpy(mask))
        torch.testing.assert_close(l2, logits, rtol=1e-12, atol=1e-12)
        named = dict(ref.named_parameters())
        want = torch.autograd.grad((gl * l2).sum() + (gv * v2).sum(), [named[k] for k in p], allow_unused=True)
        for k, a, b in zip(p, grads, want):
            zero = torch.zeros_like(p[k])                       # a weight a graph never reaches (the edge module without edges)
            a, b = zero if a is None else a, zero if b is None else b
            scale = float(b.abs().max())
            torch.testing.assert_close(a, b, rtol=0, atol=1e-12 * max(scale, 1.0), msg=f'{g.name} {k}')
