import os, sys, json
import numpy as np
sys.path.insert(0, '.')
from ddls_b200 import synth, engine
from ddls_b200.template_builder import build_template, RampShape
mode, ctant, n = sys.argv[1], sys.argv[2], int(sys.argv[3])
os.environ['RAMP_LOOKAHEAD_MODE'] = mode
if ctant != '0':
    os.environ['RAMP_LOOKAHEAD_CTA_THREADS'] = ctant
g = synth.resnet_like_graph()
ts = [build_template(g, d, RampShape(4, 4, 4)) for d in (2, 4, 8, 16)]
eng = engine.RampEngine(n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
tids = [eng.register_template(t) for t in ts]
ref, _ = eng.run_lookaheads(tids)
per = []
for t in tids:
    ids = np.full(132, t, dtype=np.int32)             # one per SM of an H100
    per.append(round(min(eng.run_lookaheads(ids)[1] for _ in range(2)), 2))
rng = np.random.default_rng(0)
ids = rng.choice(tids, size=n).astype(np.int32)
res, ms = eng.run_lookaheads(ids)
ok = all(res['jct'][k] == ref['jct'][tids.index(ids[k])] and res['status'][k] == 0 for k in range(n))
print(mode, ctant, n, 'ms', round(ms, 2), 'ok', ok, 'per-degree latency ms (132 items)', per, flush=True)
