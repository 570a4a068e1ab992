"""Latency / throughput of the thread-per-lookahead kernel on the bench job's quotient (run on the GPU box).

    python scripts/microbench_thread.py [run_times [n ...]]
"""
import json
import sys

import numpy as np

sys.path.insert(0, '.')
from ddls_b200 import synth, engine
from ddls_b200.template_builder import build_template, RampShape

mode = sys.argv[1] if len(sys.argv) > 1 else 'one_to_one'
g = synth.resnet_like_graph()
eng = engine.RampEngine(n_episodes=4096, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
tids = [eng.register_template(build_template(g, d, RampShape(4, 4, 4), run_times=mode)) for d in (2, 4, 8, 16)]
eng.run_lookaheads(np.array(tids, dtype=np.int32))
for n in [int(v) for v in sys.argv[2:]] or (1, 32, 128, 512, 1024, 2048, 4096, 8192, 16384):
    ids = np.array([tids[k % 4] for k in range(n)], dtype=np.int32)
    best = 1e9
    for _ in range(3):
        res, ms = eng.run_lookaheads(ids)
        best = min(best, ms)
    assert (res['status'] == 0).all()
    T = int(res['n_ticks'].max())
    print(json.dumps(dict(mode=mode, n=n, ms=round(best, 4), T=T, us_per_tick=round(best * 1e3 / T, 4),
                          lookaheads_per_s=round(n / best * 1e3))), flush=True)
