"""Per-lookahead latency vs concurrency for the lookahead kernel (run on the GPU box)."""
import sys, json
import numpy as np
sys.path.insert(0, '.')
from ddls_b200 import synth, engine
from ddls_b200.template_builder import build_template, RampShape
degree = int(sys.argv[1]) if len(sys.argv) > 1 else 16
t = build_template(synth.resnet_like_graph(), degree, RampShape(4, 4, 4))
eng = engine.RampEngine(n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
tid = eng.register_template(t)
eng.run_lookaheads(np.full(64, tid, dtype=np.int32))
for n in (1, 16, 132, 528, 1056, 2112, 4224, 8448):       # multiples of an H100's 132 SMs
    ids = np.full(n, tid, dtype=np.int32)
    best = min(eng.run_lookaheads(ids)[1] for _ in range(3))
    print(json.dumps(dict(n=n, ms=round(best, 3), per_s=round(n / best * 1e3))), flush=True)
