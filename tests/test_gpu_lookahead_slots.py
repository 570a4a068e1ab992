"""-m gpu: the thread kernel's HBM slab pool and the lookahead windows of overlapped steps, against the in-order path.

A window holds only its lists; a CTA claims an HBM slab from one pool shared by every launch when its chunk may spill or keeps
its trace aside (a template's first, unhinted lookaheads, or a trace the pool could not place) and releases it when the chunk
ends.  Every case runs the same seeded segments on an engine created with RAMP_STEP_OVERLAP=0 and on the default one, and
compares them bit for bit (tests/test_gpu_step_overlap.py's harness)."""
import numpy as np
import pytest
import torch

from test_gpu_step_overlap import L, _engine, _run, _same, _workload
from test_gpu_thread_kernel import FCAP, ready_flows_template

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('config', ['cfg2-resnet50-32w', 'cfg3-resnet50-64w'])
def test_first_launches_in_many_windows(config):
    """Fresh engines at bench.py's batch: every template's first lookaheads are unhinted and run in the windows of several
    steps at once, so CTAs of different launches claim and release slabs side by side."""
    B = 4096
    wl, actions = _workload(config, B, seed=21)
    _same(_run(_engine(config, B, 0, False), wl, actions), _run(_engine(config, B, 0, True), wl, actions))


def test_spilling_template_beside_hinted_ones():
    """A template whose ready-flow frontier is larger than the shared-memory list (never hinted into shared memory, so every
    chunk of it spills to a slab) placed in every step beside the workload's hinted templates."""
    config, B = 'cfg3-resnet50-64w', 1024
    from ddls_b200.engine import action_row
    wl, actions = _workload(config, B, seed=13)
    spill = ready_flows_template(FCAP + 1, simple=False)
    spill_tid = len(wl.templates)                      # registered right after the workload's templates in both engines
    for p, a in enumerate(actions):
        rows = np.flatnonzero(a['template_id'] >= 0)[p % 5::5]
        for b in rows:
            action_row(a, int(b), spill_tid, spill.mount)

    def run(overlap):
        eng = _engine(config, B, 0, overlap)
        for t in wl.templates:
            eng.register_template(t)
        assert eng.register_template(spill) == spill_tid
        out = _run(eng, wl, actions)
        return eng, out
    _, ref = run(False)
    eng, got = run(True)
    _same(ref, got)
    assert eng.template_info(spill_tid)['max_f'] == FCAP + 1


def test_resets_with_every_window_in_flight():
    """Segments enqueued back to back with no host synchronisation: each reset is queued while the previous segment's windows
    are all in flight, and the next segment's plans wait for it."""
    from ddls_b200 import engine
    config, B, segments = 'cfg3-resnet50-64w', 2048, 3
    wl, actions = _workload(config, B, seed=17)

    def run(overlap):
        eng = _engine(config, B, 0, overlap)
        for t in wl.templates:
            eng.register_template(t)
        on_dev = [torch.from_numpy(a.view(np.uint8).reshape(B, -1).copy()).cuda() for a in actions]
        torch.cuda.synchronize()
        stats = torch.empty((segments, L, B, engine.STEP_STATS_LEN), dtype=torch.float64, device='cuda')
        ncs = torch.empty((segments, L, B), dtype=torch.int32, device='cuda')
        ep = torch.empty((segments, B, engine.EP_LEN), dtype=torch.float64, device='cuda')
        for s in range(segments):
            eng.reset(wl.arrivals)
            for p in range(L):
                eng.step_device(on_dev[p].data_ptr(), True, stats[s, p].data_ptr(), ncs[s, p].data_ptr())
            eng.export_episode_state_to(ep[s].data_ptr())
        eng.sync()
        eng.check_status()
        return [x.cpu().numpy() for x in (stats, ncs, ep)]
    for x, y in zip(run(False), run(True)):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_config5_batch():
    """Config 5 at bench.py's 16,384 episodes: the most chunks per step and the largest window lists."""
    config, B = 'cfg5-mix-128w', 16384
    wl, actions = _workload(config, B, seed=9)
    _same(_run(_engine(config, B, 0, False), wl, actions), _run(_engine(config, B, 0, True), wl, actions))
