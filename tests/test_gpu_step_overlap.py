"""-m gpu: overlapped steps against the in-order path, bit for bit.

An engine created with RAMP_STEP_OVERLAP=0 plans and runs every step's lookaheads in order; the default engine plans them ahead
of the step kernels that precede them (RAMP_MEMO_REFERENCE, resident templates).  Both run the same seeded segments the way
bench.py does (reset, L x step_device on device-resident action rows with no host synchronisation, fused empty steps) and must
agree on every step's statistics row (RAMP_SS_LOOKAHEAD_RAN included), the cluster-step counts, the exported episode state and
the memo statistics."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

L = 8


def _engine(config, B, memo_mode, overlap):
    from ddls_b200 import engine, workload
    cfg = workload.CONFIGS[config]
    os.environ['RAMP_STEP_OVERLAP'] = '1' if overlap else '0'
    try:
        return engine.RampEngine(n_episodes=B, n_cluster_workers=int(np.prod(cfg['shape'])), max_jobs=L, memo_mode=memo_mode,
                                 trace_cap=4096)
    finally:
        os.environ.pop('RAMP_STEP_OVERLAP', None)


def _workload(config, B, seed):
    """bench.py's scripted workload, with template ids numbered as registration numbers them (the same in every engine)."""
    from ddls_b200 import workload
    eng = _engine(config, B, 0, False)
    tmap = {}

    def jcts(templates):
        for i, t in enumerate(templates):
            tmap[i] = eng.register_template(t)
        return eng.run_lookaheads([tmap[i] for i in range(len(templates))])[0]['jct']
    wl = workload.generate(config, jcts, n_episodes=B, n_steps=L, seed=seed)
    actions = []
    for p in range(L):
        a = wl.actions[p].copy()
        placed = a['template_id'] >= 0
        a['template_id'][placed] = np.array([tmap[int(t)] for t in a['template_id'][placed]], dtype=np.int32)
        actions.append(a)
    return wl, actions


def _run(eng, wl, actions, segments=2, rewrite=False, register_late=()):
    """Segments as bench.py's device_step runs them.  rewrite: every step's actions are copied into one buffer on the engine stream
    right before the call (so they are written in stream order after the previous step).  register_late: templates registered
    after the first step of the first segment."""
    import torch
    from ddls_b200 import engine
    B = wl.n_episodes
    for t in wl.templates:
        eng.register_template(t)
    on_dev = [torch.from_numpy(a.view(np.uint8).reshape(B, -1).copy()).cuda() for a in actions]
    buf = torch.empty_like(on_dev[0])
    ext = torch.cuda.ExternalStream(eng.stream)
    torch.cuda.synchronize()
    stats = [torch.empty((B, engine.STEP_STATS_LEN), dtype=torch.float64, device='cuda') for _ in range(L)]
    ncs = [torch.empty(B, dtype=torch.int32, device='cuda') for _ in range(L)]
    out = []
    for seg in range(segments):
        eng.reset(wl.arrivals)
        for p in range(L):
            if rewrite:
                with torch.cuda.stream(ext):
                    buf.copy_(on_dev[(p + 1) % L])      # what the speculative plan may read: the wrong step's actions
                    buf.copy_(on_dev[p])
                src = buf
            else:
                src = on_dev[p]
            eng.step_device(src.data_ptr(), True, stats[p].data_ptr(), ncs[p].data_ptr())
            if seg == 0 and p == 0:
                for t in register_late:
                    eng.register_template(t)
        ep = torch.empty((B, engine.EP_LEN), dtype=torch.float64, device='cuda')
        eng.export_episode_state_to(ep.data_ptr())
        m = eng.memo_stats()
        m['lookaheads'] -= eng.speculative_unused()     # the lookaheads a plan used
        eng.sync()
        out.append(dict(stats=torch.stack(stats).cpu().numpy(), ncs=torch.stack(ncs).cpu().numpy(), ep=ep.cpu().numpy(), memo=m))
    eng.check_status()
    return out


def _same(a, b, racy_ran=False):
    """racy_ran: RAMP_MEMO_EXACT / RAMP_MEMO_SHARED share a lookahead between episodes, and which episode of a step runs it is
    decided by an atomic race, so RAMP_SS_LOOKAHEAD_RAN is compared as a per-step sum there."""
    for sa, sb in zip(a, b):
        assert sa['memo'] == sb['memo']
        for k in ('ncs', 'ep'):
            assert np.array_equal(sa[k].view(np.uint8), sb[k].view(np.uint8)), k
        x, y = sa['stats'].copy(), sb['stats'].copy()
        if racy_ran:
            r = _ss('lookahead_ran')
            assert np.array_equal(x[:, :, r].sum(axis=1), y[:, :, r].sum(axis=1))
            x[:, :, r] = 0.0
            y[:, :, r] = 0.0
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), 'stats'


@pytest.mark.parametrize('config,B', [('cfg2-resnet50-32w', 256), ('cfg3-resnet50-64w', 1024), ('cfg5-mix-128w', 1024)])
def test_overlap_matches_in_order(config, B):
    wl, actions = _workload(config, B, seed=11)
    ref = _run(_engine(config, B, 0, False), wl, actions)
    got_eng = _engine(config, B, 0, True)
    got = _run(got_eng, wl, actions)
    _same(ref, got)
    ran = sum(float(s['stats'][:, :, _ss('lookahead_ran')].sum()) for s in got)
    assert ran > 0
    assert got_eng.speculative_unused() >= 0


def _ss(name):
    from ddls_b200 import engine
    return engine.SS[name]


def test_overlap_actions_written_in_stream_order():
    """The speculative plan may read the previous copy; the commit re-plans those episodes and the repair launch runs them."""
    config, B = 'cfg3-resnet50-64w', 512
    wl, actions = _workload(config, B, seed=5)
    ref = _run(_engine(config, B, 0, False), wl, actions, rewrite=True)
    got = _run(_engine(config, B, 0, True), wl, actions, rewrite=True)
    _same(ref, got)


def test_overlap_skips_and_unknown_templates():
    """Skip rows and template_id = -1 rows, episodes that finish mid-segment (the scripts end them), as in-order."""
    config, B = 'cfg2-resnet50-32w', 256
    wl, actions = _workload(config, B, seed=3)
    rng = np.random.default_rng(0)
    for a in actions:
        a['flags'][rng.random(B) < 0.1] |= 1            # RAMP_ACT_SKIP
        a['template_id'][rng.random(B) < 0.1] = -1
    _same(_run(_engine(config, B, 0, False), wl, actions), _run(_engine(config, B, 0, True), wl, actions))


def test_overlap_templates_registered_between_steps():
    """Templates registered after the first step: their first (unhinted) lookaheads run while other windows run hinted ones."""
    from ddls_b200 import workload
    config, B = 'cfg3-resnet50-64w', 512
    wl, actions = _workload(config, B, seed=7)
    extra = workload.build_templates('cfg2-resnet50-32w')[3]
    _same(_run(_engine(config, B, 0, False), wl, actions, register_late=extra),
          _run(_engine(config, B, 0, True), wl, actions, register_late=extra))


@pytest.mark.parametrize('memo_mode', [1, 2, 3])
def test_other_memo_modes_unchanged(memo_mode):
    """Modes other than RAMP_MEMO_REFERENCE take the in-order path in either engine."""
    config, B = 'cfg2-resnet50-32w', 256
    wl, actions = _workload(config, B, seed=2)
    _same(_run(_engine(config, B, memo_mode, False), wl, actions), _run(_engine(config, B, memo_mode, True), wl, actions),
          racy_ran=memo_mode != 2)


def test_nonresident_templates_fall_back():
    """With a template on the CTA kernel registered, steps run in order and still match."""
    config, B = 'cfg2-resnet50-32w', 128
    wl, actions = _workload(config, B, seed=4)
    os.environ['RAMP_LOOKAHEAD_MODE'] = 'cta'
    try:
        from ddls_b200 import engine, workload
        cfg = workload.CONFIGS[config]
        big = engine.RampEngine(n_episodes=B, n_cluster_workers=int(np.prod(cfg['shape'])), max_jobs=L, memo_mode=0, trace_cap=4096)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)
    ref = _run(big, wl, actions)
    _same(ref, _run(_engine(config, B, 0, True), wl, actions))
