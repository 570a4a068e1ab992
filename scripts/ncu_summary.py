"""Summarises an `ncu --set full` report of bench.py's lookahead launches (run HERE, on the report copied back in gpurun_out/):

    python scripts/ncu_summary.py gpurun_out/prof_bench.ncu-rep "<what>" [out.json] [lookaheads per launch]

Writes profiles/ncu_lookahead_summary.json by default."""
import csv, json, subprocess, sys, os

rep = sys.argv[1]
what = sys.argv[2] if len(sys.argv) > 2 else ''
raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr = rows[0]
col = {h: i for i, h in enumerate(hdr)}


def f(r, name, default=0.0):
    try:
        return float(r[col[name]])
    except Exception:
        return default


launches = []
for r in rows[2:]:
    if len(r) < len(hdr):
        continue
    name = r[col['Kernel Name']]
    if 'ramp_lookahead' not in name:
        continue
    rd, wr = f(r, 'dram__bytes_read.sum'), f(r, 'dram__bytes_write.sum')
    unit_rd = rows[1][col['dram__bytes_read.sum']]
    unit_wr = rows[1][col['dram__bytes_write.sum']]
    scale = {'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9}
    launches.append({
        'kernel': name.split('(')[0].replace('void ramp::', '').replace('ramp::', ''),
        'grid': int(f(r, 'launch__grid_size')), 'block': int(f(r, 'launch__block_size')),
        'ms': f(r, 'gpu__time_duration.sum') * {'ns': 1e-6, 'us': 1e-3, 'usecond': 1e-3, 'msecond': 1.0, 'ms': 1.0, 'second': 1e3}.get(rows[1][col['gpu__time_duration.sum']], 1e-6),
        'dram_read_MB': rd * scale.get(unit_rd, 1.0) / 1e6, 'dram_write_MB': wr * scale.get(unit_wr, 1.0) / 1e6,
        'issue_active_pct': f(r, 'smsp__issue_active.avg.pct_of_peak_sustained_active'),
        'regs': int(f(r, 'launch__registers_per_thread')),
        'warps_active_pct': f(r, 'sm__warps_active.avg.pct_of_peak_sustained_active'),
        'l2_hit_pct': f(r, 'lts__t_sector_hit_rate.pct'),
        'inst': f(r, 'smsp__inst_executed.sum'),
    })
# group launches of the same step: a bench step launches the thread kernel, the CTA kernel or both, the thread kernel first
total_bytes = sum((l['dram_read_MB'] + l['dram_write_MB']) * 1e6 for l in launches)
n_steps = sum(1 for l in launches if 'cta' not in l['kernel']) or len(launches)
out = {'_what': what, 'dram_bytes_per_launch': total_bytes / max(n_steps, 1), 'n_launches': len(launches), 'n_steps': n_steps,
       'launches': launches}
path = sys.argv[3] if len(sys.argv) > 3 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'profiles', 'ncu_lookahead_summary.json')
if len(sys.argv) > 4 and launches:
    per = float(sys.argv[4])
    thr = [l for l in launches if 'thread' in l['kernel']]
    if thr:
        # one warp carries 32 lookaheads: warp instructions x 32 / lookaheads = instructions per lookahead (thread-level stream)
        out['warp_inst_per_lookahead'] = sum(l['inst'] for l in thr) * 32.0 / (per * len(thr))
        out['lookaheads_per_launch'] = per
json.dump(out, open(path, 'w'), indent=1)
print('wrote', path, 'dram bytes per step', out['dram_bytes_per_launch'], 'over', n_steps, 'steps')
