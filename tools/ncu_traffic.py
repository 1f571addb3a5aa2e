"""Summarise an `ncu --set full` capture of one kernel: per-launch DRAM traffic and the
main pipe / stall counters. Run where `ncu` can read the .ncu-rep.

usage: python tools/ncu_traffic.py <report.ncu-rep> <kernel-substring> <workload> <batch> [out.json=render_traffic.json]
Writes/updates the JSON (one entry per workload/batch) and prints a markdown table of the main counters.
"""
import csv
import io
import json
import os
import subprocess
import sys

WANT = [
    'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'lts__t_bytes.sum', 'lts__t_sector_hit_rate.pct',
    'l1tex__t_sector_hit_rate.pct', 'sm__inst_executed.sum', 'sm__issue_active.avg.pct_of_peak_sustained_active',
    'sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
    'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active',
    'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_tensor.sum',
    'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread', 'launch__shared_mem_per_block_dynamic',
    'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'smsp__pcsamp_warps_issue_stalled_long_scoreboard',
    'smsp__pcsamp_warps_issue_stalled_wait', 'smsp__pcsamp_warps_issue_stalled_mio_throttle', 'smsp__pcsamp_warps_issue_stalled_short_scoreboard',
    'smsp__pcsamp_warps_issue_stalled_barrier', 'smsp__pcsamp_warps_issue_stalled_not_selected', 'smsp__pcsamp_warps_issue_stalled_selected',
    'smsp__pcsamp_warps_issue_stalled_math_pipe_throttle', 'smsp__pcsamp_sample_buffer_full',
]
UNIT = {'Gbyte': 1e9, 'Mbyte': 1e6, 'Kbyte': 1e3, 'byte': 1.0, 'ms': 1e-3, 'us': 1e-6, 'ns': 1e-9, 's': 1.0, 'msecond': 1e-3,
        'usecond': 1e-6, 'nsecond': 1e-9, 'second': 1.0}


def raw_rows(rep):
    out = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    return hdr, units, rows[2:]


def main():
    rep, kern, workload, batch = sys.argv[1], sys.argv[2], sys.argv[3], int(sys.argv[4])
    out_path = sys.argv[5] if len(sys.argv) > 5 else 'render_traffic.json'
    hdr, units, rows = raw_rows(rep)
    ik = hdr.index('Kernel Name')
    rows = [r for r in rows if kern in r[ik]]
    assert rows, f'no launch of {kern} in {rep}'
    vals = {}
    for name in WANT:
        if name in hdr:
            j = hdr.index(name)
            xs = []
            for r in rows:
                try:
                    xs.append(float(r[j].replace(',', '')) * UNIT.get(units[j], 1.0))
                except ValueError:
                    pass
            if xs:
                vals[name] = sum(xs) / len(xs)
    dram = vals.get('dram__bytes_read.sum', 0.0) + vals.get('dram__bytes_write.sum', 0.0)
    entry = {'workload': workload, 'batch': batch, 'kernel': rows[0][ik].split('(')[0], 'launches_averaged': len(rows),
             'dram_bytes_per_launch': dram, 'dram_read_bytes': vals.get('dram__bytes_read.sum'), 'dram_write_bytes': vals.get('dram__bytes_write.sum'),
             'duration_s_under_ncu': vals.get('gpu__time_duration.sum'), 'source': os.path.basename(rep) + ' (ncu --set full --clock-control none)',
             'metrics': vals}
    data = {'captures': []}
    if os.path.exists(out_path):
        with open(out_path) as fh:
            data = json.load(fh)
    data['captures'] = [e for e in data['captures'] if not (e['workload'] == workload and e['batch'] == batch)] + [entry]
    with open(out_path, 'w') as fh:
        json.dump(data, fh, indent=1)
    print(f'| metric | value |\n|---|---|')
    for k, v in vals.items():
        print(f'| `{k}` | {v:.6g} |')
    print(f'| dram read + write per launch | {dram / 1e6:.1f} MB |')


if __name__ == '__main__':
    main()
