"""Summarise `ncu --set full` reports into one JSON file (per-kernel duration, DRAM traffic, ...).  Usage:

    python tools/ncu_summary.py [--out ncu_summary.json] sampler=prof.ncu-rep [matmul=...]

Groups that are not given keep what the JSON already holds."""
import csv, io, json, os, subprocess, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
OUT = 'ncu_summary.json'
KEEP = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread', 'launch__grid_size',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio',
        'smsp__inst_executed.sum', 'launch__occupancy_limit_registers', 'launch__waves_per_multiprocessor',
        'lts__t_sector_hit_rate.pct', 'l1tex__t_sector_hit_rate.pct', 'sm__warps_active.avg.per_cycle_active',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'lts__t_bytes.sum', 'lts__t_sectors_op_atom.sum', 'lts__t_sectors_op_red.sum',
        'smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio']


def rows_of(path):
    txt = subprocess.run(['ncu', '-i', path, '--page', 'raw', '--csv'], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units = rows[0], rows[1]
    out = []
    for r in rows[2:]:
        d = {'Kernel Name': r[hdr.index('Kernel Name')]}
        for k in KEEP:
            if k in hdr:
                v, u = r[hdr.index(k)], units[hdr.index(k)]
                if k.startswith('dram__bytes') and u == 'byte': v = str(float(v) / 1e6)      # MB like the other rows
                if k.startswith('dram__bytes') and u == 'Kbyte': v = str(float(v) / 1e3)
                if k == 'gpu__time_duration.sum' and u == 'ns': v = str(float(v) / 1e3)        # us
                d[k] = v
        out.append(d)
    return out


def main():
    global OUT
    args = sys.argv[1:]
    if args and args[0] == '--out':
        OUT = args[1]; args = args[2:]
    cur = json.load(open(OUT)) if os.path.exists(OUT) else {}
    for arg in args:
        grp, path = arg.split('=', 1)
        cur[grp] = rows_of(path)
    json.dump(cur, open(OUT, 'w'), indent=1)
    for grp, rows in cur.items():
        for d in rows:
            print(grp, d['Kernel Name'][:60], d.get('gpu__time_duration.sum'), 'us  dram MB r/w', d.get('dram__bytes_read.sum'), d.get('dram__bytes_write.sum'))


if __name__ == '__main__':
    main()
