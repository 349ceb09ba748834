"""Summarise Nsight Compute outputs: launch list (csv) and raw-page metrics of .ncu-rep files."""
import collections, csv, subprocess, sys


def launch_list(path, top=22):
    lines = [l for l in open(path) if not l.startswith('==')]
    agg, tot = collections.OrderedDict(), 0.0
    for row in csv.DictReader(lines):
        if row.get('Metric Name') != 'gpu__time_duration.sum':
            continue
        v = float(row['Metric Value'].replace(',', ''))
        v = v / 1000.0 if row['Metric Unit'] == 'ns' else (v * 1000 if row['Metric Unit'] == 'ms' else v)
        a = agg.setdefault(row['Kernel Name'][:80], [0, 0.0])
        a[0] += 1; a[1] += v; tot += v
    out = [f'total {tot:.1f} us over {sum(a[0] for a in agg.values())} launches']
    for k, (n, v) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:top]:
        out.append(f'{v:10.1f} us {100*v/tot:5.1f}%  {n:4d} launches  avg {v/n:8.1f} us  {k}')
    return '\n'.join(out)


KEYS = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_tensor.sum', 'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread', 'launch__grid_size',
        'launch__block_size', 'smsp__inst_executed.sum', 'sm__cycles_elapsed.avg', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'lts__t_bytes.sum', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
        'smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct', 'smsp__warp_issue_stalled_barrier_per_warp_active.pct',
        'smsp__warp_issue_stalled_wait_per_warp_active.pct', 'smsp__warp_issue_stalled_short_scoreboard_per_warp_active.pct',
        'smsp__warp_issue_stalled_mio_throttle_per_warp_active.pct', 'smsp__warp_issue_stalled_lg_throttle_per_warp_active.pct']


def raw(path):
    txt = subprocess.run(['ncu', '-i', path, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    r = list(csv.reader(txt.splitlines()))
    hdr, units = r[0], r[1]
    out = []
    for row in r[2:]:
        out.append('kernel: ' + row[hdr.index('Kernel Name')])
        for k in KEYS:
            if k in hdr:
                out.append(f'  {k} = {row[hdr.index(k)]} {units[hdr.index(k)]}')
    return '\n'.join(out)


if __name__ == '__main__':
    for a in sys.argv[1:]:
        print('=====', a)
        print(launch_list(a) if a.endswith('.csv') else raw(a))
