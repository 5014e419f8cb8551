"""Print the key metrics of an .ncu-rep (development aid)."""
import csv, subprocess, sys
KEYS = ['gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'lts__t_bytes.sum', 'lts__t_sector_hit_rate.pct', 'l1tex__t_sector_hit_rate.pct', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread', 'launch__occupancy_limit_shared_mem',
        'launch__occupancy_limit_registers', 'launch__grid_size', 'launch__waves_per_multiprocessor',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_tensor.sum', 'sm__pipe_tensor_op_hmma_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active', 'l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed',
        'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'smsp__inst_executed.sum', 'sm__cycles_elapsed.avg',
        'sm__ctas_launched.sum', 'local_load', 'smsp__inst_executed_op_local_ld.sum', 'smsp__inst_executed_op_local_st.sum']
out = subprocess.run(['ncu', '-i', sys.argv[1], '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr = rows[0]
for r in rows[2:]:
    print('---', r[hdr.index('Kernel Name')][:90])
    for k in KEYS:
        if k in hdr:
            print('  %-75s %s %s' % (k, r[hdr.index(k)], rows[1][hdr.index(k)]))
    st = []
    for i, h in enumerate(hdr):
        if 'issue_stalled' in h and h.endswith('_per_issue_active.ratio') and 'not_issued' not in h:
            try:
                st.append((float(r[i]), h.replace('smsp__average_warps_issue_stalled_', '').replace('_per_issue_active.ratio', '')))
            except Exception:
                pass
    print('  stalls/issue:', ', '.join('%s %.2f' % (n, v) for v, n in sorted(st, reverse=True)[:7]))
    for i, h in enumerate(hdr):
        if 'tensor' in h and 'pct' in h:
            print('  %-75s %s' % (h, r[i]))
