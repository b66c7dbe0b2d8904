"""Prints the headline metrics of an `ncu --page raw --csv` dump (stdin or file)."""
import csv, sys
rows = list(csv.reader(open(sys.argv[1]) if len(sys.argv) > 1 else sys.stdin))
hdr, units = rows[0], rows[1]
want = ['gpu__time_duration.sum', 'smsp__inst_executed.sum', 'smsp__issue_active.avg.per_cycle_active', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'launch__registers_per_thread', 'launch__occupancy_limit', 'launch__grid_size', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
        'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum', 'smsp__average_warps_issue_stalled', 'smsp__thread_inst_executed_per_inst_executed.ratio',
        'dram__bytes_read.sum', 'dram__bytes_write.sum', 'lts__t_sector_hit_rate.pct', 'l1tex__throughput.avg.pct', 'sm__throughput.avg.pct',
        'launch__shared_mem', 'launch__waves', 'smsp__inst_executed_op_shared', 'lts__throughput.avg.pct', 'gpu__dram_throughput.avg.pct',
        'sm__cycles_elapsed.max', 'l1tex__t_sector_hit_rate.pct', 'smsp__pcsamp_sample_buffer']
for vals in rows[2:]:
    print("# kernel:", vals[hdr.index("Kernel Name")], "grid", vals[hdr.index("Grid Size")])
    for h, u, v in zip(hdr, units, vals):
        if any(h.startswith(w) for w in want) and 'pcsamp' not in h:
            print("%-90s %-16s %s" % (h, u, v))
