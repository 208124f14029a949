"""Prints the key metrics of an .ncu-rep (first kernel)."""
import csv, subprocess, sys
rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr, units = rows[0], rows[1]
keys = ['Kernel Name', 'gpu__time_duration.sum', 'launch__registers_per_thread', 'launch__grid_size', 'launch__block_size',
        'launch__shared_mem_per_block_dynamic', 'launch__occupancy_limit_registers', 'launch__occupancy_limit_shared_mem',
        'launch__occupancy_limit_warps', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active',
        'sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active',
        'dram__bytes_read.sum', 'dram__bytes_write.sum', 'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'smsp__inst_executed.sum',
        'smsp__thread_inst_executed_per_inst_executed.ratio', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
        'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum', 'sm__cycles_elapsed.avg', 'sm__cycles_active.avg',
        'smsp__inst_executed_pipe_fp64.sum', 'sm__sass_thread_inst_executed_op_dfma_pred_on.sum',
        'sm__sass_thread_inst_executed_op_dadd_pred_on.sum', 'sm__sass_thread_inst_executed_op_dmul_pred_on.sum',
        'smsp__sass_thread_inst_executed_op_dfma_pred_on.sum', 'smsp__sass_thread_inst_executed_op_dadd_pred_on.sum',
        'smsp__sass_thread_inst_executed_op_dmul_pred_on.sum', 'local_load', 'smsp__inst_executed_op_local_ld.sum']
for r in rows[2:]:
    for i, h in enumerate(hdr):
        if h in keys or ('issue_stalled' in h and h.endswith('per_warp_active.pct')):
            print(f"{h} [{units[i]}] = {r[i]}")
    print('-' * 40)
