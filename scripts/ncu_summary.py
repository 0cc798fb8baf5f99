"""Key metrics of an ncu report (first kernel) as JSON: python scripts/ncu_summary.py <rep> [out.json]"""
import csv, io, json, subprocess, sys
rep = sys.argv[1]
raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, vals = rows[0], rows[1], rows[2]
d = {h: (v, u) for h, u, v in zip(hdr, units, vals)}
want = ['Kernel Name', 'gpu__time_duration.sum', 'launch__grid_size', 'launch__block_size', 'launch__registers_per_thread',
        'launch__shared_mem_per_block_dynamic', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'smsp__issue_active.avg.pct_of_peak_sustained_active', 'smsp__warps_eligible.avg.per_cycle_active',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'smsp__inst_executed.sum', 'smsp__thread_inst_executed.sum',
        'sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active', 'sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_tc.avg.pct_of_peak_sustained_active', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_tma.avg.pct_of_peak_sustained_active',
        'l1tex__t_sector_pipe_lsu_mem_local_op_ld_hit_rate.pct', 'l1tex__t_sector_pipe_lsu_mem_local_op_st_hit_rate.pct',
        'l1tex__t_sector_pipe_lsu_mem_global_op_ld_hit_rate.pct', 'lts__t_sector_hit_rate.pct',
        'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed']
out = {}
for k in want:
    if k in d:
        v, u = d[k]
        try:
            v = float(v.replace(',', ''))
        except ValueError:
            pass
        out[k] = [v, u]
stalls = {h.split('smsp__average_warps_issue_stalled_')[-1].replace('_per_issue_active.ratio', ''): float(d[h][0])
          for h in hdr if h.startswith('smsp__average_warps_issue_stalled_') and h.endswith('_per_issue_active.ratio')}
tot = sum(stalls.values()) or 1.0
out['stall_share_pct'] = {k: round(100 * v / tot, 1) for k, v in sorted(stalls.items(), key=lambda kv: -kv[1])[:8]}
print(json.dumps(out, indent=1))
if len(sys.argv) > 2:
    json.dump(out, open(sys.argv[2], 'w'), indent=1)
