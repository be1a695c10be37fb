"""Summarise an .ncu-rep (one kernel launch, --set full) as markdown: key raw metrics, stall mix and, when the
object file is given, the per-sub-function split of samples / instructions.
usage: python scripts/ncu_summary.py x.ncu-rep [build/obj.o] > x.md"""
import csv, io, subprocess, sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
H, U, V = rows[0], rows[1], rows[2]
m = {h: (V[i], U[i]) for i, h in enumerate(H)}
keys = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static", "sm__cycles_elapsed.max",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_subpipe_hmma_cycles_active_realtime.avg", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_bytes.sum", "lts__t_sector_hit_rate.pct", "l1tex__t_requests_pipe_lsu_mem_local_op_ld.sum",
        "l1tex__t_requests_pipe_lsu_mem_local_op_st.sum", "l1tex__t_sector_pipe_lsu_mem_local_op_ld_hit_rate.pct",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"]
print("# ncu summary: %s\n" % rep.split("/")[-1])
print("Kernel: `%s`\n" % m.get("Kernel Name", ("?",))[0])
print("| metric | value | unit |\n|---|---|---|")
for k in keys:
    if k in m:
        print("| %s | %s | %s |" % (k, m[k][0], m[k][1]))
print("\n## Warp stall mix (cycles per issued instruction)\n\n| reason | ratio |\n|---|---|")
st = [(h.replace("smsp__average_warps_issue_stalled_", "").replace("_per_issue_active.ratio", ""), float(v[0]))
      for h, v in m.items() if h.startswith("smsp__average_warps_issue_stalled_") and "not_issued" not in h]
for n, v in sorted(st, key=lambda x: -x[1])[:9]:
    print("| %s | %.2f |" % (n, v))
if len(sys.argv) > 2:
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    open("/tmp/_src.csv", "w").write(src)
    out = subprocess.run([sys.executable, "scripts/ncu_by_function.py", "/tmp/_src.csv", sys.argv[2]], capture_output=True, text=True).stdout
    print("\n## Split by sub-function (sampling + executed warp instructions)\n\n```\n%s```" % out)
