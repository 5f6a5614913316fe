"""Condense an ncu --set full report (.ncu-rep) into a handful of per-kernel metrics."""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum",
        "dram__bytes_write.sum", "lts__t_bytes.sum", "lts__t_requests_srcunit_tex_op_red.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "smsp__average_warp_latency_per_inst_issued.ratio"]


def rows(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    r = list(csv.reader(io.StringIO(out)))
    return r[0], r[1], r[2:]


def to_bytes(v, u):
    v = float(v.replace(",", ""))
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)


for path in sys.argv[1:]:
    hdr, units, data = rows(path)
    for d in data:
        name = d[hdr.index("Kernel Name")]
        print(f"## {path.split('/')[-1]} :: {name[:90]}")
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                print(f"  {k:70s} {d[i]:>16s} {units[i]}")
        st = sorted(((float(d[i].replace(",", "")), h) for i, h in enumerate(hdr)
                     if h.startswith("smsp__average_warps_issue_stalled") and h.endswith("_per_issue_active.ratio")), reverse=True)[:5]
        print("  top stalls (warps per issue):", ", ".join(f"{h.split('stalled_')[1].split('_per')[0]} {v:.2f}" for v, h in st))
        if "dram__bytes_read.sum" in hdr:
            i, j = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
            print(f"  DRAM bytes per launch: {to_bytes(d[i], units[i]) + to_bytes(d[j], units[j]):.4g}")
