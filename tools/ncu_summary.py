"""`.ncu-rep` -> JSON summary of the launches it holds (one entry per kernel name: the LAST launch captured):
duration, tensor-pipe activity, DRAM bytes / throughput, occupancy, registers.
python tools/ncu_summary.py x.ncu-rep > x_ncu_summary.json"""
import csv
import io
import json
import re
import subprocess
import sys

KEEP = ["gpu__time_duration.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
        "launch__block_size", "launch__waves_per_multiprocessor", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "lts__t_sector_hit_rate.pct", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed"]


def main():
    out = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr = rows[0]
    units = rows[1]
    kn = hdr.index("Kernel Name")
    res = {}
    for r in rows[2:]:
        if len(r) != len(hdr):
            continue
        name = re.sub(r"\(.*", "", r[kn]).replace("cocos::(anonymous namespace)::", "")
        entry = {}
        for k in KEEP:
            if k in hdr:
                i = hdr.index(k)
                entry[k] = "%s %s" % (r[i], units[i])
        try:
            rd = float(r[hdr.index("dram__bytes_read.sum")].replace(",", ""))
            wr = float(r[hdr.index("dram__bytes_write.sum")].replace(",", ""))
            scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
            entry["dram_bytes_per_launch"] = rd * scale.get(units[hdr.index("dram__bytes_read.sum")], 1) + \
                wr * scale.get(units[hdr.index("dram__bytes_write.sum")], 1)
        except (ValueError, KeyError):
            pass
        res[name] = entry
    json.dump(res, sys.stdout, indent=1)


if __name__ == "__main__":
    main()
