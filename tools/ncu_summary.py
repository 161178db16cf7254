#!/usr/bin/env python
"""ncu_summary -- compact per-launch summary of an `ncu --set full` report (run where `ncu` is installed; no GPU needed):

    python tools/ncu_summary.py prof.ncu-rep prof_summary.json
"""
import csv
import json
import subprocess
import sys

METRICS = {
    "duration_us": "gpu__time_duration.sum",
    "tensor_pipe_pct_elapsed": "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "tensor_pipe_pct_active": "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm_throughput_pct": "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "dram_read_bytes": "dram__bytes_read.sum",
    "dram_write_bytes": "dram__bytes_write.sum",
    "dram_throughput_pct": "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts_throughput_pct": "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l2_to_sm_read_bytes": "l1tex__m_xbar2l1tex_read_bytes.sum",
    "smem_tc_wavefronts_pct": "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
    "smem_lsu_bank_conflicts": "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "warps_active_pct": "sm__warps_active.avg.pct_of_peak_sustained_active",
    "registers_per_thread": "launch__registers_per_thread",
    "dyn_smem_per_block_bytes": "launch__shared_mem_per_block_dynamic",
    "sm_cycles_elapsed_max": "sm__cycles_elapsed.max",
}
UNIT_SCALE = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "Kbyte/block": 1e3, "byte/block": 1.0, "msecond": 1e3, "usecond": 1.0, "nsecond": 1e-3,
              "second": 1e6}


def main():
    rep, out = sys.argv[1], sys.argv[2]
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(txt.splitlines()))
    hdr, units = rows[0], rows[1]
    col = {h: i for i, h in enumerate(hdr)}
    res = []
    for r in rows[2:]:
        if len(r) < len(hdr):
            continue
        e = {"kernel": r[col["Kernel Name"]].split("(")[0][:90], "grid": r[col["Grid Size"]], "block": r[col["Block Size"]]}
        for k, m in METRICS.items():
            if m not in col or r[col[m]] == "":
                continue
            v = float(r[col[m]].replace(",", ""))
            u = units[col[m]]
            if u in UNIT_SCALE and ("bytes" in k or k.endswith("_us")):
                v *= UNIT_SCALE[u]
            e[k] = round(v, 3)
        if "dram_read_bytes" in e and "dram_write_bytes" in e:
            e["dram_bytes"] = e["dram_read_bytes"] + e["dram_write_bytes"]
        res.append(e)
    json.dump({"source": rep, "how": "ncu --set full --clock-control none --import-source on (one launch per row; cold caches, serialised: compare shares, not absolutes)",
               "launches": res}, open(out, "w"), indent=1)
    print(len(res), "launches ->", out)


if __name__ == "__main__":
    main()
