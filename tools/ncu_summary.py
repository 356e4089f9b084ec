"""Summarise .ncu-rep files (ncu --set full) into a small markdown/JSON table:
per launch: duration, DRAM bytes read+written, DRAM / L2 / tensor-pipe / issue utilisation, occupancy, registers."""
import csv
import io
import json
import subprocess
import sys

WANT = {
    "gpu__time_duration.sum": "us",
    "dram__bytes_read.sum": "dram_rd_MB",
    "dram__bytes_write.sum": "dram_wr_MB",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed": "dram_pct",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed": "l2_pct",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "tensor_pct",
    "sm__issue_active.avg.pct_of_peak_sustained_elapsed": "issue_pct",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "occupancy_pct",
    "launch__registers_per_thread": "regs",
    "launch__grid_size": "grid",
}


def rows_of(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    r = list(csv.reader(io.StringIO(out)))
    hdr, units = r[0], r[1]
    res = []
    for row in r[2:]:
        d = {"kernel": row[hdr.index("Kernel Name")].split("(")[0].replace("void ", "").replace("hb200::", "")}
        for k, short in WANT.items():
            if k in hdr:
                i = hdr.index(k)
                v = float(row[i].replace(",", "")) if row[i] not in ("", "n/a") else None
                u = units[i]
                if v is not None and short == "us":
                    v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(u, 1.0)
                if v is not None and short.endswith("_MB"):
                    v *= {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(u, 1.0)
                d[short] = v
        res.append(d)
    return res


def main():
    allrows = []
    for rep in sys.argv[1:]:
        allrows += rows_of(rep)
    print("| kernel | grid | us | DRAM rd+wr MB | GB/s | DRAM % | L2 % | tensor % | issue % | occ % | regs |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for d in allrows:
        tr = (d.get("dram_rd_MB") or 0) + (d.get("dram_wr_MB") or 0)
        d["traffic_MB"] = tr
        gbs = tr * 1e-3 / (d["us"] * 1e-6) if d.get("us") else 0
        f = lambda k: "-" if d.get(k) is None else f"{d[k]:.1f}"  # noqa: E731
        print(f"| {d['kernel'][:60]} | {int(d.get('grid') or 0)} | {d['us']:.1f} | {tr:.1f} | {gbs:.0f} | {f('dram_pct')} | "
              f"{f('l2_pct')} | {f('tensor_pct')} | {f('issue_pct')} | {f('occupancy_pct')} | {int(d.get('regs') or 0)} |")
    json.dump(allrows, open("/dev/stderr", "w"))


if __name__ == "__main__":
    main()
