"""Turn an `ncu --set full` report into a small per-kernel summary CSV:
    python tools/ncu_summary.py prof_fwd422.ncu-rep prof_fwd422_summary.csv
One line per metric: name,unit,value, preceded by kernel name / block / grid; one such block per launch in the report."""
import csv
import io
import subprocess
import sys


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    col = {n: i for i, n in enumerate(hdr)}
    with open(out, "w") as f:
      for vals in rows[2:]:             # one block per launch in the report
        if len(vals) < len(hdr) // 2:
            continue
        f.write(f"Kernel Name,,{vals[col['Kernel Name']]}\n")
        f.write(f"Block Size,,{vals[col['Block Size']]}\n")
        f.write(f"Grid Size,,{vals[col['Grid Size']]}\n")
        keep = ("dram__", "gpu__time", "lts__t_bytes", "lts__t_sector", "l1tex__t_bytes", "sm__throughput", "sm__warps_active",
                "smsp__inst_executed.sum", "smsp__issue_active", "launch__", "smsp__average_warp", "sm__inst_executed_pipe",
                "smsp__warp_issue_stalled", "smsp__warps_issue_stalled", "gpc__cycles_elapsed.max", "sm__cycles_active.avg")
        for i, n in enumerate(hdr):
            if n.startswith(keep) and i < len(vals) and vals[i] != "":
                f.write(f"{n},{units[i]},{vals[i].replace(',', '')}\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
