"""Summarise an ncu --csv launch list carrying gpu__time_duration.sum, sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,
dram__bytes_read.sum and dram__bytes_write.sum per launch: per kernel family time share, TIME-WEIGHTED tensor-pipe %, DRAM bytes.
    python tools/layer_metrics_summary.py launches.csv [skip_first_n_launches]"""
import collections
import csv
import re
import sys


def main(path, skip=0):
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    r = csv.reader(lines)
    hdr = next(r)
    ki, ni, vi, ii, ui = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("ID"), hdr.index("Metric Unit")
    rows = collections.OrderedDict()
    for row in r:
        try:
            v = float(row[vi].replace(",", ""))
        except Exception:
            continue
        u = row[ui].lower()
        if row[ni].startswith("gpu__time"):
            v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(u, 1e-3)            # -> us
        if row[ni].startswith("dram__bytes"):
            v *= {"byte": 1.0, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1.0)  # -> bytes
        rows.setdefault(int(row[ii]), {"name": row[ki]})[row[ni]] = v
    fam = collections.OrderedDict()
    tot_t = tot_w = tot_b = 0.0
    for i, d in rows.items():
        if i < skip:
            continue
        n = d["name"]
        m = re.search(r"(conv_\w*kernel)(<[^>]*>)?", n)
        k = (m.group(1) + (m.group(2) or "")) if m else re.sub(r"<.*", "", n.split("(")[0]).replace("void ", "").replace("irn::", "")
        t = d.get("gpu__time_duration.sum", 0.0)
        tp = d.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0.0)
        b = d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)
        f = fam.setdefault(k, [0.0, 0.0, 0.0, 0])
        f[0] += t; f[1] += t * tp; f[2] += b; f[3] += 1
        tot_t += t; tot_w += t * tp; tot_b += b
    print("%-44s %10s %7s %7s %10s %9s" % ("kernel", "total us", "share", "count", "tensor %", "DRAM MB"))
    for k, (t, w, b, c) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
        print("%-44s %10.1f %6.1f%% %7d %10.1f %9.1f" % (k, t, 100 * t / tot_t, c, w / t if t else 0, b / 1e6))
    print("%-44s %10.1f %6.1f%% %7s %10.1f %9.1f   <- time-weighted tensor-pipe %% over all launches" % ("TOTAL", tot_t, 100.0, "", tot_w / tot_t, tot_b / 1e6))
    conv_t = sum(v[0] for k, v in fam.items() if k.startswith("conv_wg"))
    conv_w = sum(v[1] for k, v in fam.items() if k.startswith("conv_wg"))
    if conv_t:
        print("wgmma conv kernels only: %.1f us, time-weighted tensor pipe %.1f %%" % (conv_t, conv_w / conv_t))


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 0)
