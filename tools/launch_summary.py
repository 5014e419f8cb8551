"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel (development aid)."""
import collections
import csv
import re
import sys


def load(path):
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    r = csv.reader(lines)
    hdr = next(r)
    ki, vi, ii = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("ID")
    gi = hdr.index("Grid Size") if "Grid Size" in hdr else None
    out = []
    for row in r:
        try:
            out.append((int(row[ii]), row[ki], float(row[vi].replace(",", "")), row[gi] if gi is not None else ""))
        except Exception:
            pass
    return out


def key(n):
    k = re.sub(r"<.*", "", n.split("(")[0]).replace("void ", "").replace("irn::", "")
    m = re.search(r"(conv_wg\w*kernel)(<[^>]*>)?", n)
    if m:
        k = m.group(1) + (m.group(2) or "")
    return k


def main():
    L = load(sys.argv[1])
    tot, cnt = collections.defaultdict(float), collections.Counter()
    for _, n, v, _ in L:
        tot[key(n)] += v
        cnt[key(n)] += 1
    T = sum(tot.values())
    print("%-40s %10s %7s %7s %10s" % ("kernel", "total ms", "share", "count", "avg us"))
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        print("%-40s %10.2f %6.1f%% %7d %10.1f" % (k[:40], v / 1e6, 100 * v / T, cnt[k], v / cnt[k] / 1e3))
    print("%-40s %10.2f" % ("TOTAL", T / 1e6))


if __name__ == "__main__":
    main()
