"""Turn an `ncu --metrics gpu__time_duration.sum --csv` launch list into a markdown table."""
import csv
import sys
from collections import OrderedDict

src, title = sys.argv[1], sys.argv[2]
rows = [r for r in csv.reader(open(src)) if len(r) > 10]
hdr = rows[0]
ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
gi, bi = hdr.index("Grid Size"), hdr.index("Block Size")
agg = OrderedDict()
for r in rows[1:]:
    name = r[ki]
    ours = any(t in name for t in ("fast::", "gen::", "count::", "tpf::", "bcjr::", "ldpc::", "bulk::", "demap::", "txlink::", "turbolink::", "count_errors"))
    key = (name if ours else "(torch data-generation / copy kernels, outside the timed region)", r[gi], r[bi])
    a = agg.setdefault(key, [0, 0.0])
    a[0] += 1
    a[1] += float(r[vi].replace(",", "")) / 1000.0
tot = sum(a[1] for a in agg.values())
print("# %s\n" % title)
print("`ncu --metrics gpu__time_duration.sum --clock-control none --csv`; per-launch times are cold-cache and serialised: compare SHARES, not absolutes.\n")
print("| kernel | grid | block | launches | mean us | total us | share |\n|---|---|---|---|---|---|---|")
for (name, g, b), (n, t) in agg.items():
    print("| `%s` | %s | %s | %d | %.1f | %.1f | %.1f %% |" % (name[:110], g, b, n, t / n, t, 100 * t / tot))
