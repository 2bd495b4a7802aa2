"""One frame out of an `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv` launch list of
`tools/profile_frame.py` (all kernels captured, no -k filter: ncu's filter matches unqualified names only):
    python tools/frame_launches.py launches.csv out/prefix
keeps the launches from one LM-stack `stream_kernel` launch to the next (= one speech frame), drops the one-time weight-packing
kernels of the first frame, writes <prefix>.csv (the kept rows) and <prefix>.txt (per-kernel counts, time shares, DRAM bytes)."""
import collections
import csv
import re
import sys

src, prefix = sys.argv[1], sys.argv[2]
lines = [l for l in open(src) if not l.startswith("==")]
rows = list(csv.DictReader(lines))
byid = collections.OrderedDict()
for r in rows:
    byid.setdefault(int(r["ID"]), []).append(r)
ids = list(byid)
name = lambda i: byid[i][0]["Kernel Name"]
stream = [i for i in ids if "stream_kernel" in name(i)]
if len(stream) < 5:
    sys.exit("need at least two LM-stack launches in the capture (raise -c)")
lm_variant = re.search(r"stream_kernel<(?:\(unsigned int\))?(\d+)", name(stream[0])).group(1)      # the first stream launch of a frame is the LM stack
lm = [i for i in stream if lm_variant in name(i)]
start, end = lm[0], lm[1]
ONE_TIME = ("tile_pack_kernel", "set_float_kernel")
keep = [r for i in ids if start <= i < end for r in byid[i] if not any(k in r["Kernel Name"] for k in ONE_TIME)]
with open(prefix + ".csv", "w") as f:
    w = csv.DictWriter(f, fieldnames=list(rows[0].keys()))
    w.writeheader()
    w.writerows(keep)
agg = collections.defaultdict(lambda: [0, 0.0, 0.0, 0.0])
for r in keep:
    k = re.sub(r"\(.*", "", r["Kernel Name"]).replace("void ", "")
    m2 = re.search(r"stream_kernel<(?:\(unsigned int\))?(\d+)", r["Kernel Name"])
    if m2:
        k = "vv::stream_kernel<%s>" % m2.group(1)
    v = float(r["Metric Value"].replace(",", ""))
    a = agg[k]
    if r["Metric Name"] == "gpu__time_duration.sum":
        a[0] += 1; a[1] += v / 1e3
    elif r["Metric Name"] == "dram__bytes_read.sum":
        a[2] += v / 1e6
    elif r["Metric Name"] == "dram__bytes_write.sum":
        a[3] += v / 1e6
tot = sum(a[1] for a in agg.values())
out = ["%-44s %6s %10s %7s %13s %14s" % ("kernel", "count", "time us", "share", "dram read MB", "dram write MB")]
for k, a in sorted(agg.items(), key=lambda x: -x[1][1]):
    out.append("%-44s %6d %10.1f %6.1f%% %13.1f %14.1f" % (k[:44], a[0], a[1], 100 * a[1] / tot, a[2], a[3]))
R, W = sum(a[2] for a in agg.values()), sum(a[3] for a in agg.values())
out.append("%-44s %6d %10.1f %7s %13.1f %14.1f" % ("TOTAL", sum(a[0] for a in agg.values()), tot, "", R, W))
out.append("frame DRAM traffic = %.3f GB read + %.3f GB written = %.3f GB" % (R / 1e3, W / 1e3, (R + W) / 1e3))
open(prefix + ".txt", "w").write("\n".join(out) + "\n")
print("\n".join(out))
