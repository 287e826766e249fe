"""dram__bytes_read.sum + dram__bytes_write.sum per launch of the two pair kernels from an `ncu --set full` capture
-> profiles/dram_traffic.json (what bench.py reports as roofline.traffic).

    python tools/ncu_dram_traffic.py prof.ncu-rep dragon_bath profiles/pair_kernels_ncu.txt
"""
import csv, io, json, os, subprocess, sys

rep, workload, source = sys.argv[1], sys.argv[2], sys.argv[3]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
kn, rd, wr = hdr.index("Kernel Name"), hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
acc = {"density": [], "force": []}
for r in rows[2:]:
    kind = "density" if "k_density" in r[kn] else "force" if "k_force" in r[kn] else None
    if kind:
        acc[kind].append(float(r[rd]) * scale[units[rd]] + float(r[wr]) * scale[units[wr]])
path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "dram_traffic.json")
try:
    out = json.load(open(path))
except Exception:
    out = {}
out[workload] = {k: sum(v) / len(v) for k, v in acc.items() if v}
out[workload]["source"] = source
out[workload]["note"] = ("per launch, ncu --set full --clock-control none (ncu flushes the caches before every replay: the "
                         "neighbour lists the density pass has just written are re-read from DRAM here, from L2 in a real step)")
json.dump(out, open(path, "w"), indent=1)
print(json.dumps(out[workload]))
