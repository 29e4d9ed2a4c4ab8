"""ncu per-launch metrics CSV of ONE forward + pose solve at the bench shape (scripts/one_forward.py; the launches from the
last stem kernel on) -> per-kernel-family table with DRAM bytes, achieved DRAM GB/s, tensor-pipe activity, and a JSON summary
(the `backbone` block is what bench.py's roofline.traffic reads).
usage: launch_metrics_table.py <csv> <out.json> [hbm_peak_gbs]"""
import collections, csv, json, sys
rows = list(csv.reader(open(sys.argv[1])))
peak = float(sys.argv[3]) if len(sys.argv) > 3 else 6567.1
hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r); h = rows[hi]
idi, ki, mi, vi, ui = h.index("ID"), h.index("Kernel Name"), h.index("Metric Name"), h.index("Metric Value"), h.index("Metric Unit")
d, names = collections.OrderedDict(), {}
for r in rows[hi + 1:]:
    if len(r) > vi and r[vi]:
        d.setdefault(int(r[idi]), {})[r[mi]] = (float(r[vi].replace(",", "")), r[ui])
        names[int(r[idi])] = r[ki].split("(")[0].split("::")[-1]
ids = sorted(d)
stems = [i for i in ids if "stem" in names[i]]
ids = [i for i in ids if i >= stems[-1]]                      # the last forward
SC = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
def b(x): return x[0] * SC[x[1]]
BACKBONE = ["layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv1", "layer1.1.conv2", "layer2.0.conv1", "layer2.0.down",
            "layer2.0.conv2", "layer2.1.conv1", "layer2.1.conv2", "layer3.0.conv1", "layer3.0.down", "layer3.0.conv2",
            "layer3.1.conv1", "layer3.1.conv2", "layer3_outconv", "layer2_outconv", "layer2_outconv2.0", "layer2_outconv2.3",
            "layer1_outconv", "layer1_outconv2.0", "layer1_outconv2.3"]
recs, n_conv = [], 0
for i in ids:
    m = d[i]
    t = m["gpu__time_duration.sum"]; us = t[0] / 1e3 if t[1].startswith("n") else t[0]
    name = names[i]
    label = name
    if name.startswith("conv_gemm"):
        label = BACKBONE[n_conv] if n_conv < len(BACKBONE) else "gemm#%d" % n_conv
        n_conv += 1
    rd, wr = b(m["dram__bytes_read.sum"]), b(m["dram__bytes_write.sum"])
    recs.append({"id": i, "kernel": name, "label": label, "us": round(us, 2), "dram_read": rd, "dram_write": wr,
                 "dram_gbs": round((rd + wr) / us / 1e3, 1) if us > 0 else 0.0, "l2_bytes": b(m["lts__t_bytes.sum"]),
                 "tensor_active_pct": m["sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"][0],
                 "sm_ghz": round(m["sm__cycles_elapsed.avg.per_second"][0] / 1e9, 3)})
# the correlation GEMM is the conv_gemm launch right before stats_fused
for k, r in enumerate(recs):
    if r["kernel"].startswith("stats_fused") and k > 0:
        j = k - 1
        while j >= 0 and not recs[j]["kernel"].startswith("conv_gemm"): j -= 1
        recs[j]["label"] = "correlation (X.Y^T -> S)"
tot_us = sum(r["us"] for r in recs)
print(f"{len(recs)} launches of one forward + pose solve, {tot_us:.1f} us (serialised, cold-cache ncu replay times); HBM peak {peak} GB/s (measured)")
print(f"{'launch':28s} {'us':>8s} {'DRAM rd MB':>10s} {'DRAM wr MB':>10s} {'GB/s':>7s} {'of peak':>7s} {'tensor %':>8s} {'SM GHz':>6s}")
def row(label, rs):
    us = sum(r["us"] for r in rs); rd = sum(r["dram_read"] for r in rs); wr = sum(r["dram_write"] for r in rs)
    ta = sum(r["tensor_active_pct"] * r["us"] for r in rs) / us if us else 0
    print(f"{label:28s} {us:8.1f} {rd/1e6:10.1f} {wr/1e6:10.1f} {(rd+wr)/us/1e3:7.0f} {(rd+wr)/us/1e3/peak:7.2f} {ta:8.1f} {sum(r['sm_ghz']*r['us'] for r in rs)/us:6.3f}")
for r in recs:
    if r["label"] in BACKBONE or r["label"].startswith("correlation"):
        row(r["label"], [r])
groups = collections.OrderedDict()
for r in recs:
    if r["label"] in BACKBONE: g = "= backbone (21 conv launches)"
    elif r["label"].startswith("correlation"): continue
    elif r["kernel"].startswith("conv_gemm"): g = "= other tensor-core GEMMs (q|k|v, fine level)"
    else: g = r["kernel"]
    groups.setdefault(g, []).append(r)
print("-- by kernel family")
for g, rs in sorted(groups.items(), key=lambda kv: -sum(r["us"] for r in kv[1])):
    row(f"{g[:24]} x{len(rs)}", rs)
bb = [r for r in recs if r["label"] in BACKBONE]
out = {"launches": recs, "backbone": {k: sum(r[k] for r in bb) for k in ("us", "dram_read", "dram_write", "l2_bytes")},
       "backbone_tensor_active_pct_time_weighted": sum(r["tensor_active_pct"] * r["us"] for r in bb) / max(1e-9, sum(r["us"] for r in bb)),
       "total_us": tot_us}
print(f"backbone time-weighted tensor-pipe active: {out['backbone_tensor_active_pct_time_weighted']:.1f} %")
json.dump(out, open(sys.argv[2], "w"), indent=1)
