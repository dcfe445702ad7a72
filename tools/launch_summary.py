#!/usr/bin/env python
"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel (shares, not absolutes)."""
import collections, csv, re, signal, sys
signal.signal(signal.SIGPIPE, signal.SIG_DFL)
path = sys.argv[1]
lines = [l for l in open(path) if not l.startswith("==")]
agg = collections.defaultdict(lambda: [0, 0.0]); tot = 0.0
for row in csv.DictReader(lines):
    try:
        v = float(row["Metric Value"].replace(",", ""))
    except Exception:
        continue
    unit = row["Metric Unit"]
    v = v / 1e3 if unit == "ns" else v * 1e3 if unit == "ms" else v
    name = re.sub(r"\(.*", "", row["Kernel Name"]).replace("<unnamed>::", "")
    m = re.search(r"gemm_simt_kernel<(\d), (\d)>", row["Kernel Name"])
    if m:
        name = {"21": "gemm_simt<A_GATHER,B_NC> (SIMT conv fprop/dgrad, small linears)",
                "12": "gemm_simt<A_MC,B_GATHER> (SIMT conv wgrad split-K)"}.get(m.group(1) + m.group(2),
                "gemm_simt<%s,%s> (attention batched GEMM)" % m.groups())
    m = re.search(r"conv_tc_kernel<(\d+)>", row["Kernel Name"])
    if m:
        name = "conv_tc_kernel<BN=%s> (3xTF32 fprop/dgrad)" % m.group(1)
    m = re.search(r"wgrad_tc_kernel", row["Kernel Name"])
    if m:
        name = "wgrad_tc_kernel (fp16 wgmma, 3-product fp16 split: wgrad)"
    for kn, label in (("conv_tc_ps_kernel", "conv_tc_ps_kernel (fp16 wgmma, 3-product fp16 split: fprop/dgrad/NT GEMM, persistent)"),
                      ("conv_tc_ts_kernel", "conv_tc_ts_kernel<64> (3xTF32 fprop/dgrad, <= 64 channels)"),
                      ("conv_bf16_kernel", "conv_bf16_kernel (bf16 wgmma fprop/dgrad, persistent)"),
                      ("wgrad_bf16_kernel", "wgrad_bf16_kernel (bf16 wgmma wgrad)")):
        if kn in row["Kernel Name"]:
            name = label
    agg[name][0] += 1; agg[name][1] += v; tot += v
print(f"total {tot/1e3:.2f} ms over {sum(n for n, _ in agg.values())} launches\n")
print("| kernel | launches | time (ms) | share |\n|---|---:|---:|---:|")
for k, (n, t) in sorted(agg.items(), key=lambda x: -x[1][1]):
    print(f"| `{k.strip()[:100]}` | {n} | {t/1e3:.3f} | {100*t/tot:.2f}% |")
