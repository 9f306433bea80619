"""Summarise an `ncu --csv --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,
sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active` capture of one step into the JSON the bench line quotes
(e.g. out/conv_traffic.json).   python tools/ncu_conv_summary.py capture.csv out.json "source description" """
import csv
import json
import sys

rows = [r for r in csv.reader(open(sys.argv[1], errors="replace")) if len(r) > 14 and r[0].isdigit()]
per = {}
for r in rows:
    per.setdefault(r[0], {"name": r[4]})[r[12]] = float(r[14].replace(",", ""))
conv = [v for v in per.values() if "conv_tc" in v["name"]]
other = [v for v in per.values() if "conv_tc" not in v["name"]]
tk = "gpu__time_duration.sum"
pk = "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"
t_conv = sum(v[tk] for v in conv)
t_all = sum(v[tk] for v in per.values())
out = {"kernel": "conv_tc_kernel", "launches_per_step": len(conv),
       "mean_dram_bytes_per_launch": sum(v["dram__bytes_read.sum"] + v["dram__bytes_write.sum"] for v in conv) / max(1, len(conv)),
       "dram_read_bytes_per_step": sum(v["dram__bytes_read.sum"] for v in conv),
       "dram_write_bytes_per_step": sum(v["dram__bytes_write.sum"] for v in conv),
       "sum_kernel_time_us_under_ncu": t_conv / 1e3,
       "share_of_step_under_ncu": t_conv / t_all if t_all else None,
       "tensor_pipe_active_pct_time_weighted": sum(v[tk] * v.get(pk, 0.0) for v in conv) / t_conv if t_conv else None,
       "other_kernels": {v["name"][:40]: round(v[tk] / 1e3, 1) for v in other},
       "source": sys.argv[3] if len(sys.argv) > 3 else ""}
json.dump(out, open(sys.argv[2], "w"), indent=1)
print(json.dumps({k: v for k, v in out.items() if k != "other_kernels"}, indent=1))
