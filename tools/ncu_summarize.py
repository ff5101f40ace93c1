"""Post-process `ncu --csv --log-file` output of one training step (tools/profile_step.py) into the two committed artefacts:

  profiles/r02_step_launches_ncu.csv   one row per launch: kernel, grid, block, time (us), DRAM read/write bytes, tensor-pipe %
  profiles/r02_gemm_traffic.json       DRAM bytes per cb_gemm launch + the sha1 of cb_gemm.cu they were measured on
                                       (bench.py reports roofline.traffic only while that sha1 matches the source tree)

    python tools/ncu_summarize.py tools_out/r02_step_metrics_ncu.csv
"""
import collections
import csv
import hashlib
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main(path, tag="r02"):
    with open(path) as f:
        lines = [l for l in f if l.startswith('"')]
    rows = collections.OrderedDict()
    for x in csv.DictReader(lines):
        k = x["ID"]
        r = rows.setdefault(k, {"kernel": x["Kernel Name"], "grid": x["Grid Size"], "block": x["Block Size"]})
        r[x["Metric Name"]] = float(x["Metric Value"].replace(",", "")) if x["Metric Value"] not in ("", "n/a") else 0.0
        r[x["Metric Name"] + "#unit"] = x["Metric Unit"]

    def byt(r, name):
        v, u = r.get(name, 0.0), r.get(name + "#unit", "byte")
        return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)

    def usec(r):
        v, u = r.get("gpu__time_duration.sum", 0.0), r.get("gpu__time_duration.sum#unit", "ns")
        return v * {"ns": 1e-3, "us": 1.0, "ms": 1e3, "usecond": 1.0, "nsecond": 1e-3, "msecond": 1e3}.get(u, 1e-3)
    out_csv = os.path.join(ROOT, "profiles", f"{tag}_step_launches_ncu.csv")
    agg = collections.defaultdict(lambda: [0, 0.0, 0.0, 0.0])
    tot = 0.0
    with open(out_csv, "w") as f:
        f.write("# ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,"
                "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active --clock-control none --profile-from-start off "
                "python tools/profile_step.py full   (ONE training step, eager; per-launch times are cold-cache and serialised)\n")
        f.write("id,kernel,grid,block,time_us,dram_read_bytes,dram_write_bytes,tensor_pipe_pct\n")
        for k, r in rows.items():
            name = re.sub(r"\(.*", "", r["kernel"]).replace("void ", "")
            t = usec(r)
            rd, wr = byt(r, "dram__bytes_read.sum"), byt(r, "dram__bytes_write.sum")
            tp = r.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0.0)
            f.write(f'{k},"{name}","{r["grid"]}","{r["block"]}",{t:.2f},{rd:.0f},{wr:.0f},{tp:.1f}\n')
            short = re.sub(r"<.*", "", name)
            a = agg[short]
            a[0] += 1
            a[1] += t
            a[2] += rd + wr
            a[3] += tp * t
            tot += t
    print(f"{len(rows)} launches, {tot / 1e3:.2f} ms serialised")
    summ = []
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        summ.append({"kernel": k, "launches": v[0], "total_us": round(v[1], 1), "share": round(v[1] / tot, 4),
                     "dram_bytes": v[2], "tensor_pipe_pct_time_weighted": round(v[3] / max(v[1], 1e-9), 1)})
        print(f"{k:44s} n={v[0]:5d} {v[1]:9.1f} us {100 * v[1] / tot:5.1f}%  dram {v[2] / 1e6:9.1f} MB  tensor {v[3] / max(v[1], 1e-9):5.1f}%")
    with open(os.path.join(ROOT, "profiles", f"{tag}_step_kernel_shares.json"), "w") as f:
        json.dump({"launches": len(rows), "serialised_ms": tot / 1e3, "kernels": summ}, f, indent=1)
    gem = [r for r in rows.values() if "cb_gemm" in r["kernel"]]
    if gem:
        rd = sum(byt(r, "dram__bytes_read.sum") for r in gem)
        wr = sum(byt(r, "dram__bytes_write.sum") for r in gem)
        tt = sum(usec(r) for r in gem)
        tp = sum(r.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0.0) * usec(r) for r in gem) / max(tt, 1e-9)
        sha = hashlib.sha1(open(os.path.join(ROOT, "celebbasis_b200", "csrc", "cb_gemm.cu"), "rb").read()).hexdigest()
        j = {"source": "ncu metrics pass over tools/profile_step.py full (one training step; cold caches per launch), post-processed "
                       "by tools/ncu_summarize.py", "kernel_source_sha1": sha, "launches": len(gem),
             "dram_read_bytes_per_step": rd, "dram_write_bytes_per_step": wr, "traffic_bytes_per_launch": (rd + wr) / len(gem),
             "sum_duration_us_cold": tt, "tensor_pipe_active_pct_time_weighted": tp}
        with open(os.path.join(ROOT, "profiles", f"{tag}_gemm_traffic.json"), "w") as f:
            json.dump(j, f, indent=1)
        print(json.dumps(j))


if __name__ == "__main__":
    main(sys.argv[1], *(sys.argv[2:3]))
