"""A/B bench.py environment knobs on one box: python tools/ab_bench.py - CB_FE_CTAS=48 CB_GEMM_CLUSTER_SK=0,CB_FE_CTAS=64 [-- extra
bench args].  Every argument is one configuration (comma-separated KEY=VALUE pairs, "-" = the defaults); one JSON line each."""
import json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
args = sys.argv[1:]
extra = []
if "--" in args:
    i = args.index("--")
    args, extra = args[:i], args[i + 1:]
for cfg in args:
    kv = dict(x.split("=", 1) for x in cfg.split(",")) if cfg != "-" else {}
    env = dict(os.environ, **kv)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "30", "--warmup", "5",
                          "--skip-cpu-baseline"] + extra, env=env, capture_output=True, text=True)
    line = None
    for l in out.stdout.splitlines():
        try:
            line = json.loads(l)
        except Exception:
            pass
    if line is None:
        print(json.dumps({"config": cfg, "failed": out.stderr[-2000:]}), flush=True)
        continue
    roof = line.get("roofline") or {}
    print(json.dumps({"config": cfg, "ms_per_step": line["ms_per_step"], "value": line["value"], "e2e": line["e2e"]["value"],
                      "gemm_ms_per_step": roof.get("gemm_ms_per_step"), "roofline_frac": roof.get("frac"),
                      "gemm_launches": roof.get("launches_per_step"), "pipeline": line.get("pipeline"),
                      "launches": line.get("gpu_launches_per_step"), "clocks": line.get("clocks")}), flush=True)
