"""Where does the step's GEMM time go?  Records every cb_gemm descriptor of one training step, groups them by shape
signature, replays each group alone as a CUDA graph and prints time / TFLOP/s per group (sorted by total time)."""
import collections, ctypes, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import lib, ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from celebbasis_b200.train_step import CelebBasisStep
from oracle import torch_ref

kind = sys.argv[1] if len(sys.argv) > 1 else "full"
dev = torch.device("cuda:0")
params = workload.model_params(kind)
om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers(kind))
sd = synth.synth_state_dict(om, seed=0)
del om
eng = CelebBasisStep(params, sd, synth.synth_celeb_basis(seed=0), dev, tokenizer=SyntheticCLIPTokenizer())
batch, draws = workload.synth_batch(kind, B=1, seed=1234)
st_ = {"image": batch["image"].to(dev), "faces": batch["image_ori"]["faces"].to(dev), "t": draws["t"].to(dev),
       "noise": draws["noise"].to(dev), "eps": draws["posterior_eps"].to(dev)}
ids, map_np, _ = eng.prepare(batch["caption"])
ids_dev, map_dev = ids.to(dev), torch.from_numpy(map_np).to(dev)
ids_person = batch["image_ori"]["ids"].to(dev)

def step_device():
    return eng.run(st_["image"], st_["faces"], ids_person, ids_dev, map_dev, st_["t"], st_["noise"], st_["eps"])

for _ in range(2):
    step_device()
torch.cuda.synchronize()
step_graph = torch.cuda.CUDAGraph()          # kept alive: its private pool holds every buffer the descriptors point to
ops.GEMM_RECORD = []
with torch.cuda.graph(step_graph):
    step_device()
rec, ops.GEMM_RECORD = ops.GEMM_RECORD, None
step_graph.replay()
torch.cuda.synchronize()

L = lib.load()
groups = collections.OrderedDict()
for raw, flops in rec:
    g = lib.GemmDesc.from_buffer_copy(raw)
    key = (g.M, g.N, g.K, g.batch, g.batch_inner, g.conv, g.kh, g.stride, g.a_major, g.b_major, g.flip_taps, g.d_dtype,
           g.d_transposed, 1 if g.R else 0, g.act, g.img_h if g.conv else 0)
    groups.setdefault(key, []).append((g, flops))

rows = []
for key, items in groups.items():
    g0 = items[0][0]
    def run():
        lib.check(L.cb_gemm(ctypes.byref(g0), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "replay")
    run(); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(20):
            run()
    gr.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        gr.replay()
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / 60
    fl = items[0][1]
    rows.append(dict(M=key[0], N=key[1], K=key[2], batch=key[3], inner=key[4], conv=key[5], kh=key[6], stride=key[7], amaj=key[8],
                     bmaj=key[9], flip=key[10], dd=key[11], dT=key[12], R=key[13], act=key[14], h=key[15], count=len(items), us=round(us, 2),
                     total_us=round(us * len(items), 1), tflops=round(fl / us / 1e6, 1), gflop=round(fl / 1e9, 3),
                     cfg=[g0.tile_n, g0.splits, g0.stages, g0.cta_pair, g0.splitk_cluster]))
rows.sort(key=lambda r: -r["total_us"])
tot = sum(r["total_us"] for r in rows); totf = sum(r["gflop"] * r["count"] for r in rows)
print(f"# {len(rec)} GEMMs, {len(rows)} shapes, sum of isolated times {tot/1000:.2f} ms, {totf:.0f} GFLOP -> {totf/tot*1e3/1e3:.1f} TFLOP/s")
out = os.path.join(ROOT, "tools_out", "gemm_breakdown.jsonl")
with open(out, "w") as f:
    for r in rows:
        f.write(json.dumps(r) + "\n")
for r in rows[:60]:
    print(json.dumps(r))
