"""How far is each GEMM shape of the training step from what the H100 can do?  Records every cb_gemm descriptor of one
step (bs=1) as the benchmark's step issues them (stage_prefetch + stage_main: the same streams and workspace lanes, so
each descriptor carries the configuration its lane runs), groups them by shape, replays each group alone as a CUDA graph
and prints, per shape: time, FLOP, unique bytes (weights + A + D + R), the compute floor (989 TFLOP/s dense fp16) and the HBM floor (3.35 TB/s), the name of the
floor that bounds, the fraction of it achieved, and the launch configuration (the descriptor's autotuned tile width,
split, ring depth and reduction path -- 0 means the library's own choice -- plus the number of CTAs the launch ran).

    python tools/gemm_floors.py [tag]      -> tools_out/gemm_floors[_tag].jsonl, one JSON line per shape + a summary line
"""
import collections, ctypes, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import lib, ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from celebbasis_b200.train_step import CelebBasisStep
from oracle import torch_ref

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35          # H100 SXM data sheet: dense fp16 tensor rate, HBM3 bandwidth
tag = sys.argv[1] if len(sys.argv) > 1 else ""
dev = torch.device("cuda:0")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()

params = workload.model_params("full")
om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers("full"))
sd = synth.synth_state_dict(om, seed=0)
del om
eng = CelebBasisStep(params, sd, synth.synth_celeb_basis(seed=0), dev, tokenizer=SyntheticCLIPTokenizer())
batch, draws = workload.synth_batch("full", B=1, seed=1234)
st_ = {"image": batch["image"].to(dev), "faces": batch["image_ori"]["faces"].to(dev), "t": draws["t"].to(dev),
       "noise": draws["noise"].to(dev), "eps": draws["posterior_eps"].to(dev)}
ids, map_np, _ = eng.prepare(batch["caption"])
ids_dev, map_dev = ids.to(dev), torch.from_numpy(map_np).to(dev)
ids_person = batch["image_ori"]["ids"].to(dev)


def step_device():
    z, v = eng.stage_prefetch(st_["image"], st_["faces"], ids_person.shape[1], st_["eps"])
    return eng.stage_main(z, v, ids_person, ids_dev, map_dev, st_["t"], st_["noise"])


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
    key = (g.M, g.N, g.K, g.batch, g.batch_inner, g.conv, g.img_n, g.img_h, g.kh, g.stride, g.a_major, g.b_major,
           g.flip_taps, g.d_dtype, g.d_transposed, 1 if g.R else 0, g.act, g.glu)
    groups.setdefault(key, []).append((g, flops))


def unique_bytes(g):
    taps = g.kh * g.kw if g.conv else 1
    M = g.img_n * g.out_h * g.out_w if g.conv else g.M
    a = (g.img_n * g.img_h * g.img_w * g.K if g.conv else M * g.K * g.batch) * 2
    b_batches = g.batch if (g.b_batch_stride or g.b_batch_stride2) else 1
    w = taps * g.N * g.K * 2 * b_batches
    des = 4 if g.d_dtype == lib.CB_F32 else 2
    d = (M * g.N * g.batch * des if g.D else 0) + (M * (g.N // 2 if g.glu else g.N) * (4 if g.d2_dtype == lib.CB_F32 else 2)
                                                  if g.D2 else 0)
    r = M * g.N * g.batch * (4 if g.r_dtype == lib.CB_F32 else 2) if g.R else 0
    return w + a + d + r, w


timeline = torch.zeros(8 * 65536, dtype=torch.int64, device=dev)
rows = []
for key, items in groups.items():
    g0 = items[0][0]
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        lib.check(L.cb_gemm(ctypes.byref(g0), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "replay")
    # CTA count of the launch: every CTA stamps its slot of the debug timeline (separate launch, not timed)
    timeline.zero_()
    gt = lib.GemmDesc.from_buffer_copy(bytes(g0))
    gt.debug_timeline = timeline.data_ptr()
    lib.check(L.cb_gemm(ctypes.byref(gt), s), "timeline")
    torch.cuda.synchronize()
    ctas = int((timeline.view(-1, 8)[:, 7] != 0).sum().item())
    run(); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(20):
            run()
    for _ in range(2):
        gr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        gr.replay()
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / 100
    fl = items[0][1]
    ub, wb = unique_bytes(g0)
    t_comp, t_mem = fl / PEAK_TFLOPS / 1e6, ub / PEAK_TBS / 1e6
    floor = max(t_comp, t_mem)
    M = g0.img_n * g0.out_h * g0.out_w if g0.conv else g0.M
    rows.append(dict(M=M, N=g0.N, K=g0.K * (g0.kh * g0.kw if g0.conv else 1), batch=g0.batch, conv=g0.conv,
                     h=g0.img_h if g0.conv else 0, kh=g0.kh if g0.conv else 0, stride=g0.stride if g0.conv else 0,
                     amaj=g0.a_major, bmaj=g0.b_major, flip=g0.flip_taps, dd=g0.d_dtype, R=key[15], glu=g0.glu,
                     count=len(items), us=round(us, 2), total_us=round(us * len(items), 1), gflop=round(fl / 1e9, 3),
                     mb=round(ub / 1e6, 2), weight_mb=round(wb / 1e6, 2), floor_compute_us=round(t_comp, 2),
                     floor_hbm_us=round(t_mem, 2), bound="compute" if t_comp >= t_mem else "hbm",
                     frac_of_floor=round(floor / us, 3), tflops=round(fl / us / 1e6, 1), ctas=ctas,
                     cfg=dict(tile_n=g0.tile_n, splits=g0.splits, stages=g0.stages, cta_pair=g0.cta_pair,
                              splitk_cluster=g0.splitk_cluster)))
rows.sort(key=lambda r: -r["total_us"])
tot = sum(r["total_us"] for r in rows)
sub = sum(r["total_us"] for r in rows if r["ctas"] < torch.cuda.get_device_properties(dev).multi_processor_count * 2)
totf = sum(r["gflop"] * r["count"] for r in rows)
floor_tot = sum(max(r["floor_compute_us"], r["floor_hbm_us"]) * r["count"] for r in rows)
summary = dict(card=card, gemms=len(rec), shapes=len(rows), sum_isolated_ms=round(tot / 1000, 3),
               sum_floor_ms=round(floor_tot / 1000, 3), gflop=round(totf, 1), tflops=round(totf / tot * 1e3, 1),
               ms_in_launches_under_two_waves=round(sub / 1000, 3))
os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
out = os.path.join(ROOT, "tools_out", f"gemm_floors{'_' + tag if tag else ''}.jsonl")
with open(out, "w") as f:
    f.write(json.dumps({"summary": summary}) + "\n")
    for r in rows:
        f.write(json.dumps(r) + "\n")
print(json.dumps({"summary": summary}))
for r in rows[:40]:
    print(json.dumps(r))
