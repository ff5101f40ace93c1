"""How far is each flash-attention launch of the training step from what the H100 can do?  Records every
ops.attention_fwd / attention_bwd_dq / attention_bwd call of one step (bs=1), run as the benchmark's step runs it
(stage_prefetch + stage_main) -- so the shapes and paths are the ones the engines actually take -- groups them by
(kernel, shape), replays each group alone as a CUDA graph and prints, per group:
time per call, calls per step and time per step; the algorithmic FLOP and the MMA FLOP the kernel issues (head dim
padded to 16, PV / accumulation MMAs at N = 64 or 128, the statistics pass of the two-pass forward); the exp2 count; the
tensor floor (989 TFLOP/s dense fp16) and the exp floor (16 exp2 per clock per SM at the card's max SM clock); the
fraction of the bounding floor reached, the CTA count and the kernel instantiation.

cb_attention_bwd is two launches (dQ, then dK/dV): the dQ launch is timed alone through cb_attention_bwd_dq on the same
operands, and the dK/dV launch is the difference.

    python tools/attn_floors.py [tag]      -> tools_out/attn_floors[_tag].jsonl, one JSON line per group + a summary line
"""
import collections, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from celebbasis_b200.train_step import CelebBasisStep
from oracle import torch_ref

PEAK_TFLOPS = 989.0          # H100 SXM data sheet: dense fp16 / bf16 tensor rate
EXP2_PER_CLK_SM = 16         # MUFU ex2 throughput per SM per clock
BQ, BKV = 128, 64            # query (stationary) rows per CTA, keys (streamed items) per block
tag = sys.argv[1] if len(sys.argv) > 1 else ""
dev = torch.device("cuda:0")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                      capture_output=True, text=True).stdout.strip()
max_sm_mhz = float(card.split(",")[2])
n_sm = torch.cuda.get_device_properties(dev).multi_processor_count

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


# record the attention calls of one captured step (the graph is kept alive: its pool holds the recorded operands)
RECORD = None
_orig = {name: getattr(ops, name) for name in ("attention_fwd", "attention_bwd_dq", "attention_bwd")}


def _recorder(name):
    def wrapped(*args, **kw):
        if RECORD is not None:
            RECORD.append((name, args, dict(kw)))
        return _orig[name](*args, **kw)
    return wrapped


for name in _orig:
    setattr(ops, name, _recorder(name))
for _ in range(2):
    step_device()
torch.cuda.synchronize()
step_graph = torch.cuda.CUDAGraph()
RECORD = []
with torch.cuda.graph(step_graph):
    step_device()
rec, RECORD = RECORD, None
step_graph.replay()
torch.cuda.synchronize()


def pairs(nq, nk, causal):
    """(query, key) pairs the attention computes: all of them, or keys <= query."""
    if not causal:
        return nq * nk
    return sum(min(q + 1, nk) for q in range(nq))


def counts(kernel, nq, nk, d, heads, images, causal, two_pass=False):
    """(CTAs, MMA FLOP issued, exp2 count) of one launch, block for block as the kernel walks them."""
    ks = (d + 15) // 16
    no = 64 * ((ks + 3) // 4)
    qk = 2 * BQ * BKV * 16 * ks                         # one T = X Y^T group over 64 streamed items
    acc = 2 * BQ * BKV * no                             # one accumulation group over 64 streamed items
    n_stat, n_stream = (nk, nq) if kernel == "bwd_dkdv" else (nq, nk)
    tiles = (n_stat + BQ - 1) // BQ
    blocks = 0
    mma = 0
    for t in range(tiles):
        x0 = t * BQ
        jbeg, jend = 0, (n_stream + BKV - 1) // BKV
        if causal:
            if kernel == "bwd_dkdv":
                jbeg = x0 // BKV
            else:
                jend = min(jend, (min(x0 + BQ, n_stat) + BKV - 1) // BKV)
        nb = max(0, jend - jbeg)
        if kernel == "fwd":
            nv = 2 * nb if two_pass else nb
            mma += nv * qk + nb * acc
            blocks += nv
        elif kernel == "bwd_dq":
            mma += nb * (2 * qk + acc)
            blocks += nb
        else:
            mma += nb * (2 * qk + 2 * acc)
            blocks += nb
    return tiles * heads * images, mma * heads * images, blocks * BQ * BKV * heads * images


def timed(fn, reps=20, rounds=5):
    fn(); torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(reps):
            fn()
    for _ in range(2):
        gr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(rounds):
        gr.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000 / (reps * rounds)


groups = collections.OrderedDict()
for name, args, kw in rec:
    q = args[0]
    shape = (kw["images"], kw["heads"], kw["dh"], kw["nq"], kw["nk"], bool(kw.get("causal", False)), str(q.dtype))
    if name == "attention_fwd":
        key = ("fwd_2pass_P" if kw.get("want_p") else "fwd",) + shape
    elif name == "attention_bwd_dq":
        key = ("bwd_dq_dS",) + shape
    else:
        key = ("bwd",) + shape
    groups.setdefault(key, []).append((name, args, kw))

rows = []
for key, items in groups.items():
    kind, images, heads, d, nq, nk, causal, dtype = key
    name, args, kw = items[0]
    run = lambda: _orig[name](*args, **kw)
    if kind == "bwd":
        # same operands, dQ launch only (delta is recomputed there, dS not exported)
        q, k, v, o, dO, lse, dq = args[:7]
        run_dq = lambda: _orig["attention_bwd_dq"](q, k, v, o, dO, lse, dq, None, **kw)
        us_all, us_dq = timed(run), timed(run_dq)
        parts = [("bwd_dq", us_dq), ("bwd_dkdv", us_all - us_dq)]
    else:
        parts = [("fwd" if kind.startswith("fwd") else "bwd_dq", timed(run))]
    ks = (d + 15) // 16
    for kernel, us in parts:
        ctas, mma, exps = counts(kernel, nq, nk, d, heads, images, causal, two_pass=kind == "fwd_2pass_P")
        n_mm = {"fwd": 2, "bwd_dq": 3, "bwd_dkdv": 4}[kernel]
        alg = 2 * n_mm * pairs(nq, nk, causal) * d * heads * images
        t_tensor = mma / PEAK_TFLOPS / 1e6
        t_exp = exps / (EXP2_PER_CLK_SM * n_sm * max_sm_mhz)
        floor = max(t_tensor, t_exp)
        rows.append(dict(kernel=kernel, path=kind, images=images, heads=heads, d=d, nq=nq, nk=nk, causal=causal,
                         dtype=dtype.replace("torch.", ""), count=len(items), us=round(us, 2),
                         total_us=round(us * len(items), 1), alg_gflop=round(alg / 1e9, 3),
                         mma_gflop=round(mma / 1e9, 3), exp2_m=round(exps / 1e6, 3),
                         floor_tensor_us=round(t_tensor, 2), floor_exp_us=round(t_exp, 2),
                         bound="tensor" if t_tensor >= t_exp else "exp", frac_of_floor=round(floor / us, 3),
                         mma_tflops=round(mma / us / 1e6, 1), ctas=ctas,
                         inst=("cb_attention_fwd_kernel<%d>" % ks) if kernel == "fwd" else
                         ("cb_attention_bwd_kernel<%d,%d>" % (ks, 0 if kernel == "bwd_dq" else 1))))
rows.sort(key=lambda r: -r["total_us"])
tot = sum(r["total_us"] for r in rows)
summary = dict(card=card, max_sm_mhz=max_sm_mhz, sms=n_sm, calls=len(rec), groups=len(groups),
               sum_isolated_ms=round(tot / 1000, 3),
               sum_floor_ms=round(sum(max(r["floor_tensor_us"], r["floor_exp_us"]) * r["count"] for r in rows) / 1000, 3),
               by_kernel_ms={k: round(sum(r["total_us"] for r in rows if r["kernel"] == k) / 1000, 3)
                             for k in ("fwd", "bwd_dq", "bwd_dkdv")})
os.makedirs(os.path.join(ROOT, "tools_out"), exist_ok=True)
out = os.path.join(ROOT, "tools_out", f"attn_floors{'_' + tag if tag else ''}.jsonl")
with open(out, "w") as f:
    f.write(json.dumps({"summary": summary}) + "\n")
    for r in rows:
        f.write(json.dumps(r) + "\n")
print(json.dumps({"summary": summary}))
for r in rows:
    print(json.dumps(r))
