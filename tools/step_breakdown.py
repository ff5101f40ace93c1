"""Device time of the step's phases, each replayed alone as a CUDA graph, on the streams and workspace lanes of the
benchmark's step: front end (stage_prefetch: VAE encode || face net) | chain (stage_main: celeb-basis MLP -> CLIP text
|| UNet prefix -> UNet -> loss -> UNet / CLIP / celeb-basis backward -> EMA) | UNet fwd | UNet fwd + bwd | AdamW."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from celebbasis_b200.train_step import CelebBasisStep
from oracle import torch_ref

dev = torch.device("cuda:0")
params = workload.model_params("full")
om = torch_ref.OracleModel(params, clip_layers=12)
sd = synth.synth_state_dict(om, seed=0)
del om
eng = CelebBasisStep(params, sd, synth.synth_celeb_basis(seed=0), dev, tokenizer=SyntheticCLIPTokenizer())
del sd
batch, draws = workload.synth_batch("full", B=1, seed=1234)
image, faces = batch["image"].to(dev), batch["image_ori"]["faces"].to(dev)
t, noise, peps = draws["t"].to(dev), draws["noise"].to(dev), draws["posterior_eps"].to(dev)
ids, map_np, _ = eng.prepare(batch["caption"])
ids_dev, map_dev = ids.to(dev), torch.from_numpy(map_np).to(dev)
ids_person = batch["image_ori"]["ids"].to(dev)
for _ in range(2):
    z, v = eng.stage_prefetch(image, faces, ids_person.shape[1], peps)
    eng.stage_main(z, v, ids_person, ids_dev, map_dev, t, noise)
    eng.optimizer_step()
torch.cuda.synchronize()
st = {}

def timeit(name, fn, n=3):
    fn(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        g.replay()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(json.dumps({"phase": name, "ms": round(ms, 3)}), flush=True)
    return g

def front_end():
    st["z"], st["v"] = eng.stage_prefetch(image, faces, ids_person.shape[1], peps)

def chain():
    eng.stage_main(st["z"], st["v"], ids_person, ids_dev, map_dev, t, noise)
    st["xn"], st["ctx"] = eng.last["x_noisy"], eng.last["context"]

def unet_fwd():
    st["eps"] = eng.unet.forward(st["xn"], t, st["ctx"], need_grad=True)
    st["loss"], st["d_eps"] = ops.mse_fwd_bwd(st["eps"], noise.contiguous(), 1.0, want_grad=True)

keep = []
keep.append(timeit("front_end", front_end))
keep.append(timeit("chain", chain))
# forward/backward pairs: the tape is consumed by backward, so capture fwd+bwd together and subtract
keep.append(timeit("unet_fwd+loss", unet_fwd))
def unet_fwd_bwd():
    unet_fwd()
    eng.unet.backward(st["d_eps"])
keep.append(timeit("unet_fwd+loss+unet_bwd", unet_fwd_bwd))
keep.append(timeit("adamw", eng.optimizer_step))
