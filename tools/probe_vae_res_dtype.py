"""Probe: VAE encoder with an fp32 vs fp16 residual stream -- latent parity against the reference fixture and time."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops, synth, workload
from celebbasis_b200.vae_engine import VAEEncoderEngine
from oracle import torch_ref
dev = torch.device("cuda:0")
gold = torch.load(os.path.join(ROOT, "tests", "golden", "step_full.pt"))
params = workload.model_params("full")
om = torch_ref.OracleModel(params, clip_layers=12)
sd = synth.synth_state_dict(om, seed=0)
del om
fs = params["first_stage_config"]["params"]
sub = {k[len("first_stage_model."):]: v for k, v in sd.items() if k.startswith("first_stage_model.")}
batch, draws = workload.synth_batch("full", B=1, seed=1234)
x = batch["image"].to(dev).permute(0, 3, 1, 2).contiguous()
for rt in (torch.float32, torch.float16):
    eng = VAEEncoderEngine(fs["ddconfig"], fs["embed_dim"], sub, dev, res_dtype=rt)
    for _ in range(2):
        mom = eng.encode_moments(x)
    z = ops.posterior_sample(mom, draws["posterior_eps"].to(dev).contiguous(), 0.18215)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.encode_moments(x)
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5): g.replay()
    e1.record(); torch.cuda.synchronize()
    rel = ((z.cpu() - gold["z"]).norm() / gold["z"].norm()).item()
    relm = ((mom.cpu() - gold["moments"]).norm() / gold["moments"].norm()).item()
    print(rt, "z rel", rel, "moments rel", relm, "ms", e0.elapsed_time(e1) / 5, flush=True)
