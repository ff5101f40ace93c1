"""The two samplers LatentDiffusion.sample_log can log with, at the SD-v1 size, alternating in one process: ancestral
DDPM sampling over all 1000 timesteps (ddim=False: LatentDiffusion.sample, one UNet call + one cb_p_sample launch per
step) and 50-step DDIM (ddim=True, eta 1: DDIMSampler.sample).  No guidance, as sample_log's first call; latents only
(the VAE decode is the same for both).  Synthetic weights and coefficients.

Prints one JSON line per arm (images/s, ms per step and launches per step; medians of `--reps` alternating rounds),
then one line with cb_p_sample's kernel time from a separate torch.profiler pass over `--profile-steps` DDPM steps.
Every line carries the GPU's name, power limit and max SM clock, read in the same call."""
import argparse, json, os, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F

ap = argparse.ArgumentParser()
ap.add_argument("--n-samples", type=int, default=8)
ap.add_argument("--ddim-steps", type=int, default=50)
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--profile-steps", type=int, default=100)
ap.add_argument("--kind", default="full")
args = ap.parse_args()

from celebbasis_b200 import lib, synth, workload
from ldm.models.diffusion.ddpm import LatentDiffusion

assert torch.cuda.is_available(), "bench_ddpm measures on the GPU"
dev = torch.device("cuda:0")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True).stdout.strip()
gpu = dict(zip(("name", "power_limit", "max_sm_clock"), [s.strip() for s in q.split(",")])) if q else \
    {"name": torch.cuda.get_device_name(0)}

params = workload.model_params(args.kind)
params["cond_stage_config"]["params"].update(device="cuda")
model = LatentDiffusion(**params)
sd = synth.synth_state_dict(model, seed=0)
model.load_state_dict(sd, strict=False)
del sd
model = model.to(dev).eval()
model.cond_stage_model.celeb_embeddings = synth.synth_celeb_basis(seed=0).to(dev)
g = torch.Generator().manual_seed(3)
model.embedding_manager.id_coefficients = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
B = args.n_samples
image_ori = {"faces": None, "ids": [[i % 10, i % 10] for i in range(B)], "num_ids": torch.ones(B, dtype=torch.long)}
with torch.no_grad():
    c = model.get_learned_conditioning(["a photo of sks person"] * B, image_ori=image_ori)


def run_ddpm(steps=None):
    with torch.no_grad():
        if steps is None:
            return model.sample_log(cond=c, batch_size=B, ddim=False, ddim_steps=None, eta=1.0)[0]
        return model.sample(c, batch_size=B, timesteps=steps)


def run_ddim():
    with torch.no_grad():
        return model.sample_log(cond=c, batch_size=B, ddim=True, ddim_steps=args.ddim_steps, eta=1.0)[0]


ARMS = {"ddpm": (run_ddpm, model.num_timesteps), "ddim": (run_ddim, args.ddim_steps)}
run_ddpm(4)                               # warm-up: engines, autotuned GEMM shapes
run_ddim()
torch.cuda.synchronize()

ms = {k: [] for k in ARMS}
launches = {}
for _ in range(args.reps):
    for name, (fn, _) in ARMS.items():
        torch.cuda.synchronize()
        n0 = lib.launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        x = fn()
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(x).all()
        ms[name].append(e0.elapsed_time(e1))
        launches[name] = lib.launch_count() - n0
cfg = {"n_samples": B, "latent": list(x.shape[1:]), "unet_batch": B, "reps": args.reps, "kind": args.kind,
       "data": "synthetic"}
for name, (_, steps) in ARMS.items():
    med = statistics.median(ms[name])
    print(json.dumps({"arm": name, "steps": steps, "images_per_s": B / (med / 1e3), "ms_per_step": med / steps,
                      "cb_launches_per_step": launches[name] / steps, "ms_per_batch_all": ms[name], "gpu": gpu,
                      "config": cfg}))

from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    run_ddpm(args.profile_steps)
    torch.cuda.synchronize()
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
ps = [e.device_time for e in ev if "p_sample_kernel" in e.name]
total = sum(e.device_time for e in ev)
print(json.dumps({"metric": "cb_p_sample kernel time per DDPM step (torch.profiler)", "unit": "us",
                  "value": statistics.median(ps), "launches": len(ps), "steps": args.profile_steps,
                  "share_of_gpu_time": sum(ps) / total, "gpu_kernel_us_per_step": total / args.profile_steps,
                  "gpu": gpu, "config": cfg}))
