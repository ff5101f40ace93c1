"""bench.py -- CelebBasis training steps/sec (SD-v1 UNet 512^2, bs=1/GPU) on N H100s  (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--dump-outputs DIR]   # our arm (N>1: launched by torchrun)
    python bench.py --impl reference --gpus N --steps K --warmup W      # the reference's CPU path (oracle port)

One step = SURVEY.md §8 rows a1-a31 for one sample per GPU: VAE encode, CosFace R100 on the 2 face crops, celeb-basis
MLP + inject, CLIP text fwd, UNet fwd, eps-MSE, full backward to the 1024x512 MLP, gradient all-reduce, AdamW.
Synthetic 512x512 inputs / 77-token prompt, deterministic synthetic SD-v1 / CLIP / CosFace weights (no network).

Output: ONE JSON line (rank 0).  `value` = whole-job steps/s with inputs resident in HBM (CUDA events, max over ranks);
`e2e` = the same step driven from pinned HOST buffers (H2D of image/faces/draws + D2H of the loss every step);
`roofline` = tensor-pipe fraction of the dominant kernel (cb_gemm_kernel: every conv / linear / attention GEMM),
measured live by replaying exactly the step's GEMM launches as their own CUDA graph under CUDA events;
`cpu_baseline` = the oracle port of the reference step on this box's host cores.
--dump-outputs DIR: after the timed steps, what the last timed step computed (loss, predicted noise, gradient of the
trainable MLP, its weights after AdamW) as DIR/<name>.npy in float32.  Inputs and weights are seeded, so two builds run
with the same arguments can be compared output for output.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "celeb-basis training steps/sec (SD-v1 UNet 512^2, bs=1/GPU)"
WORKLOAD = "configs[1]: single identity per GPU, 512x512, bs=1, SD-v1 UNet + CLIP text fwd/bwd + VAE encode + CosFace R100, AdamW on the 525,312 MLP weights"


def _peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            p = json.load(f)
        return p, "measured (MEASURED_PEAKS.json)"
    except Exception:
        # NVIDIA H100 SXM data sheet (700 W): HBM3 3.35 TB/s, dense BF16 989 TFLOP/s -- never reached, and less on a
        # power-limited card
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "H100 SXM data sheet (dense BF16)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    def __init__(self, gpu_index=0):
        self.rows, self.proc, self.idx = [], None, gpu_index

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "100",
                                          "-i", str(self.idx)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            parts = [p.strip() for p in r.split(",")]
            if len(parts) < 7:
                continue
            try:
                sm.append(float(parts[0]))
                mx = float(parts[1])
            except ValueError:
                continue
            for n, v in zip(names, parts[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


# ------------------------------------------------------------------------------------------------ reference / CPU arm
def host_cpu_limits():
    """Cores this process may actually use: scheduler affinity, capped by the cgroup CPU quota (v2 cpu.max, v1
    cfs_quota_us).  os.cpu_count() reports the machine (128 on the GPU boxes) even when the container gets a slice."""
    aff = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    quota = None
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            quota = float(q) / float(per)
    except Exception:
        try:
            q = float(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / per
        except Exception:
            pass
    limit = aff if quota is None else max(1, min(aff, int(quota + 0.5)))
    return {"cpu_count": os.cpu_count(), "affinity": aff, "cgroup_quota": quota, "limit": limit}


def pick_cpu_threads():
    """Thread count for the CPU arm: the quota/affinity limit, checked by a ~3 s calibration (a 3x3 fp32 convolution of
    the VAE's 256^2 level, the dominant CPU op of the step) over {limit, limit/2, limit/4, 32, 16, 8} -- a pool wider
    than the cores the container really gets runs many times slower (round 1: 327 s/step with 128 threads)."""
    import torch
    info = host_cpu_limits()
    lim = info["limit"]
    cands = sorted({c for c in (lim, lim // 2, lim // 4, 32, 16, 8) if 1 <= c <= lim} | {min(lim, 8)})
    if len(cands) == 1:
        info["threads"], info["calibration_ms"] = cands[0], {}
        torch.set_num_threads(cands[0])
        return info
    x = torch.randn(1, 128, 256, 256)
    w = torch.randn(128, 128, 3, 3)
    res = {}
    for c in cands:
        torch.set_num_threads(c)
        with torch.no_grad():
            torch.nn.functional.conv2d(x, w, padding=1)
            t0 = time.perf_counter()
            for _ in range(3):
                torch.nn.functional.conv2d(x, w, padding=1)
            res[c] = (time.perf_counter() - t0) / 3 * 1e3
    best = min(res, key=res.get)
    info["threads"], info["calibration_ms"] = best, {str(k): round(v, 1) for k, v in res.items()}
    torch.set_num_threads(best)
    return info


def cpu_reference_steps(n_timed, budget_s, min_steps=3):
    """The reference step (oracle port of LatentDiffusion.shared_step + backward + AdamW, fp32) on the host cores.
    Always runs >= min_steps steps (the first is cold: oneDNN primitive creation, page faults on 4.4 GB of weights) unless
    a single step alone exceeds the budget; returns per-step seconds, losses and the host description."""
    import torch
    from celebbasis_b200 import synth, workload
    from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
    from oracle import torch_ref
    info = pick_cpu_threads()
    min_steps = int(os.environ.get("CB_BENCH_CPU_MIN_STEPS", min_steps))      # test knob (tests/test_host_logic.py)
    params = workload.model_params("full")
    om = torch_ref.OracleModel(params, clip_layers=12)
    om.load_state_dict(synth.synth_state_dict(om, seed=0))
    om.eval()
    W, b = om.trainable()
    W.requires_grad_(True)
    b.requires_grad_(True)
    opt = torch.optim.AdamW([W, b], lr=5e-3)
    basis = synth.synth_celeb_basis(seed=0)
    tok = SyntheticCLIPTokenizer()
    times, losses = [], []
    t_start = time.perf_counter()
    want = max(min_steps, n_timed + 1)
    for i in range(want):
        batch, draws = workload.synth_batch("full", B=1, seed=1234, step=i)
        t0 = time.perf_counter()
        out = om.step(batch, draws, tok(batch["caption"])["input_ids"], basis, tok.word_id("sks"))
        opt.zero_grad(set_to_none=True)
        out["loss"].backward()
        opt.step()
        times.append(time.perf_counter() - t0)
        losses.append(float(out["loss"]))
        elapsed = time.perf_counter() - t_start
        if len(times) >= min_steps and elapsed + times[-1] > budget_s:
            break
        if elapsed + times[-1] > 2.0 * budget_s:      # hard stop: never more than twice the budget
            break
    return times, losses, info


def summarize_cpu(times):
    """Drop the cold first step whenever more than one was run; median of the rest."""
    timed = times[1:] if len(times) > 1 else times
    return statistics.median(timed), len(timed)


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    times, losses, info = cpu_reference_steps(args.steps, budget_s=200.0)
    sec, n_timed = summarize_cpu(times)
    val = 1.0 / sec
    sample = (f"{len(times)} full bs=1 steps (fwd+bwd+AdamW, fp32, oracle/torch_ref.py) on {info['threads']} threads "
              f"(affinity {info['affinity']}, cgroup quota {info['cgroup_quota']}, os.cpu_count {info['cpu_count']}); "
              f"first step dropped as cold, median of the other {n_timed}; per-step s: {[round(t, 1) for t in times]}")
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": val, "unit": "steps/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": bench_config(args.gpus),
        "cpu_baseline": {"value": val, "unit": "steps/s", "cores": info["threads"], "kind": "port", "sample": sample,
                         "thread_calibration_ms": info["calibration_ms"], "loss_first": losses[0]},
        "e2e": {"value": val, "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


# ------------------------------------------------------------------------------------------------ our arm
def dump_outputs(out_dir, arrays):
    """Each tensor as out_dir/<name>.npy in float32 (the step's outputs are a few MB in all, far below 64 MB)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), t.detach().float().cpu().numpy().astype(np.float32))


def bench_config(world):
    """The workload description both arms print (identical dicts => the driver's same_config check holds)."""
    return {"workload": WORKLOAD, "per_gpu_batch": 1, "parallelism": f"dp{world}",
            "l2": "inputs larger than L2: 2.1 GB of 16-bit weights + ~4 GB of activations are streamed every step (L2 = 50 MB)"}


def _file_sha1(path):
    import hashlib
    with open(path, "rb") as f:
        return hashlib.sha1(f.read()).hexdigest()


def _ncu_traffic():
    """DRAM bytes per cb_gemm launch (dram__bytes_read.sum + dram__bytes_write.sum averaged over the step's launches) from
    the newest committed `ncu` pass under profiles/ -- reported only if that pass was taken on THIS version of the kernel
    (the pass records the sha1 of cb_gemm.cu); otherwise null, never a stale constant."""
    import glob
    cur = _file_sha1(os.path.join(ROOT, "celebbasis_b200", "csrc", "cb_gemm.cu"))
    for f in sorted(glob.glob(os.path.join(ROOT, "profiles", "r*_gemm_traffic*.json")), reverse=True):
        try:
            j = json.load(open(f))
        except Exception:
            continue
        if j.get("kernel_source_sha1") == cur:
            return j.get("traffic_bytes_per_launch"), os.path.basename(f)
    return None, None


def run_ours(args):
    import torch
    import torch.distributed as dist
    from celebbasis_b200 import dist as cbd
    from celebbasis_b200 import lib, ops, synth, workload
    from celebbasis_b200.compat import pytorch_lightning as pl
    from ldm.models.diffusion.ddpm import LatentDiffusion

    world, rank, local = cbd.init()
    json_out, sys.stdout = sys.stdout, sys.stderr       # stdout carries exactly one JSON line; library chatter -> stderr
    torch.manual_seed(1000 + rank)                      # t / noise / posterior draws: identical inputs from run to run
    assert torch.cuda.is_available(), "bench.py needs a GPU (no CPU fallback in the product path)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    assert lib.load().cb_device_ok() == 1, "not an sm_90 (H100) device"
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    B = 1

    # ---- the model through the reference-facing API: ldm.models.diffusion.ddpm.LatentDiffusion(**aigc_id.yaml params) ----
    params = workload.model_params("full")
    params["cond_stage_config"]["params"].update(device="cuda")
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model = model.to(dev)
    model.cond_stage_model.celeb_embeddings = synth.synth_celeb_basis(seed=0).to(dev)
    model.learning_rate = cbd.scaled_lr(5e-3, B) if world > 1 else 5e-3      # main_id_embed.py:778-779
    model.train()

    # ---- host-side batches (pinned, as a DataLoader with pin_memory yields them): face_id.py:598-644 layout ------------
    n_host = 4
    host = []
    for i in range(n_host):
        batch, _ = workload.synth_batch("full", B=B, seed=1234 + 101 * rank, step=i)
        batch["image"] = batch["image"].pin_memory()
        batch["image_ori"]["faces"] = batch["image_ori"]["faces"].pin_memory()
        batch["image_ori"]["ids"] = torch.full((B, 2), rank % 10, dtype=torch.long).pin_memory()
        host.append(batch)
    h2d_bytes = sum(t.numel() * t.element_size() for t in (host[0]["image"], host[0]["image_ori"]["faces"],
                                                           host[0]["image_ori"]["ids"], host[0]["image_ori"]["num_ids"]))
    h2d_bytes += 4 * 64 * 64 * 4 + 77 * 8 + 77 * 4        # posterior eps (CPU generator, as the reference), token ids, row map

    # ---- first API step builds the fused engine: eager warm-up (GEMM autotune), then the three step graphs -------------
    opt = model.configure_optimizers()
    dev_batch = {"image": host[0]["image"].to(dev), "caption": host[0]["caption"],
                 "image_ori": {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in host[0]["image_ori"].items()}}
    loss, _ = model.shared_step(dev_batch)
    loss.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    G = model._fused
    assert G is not None, "the fused CUDA-graph step did not engage"
    eng = G.eng
    launches_per_step = G.launches["pipe"] + 1              # chain + next batch's front end + AdamW

    # ---- leg 1 (`value`): inputs resident in HBM; one step = one replay of G_pipe (this batch's trainable chain || the
    #      next batch's frozen front end) + gradient all-reduce + AdamW ---------------------------------------------------
    G.load_next(dev_batch["image"], dev_batch["image_ori"]["faces"], torch.randn(list(G.peps_n.shape)))
    G.prefetch()

    def one_step():
        G.step(lookahead=True)
        cbd.allreduce_mean_(eng.grad)     # the single per-step collective (no-op at N=1)
        eng.optimizer_step()

    def timed(fn, n):
        cbd.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        cbd.barrier()
        return float(ms.item())

    warm = max(args.warmup, 3)
    for _ in range(warm):
        one_step()
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()
    ms_per_step = timed(one_step, args.steps) / args.steps
    value = world * B * 1000.0 / ms_per_step
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"loss": G.loss, "eps": eng.last["eps"], "grad": eng.grad, "mlp_weight": eng.W,
                                         "mlp_bias": eng.b})
    # un-pipelined reference point: front end, then chain, back to back
    def serial_step():
        G.prefetch()
        G.step(lookahead=False)
        cbd.allreduce_mean_(eng.grad)
        eng.optimizer_step()
    serial_step()
    ms_serial = timed(serial_step, max(3, args.steps // 2)) / max(3, args.steps // 2)

    # ---- leg 2 (`e2e`): the call a user of the reference makes -- Trainer.fit(model, data) (main_id_embed.py:748,812)
    #      over HOST batches: per step H2D of the batch, tokenisation + row map on the host, t / noise draws, the fused
    #      shared_step, loss.backward(), gradient all-reduce, FusedAdamW.step(), and a D2H read of the loss ------------------
    class HostData:
        def __init__(self, n):
            self.n = n

        def __iter__(self):
            for i in range(self.n):
                yield host[i % n_host]

    class Timer(pl.Callback):
        def __init__(self, w, k):
            self.w, self.k, self.ms, self.last_loss = w, k, None, None
            self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def on_train_batch_start(self, trainer, module, batch, batch_idx, dl=0):
            if batch_idx == self.w:
                torch.cuda.synchronize()
                cbd.barrier()
                self.e0.record()

        def on_train_batch_end(self, trainer, module, outputs, batch, batch_idx, dl=0):
            self.last_loss = float(outputs["loss"].item())       # D2H read of the step's loss, every step
            if batch_idx == self.w + self.k - 1:
                self.e1.record()
                torch.cuda.synchronize()
                self.ms = self.e0.elapsed_time(self.e1)

    timer = Timer(warm, args.steps)
    trainer = pl.Trainer(gpus=f"{local},", max_steps=warm + args.steps, callbacks=[timer])
    trainer.fit(model, train_dataloaders=HostData(warm + args.steps))
    ms_e2e_t = torch.tensor([timer.ms], device=dev)
    if world > 1:
        dist.all_reduce(ms_e2e_t, op=dist.ReduceOp.MAX)
    ms_e2e = float(ms_e2e_t.item()) / args.steps
    clk = clocks.stop() if rank == 0 else None
    final_loss = timer.last_loss

    # ---- roofline of the dominant kernel: replay exactly one step's GEMM launches as their own graph ------------------
    roof = None
    if rank == 0:
        import ctypes
        from celebbasis_b200.lib import GemmDesc
        L = lib.load()
        gemm_record = G.gemm_record      # one step's GEMM launches as captured (buffers live in the graphs' memory pool)
        descs = [GemmDesc.from_buffer_copy(b) for b, _ in gemm_record]
        flops = sum(f for _, f in gemm_record)
        sp = ctypes.c_void_p

        def launch_all():
            s = sp(torch.cuda.current_stream().cuda_stream)
            for d in descs:
                L.cb_gemm(ctypes.byref(d), s)
        gg = torch.cuda.CUDAGraph()
        launch_all()
        torch.cuda.synchronize()
        with torch.cuda.graph(gg):
            launch_all()
        for _ in range(3):
            gg.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        e0.record()
        for _ in range(reps):
            gg.replay()
        e1.record()
        torch.cuda.synchronize()
        gemm_ms = e0.elapsed_time(e1) / reps
        peaks, src = _peaks()
        peak = float(peaks.get("bf16_tflops", 989.0))
        ach = flops / (gemm_ms * 1e-3) / 1e12
        traffic, traffic_src = _ncu_traffic()
        roof = {"bound": "tensor", "kernel": "cb_gemm_kernel (wgmma GEMM / implicit-GEMM conv, all instantiations)",
                "achieved": ach, "peak": peak, "unit": "TFLOP/s", "frac": ach / peak, "traffic": traffic,
                "traffic_source": traffic_src,
                "peak_source": src + " bf16_tflops",
                "launches_per_step": len(descs), "avg_launch_us": gemm_ms * 1e3 / len(descs),
                "algorithmic_gflop_per_step": flops / 1e9, "gemm_ms_per_step": gemm_ms,
                "gemm_share_of_serial_step": gemm_ms / ms_serial,
                "whole_step_tflops": 2861.0 / ms_per_step, "whole_step_frac": 2861.0 / ms_per_step / peak}

    # ---- CPU baseline (rank 0, N=1 only): the oracle port on this box's host cores --------------------------------
    cpu = None
    if rank == 0 and world == 1 and not args.skip_cpu_baseline:
        del model, G, eng, trainer, opt
        torch.cuda.empty_cache()
        times, _, info = cpu_reference_steps(2, budget_s=90.0)
        sec, n_timed = summarize_cpu(times)
        cpu = {"value": 1.0 / sec, "unit": "steps/s", "cores": info["threads"], "kind": "port",
               "sample": f"{len(times)} full bs=1 steps (fwd+bwd+AdamW, fp32, oracle/torch_ref.py) on {info['threads']} "
                         f"threads (affinity {info['affinity']}, cgroup quota {info['cgroup_quota']}); first dropped as "
                         f"cold, median of the other {n_timed}; per-step s: {[round(t, 1) for t in times]}"}

    if rank == 0:
        out = {
            "metric": METRIC, "value": value, "unit": "steps/s", "n_gpus": world, "steps": args.steps,
            "warmup": warm, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f16 operands / f32 accumulate+residual (reference: f32 with TF32 convs)",
            "data": "synthetic",
            "config": bench_config(world),
            "e2e": {"value": world * B * 1000.0 / ms_e2e, "unit": "steps/s", "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 4,
                    "api": "celebbasis_b200.compat pytorch_lightning.Trainer.fit(ldm LatentDiffusion, host batches): "
                           "training_step -> loss.backward() -> grad all-reduce -> FusedAdamW.step() -> loss.item()"},
            "gpu_launches": int(launches_per_step * args.steps),
            "gpu_launches_per_step": int(launches_per_step),
            "pipeline": {"ms_per_step_pipelined": ms_per_step, "ms_per_step_serial": ms_serial,
                         "note": "pipelined: the frozen no-grad front end (VAE encode, CosFace R100) of batch i+1 runs "
                                 "concurrently with batch i's trainable chain; every step does all of its work once"},
            "notes": {"cuda_graph": True, "final_loss": final_loss, "v100_published_it_s": 2.75},
            "clocks": clk, "roofline": roof, "cpu_baseline": cpu,
        }
        print(json.dumps(out), file=json_out, flush=True)
    sys.stdout = json_out
    if world > 1:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------ config 4: txt2img
T2I_METRIC = "DDIM txt2img images/sec (scripts/stable_txt2img.py semantics: 50 steps, eta 0, CFG 10, 512x512, 8 images/GPU)"
T2I_WORKLOAD = ("configs[3]: DDIM txt2img, 50 steps, 512x512, n_samples 8 per GPU (UNet batch 16 under classifier-free "
                "guidance), fp16 operands, + VAE decode; replicas across GPUs (no collective)")


def t2i_config(world):
    return {"workload": T2I_WORKLOAD, "per_gpu_batch": 8, "parallelism": f"replicas x{world}",
            "l2": "inputs larger than L2: 1.7 GB of UNet weights + ~6 GB of batch-16 activations per UNet call (L2 = 50 MB)"}


def run_txt2img(args):
    """BASELINE config 4 through the reference-facing API: get_learned_conditioning -> DDIMSampler.sample ->
    decode_first_stage (scripts/stable_txt2img.py:320-347).  `value`: conditioning + 50 DDIM steps + decode with the
    prompts' conditioning resident; `e2e`: the whole script body per batch, host prompts in, images copied to the host."""
    import torch
    import torch.distributed as dist
    import torch.nn.functional as F
    from celebbasis_b200 import dist as cbd
    from celebbasis_b200 import lib, ops, synth, workload
    from ldm.models.diffusion.ddim import DDIMSampler
    from ldm.models.diffusion.ddpm import LatentDiffusion
    world, rank, local = cbd.init()
    json_out, sys.stdout = sys.stdout, sys.stderr
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    assert lib.load().cb_device_ok() == 1 and world == args.gpus
    params = workload.model_params("full")
    params["cond_stage_config"]["params"].update(device="cuda")
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model = model.to(dev).eval()
    model.cond_stage_model.celeb_embeddings = synth.synth_celeb_basis(seed=0).to(dev)
    g = torch.Generator().manual_seed(3 + rank)
    model.embedding_manager.id_coefficients = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    B, steps, scale = 8, 50, 10.0
    prompts = ["a photo of sks person"] * B
    image_ori = {"faces": None, "ids": [[i % 10, i % 10] for i in range(B)], "num_ids": torch.ones(B, dtype=torch.long)}
    sampler = DDIMSampler(model)
    host_img = torch.empty(B, 3, 512, 512, dtype=torch.float32).pin_memory()

    def conditioning():
        with torch.no_grad():
            return model.get_learned_conditioning([""] * B), model.get_learned_conditioning(prompts, image_ori=image_ori)

    def sample(uc, c, n_steps):
        with torch.no_grad():
            x_T = torch.randn(B, 4, 64, 64, device=dev)
            z, _ = sampler.sample(S=n_steps, conditioning=c, batch_size=B, shape=[4, 64, 64], verbose=False,
                                  unconditional_guidance_scale=scale, unconditional_conditioning=uc, eta=0.0, x_T=x_T)
            return model.decode_first_stage(z)

    from ldm.modules.diffusionmodules.openaimodel import UNetModel
    UNetModel.CAPTURE_GEMM_SINK = gemm_record = []   # the UNet's batch-16 GEMMs, recorded while its graph is captured
    uc, c = conditioning()
    sample(uc, c, 2)                          # builds engines, autotunes, captures the UNet graph
    UNetModel.CAPTURE_GEMM_SINK = None
    torch.cuda.synchronize()

    def timed(fn, n):
        cbd.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        cbd.barrier()
        return float(ms.item())

    n_batches = max(1, args.steps // 10)      # a "step" of this workload is one batch of 8 images (50 DDIM steps)
    unet = model.model.diffusion_model
    n0 = lib.launch_count() + unet.__dict__.get("_replayed_launches", 0)
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()
    ms_batch = timed(lambda: sample(uc, c, steps), n_batches) / n_batches
    launches = (lib.launch_count() + unet.__dict__.get("_replayed_launches", 0) - n0) // n_batches   # incl. graph replays

    def e2e_batch():
        u, cc = conditioning()
        img = sample(u, cc, steps)
        host_img.copy_(torch.clamp((img + 1.0) / 2.0, 0.0, 1.0), non_blocking=True)      # stable_txt2img.py:348-349
        torch.cuda.current_stream().synchronize()
    ms_e2e = timed(e2e_batch, n_batches) / n_batches
    clk = clocks.stop() if rank == 0 else None
    roof = None
    if rank == 0 and gemm_record:
        import ctypes
        from celebbasis_b200.lib import GemmDesc
        L = lib.load()
        descs = [GemmDesc.from_buffer_copy(b) for b, _ in gemm_record]
        flops = sum(f for _, f in gemm_record)
        gg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gg):
            s_ = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            for d in descs:
                L.cb_gemm(ctypes.byref(d), s_)
        for _ in range(2):
            gg.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            gg.replay()
        e1.record()
        torch.cuda.synchronize()
        gemm_ms = e0.elapsed_time(e1) / 5
        peaks, src = _peaks()
        peak = float(peaks.get("bf16_tflops", 989.0))
        ach = flops / (gemm_ms * 1e-3) / 1e12
        roof = {"bound": "tensor", "kernel": "cb_gemm_kernel launches of ONE UNet forward at batch 16 (one DDIM step)",
                "achieved": ach, "peak": peak, "unit": "TFLOP/s", "frac": ach / peak, "traffic": None,
                "peak_source": src + " bf16_tflops", "launches": len(descs), "gemm_ms_per_unet_call": gemm_ms,
                "algorithmic_gflop_per_unet_call": flops / 1e9,
                "whole_job_tflops_per_gpu": 82.9 * B / (ms_batch * 1e-3),
                "whole_job_frac": 82.9 * B / (ms_batch * 1e-3) / peak}
    if rank == 0:
        out = {"metric": T2I_METRIC, "value": world * B * 1000.0 / ms_batch, "unit": "images/s", "n_gpus": world,
               "steps": n_batches, "warmup": 1, "ms_per_step": ms_batch, "higher_is_better": True, "scaling": "weak",
               "vs_baseline": None, "dtype": "f16 operands / f32 accumulate (reference: fp16 autocast)", "data": "synthetic",
               "config": t2i_config(world),
               "e2e": {"value": world * B * 1000.0 / ms_e2e, "unit": "images/s", "ms_per_step": ms_e2e,
                       "h2d_bytes_per_step": 2 * B * 77 * 8, "d2h_bytes_per_step": B * 3 * 512 * 512 * 4,
                       "api": "ldm LatentDiffusion.get_learned_conditioning + DDIMSampler.sample + decode_first_stage"},
               "gpu_launches": int(launches * n_batches), "gpu_launches_per_step": int(launches),
               "notes": {"v100_published_img_s": 0.243, "algorithmic_tflop_per_image": 82.9},
               "clocks": clk, "roofline": roof, "cpu_baseline": None}
        print(json.dumps(out), file=json_out, flush=True)
    sys.stdout = json_out
    if world > 1:
        dist.destroy_process_group()


def run_txt2img_reference(args):
    """The reference's CPU path for config 4 (oracle port): a bounded sample -- 2 CFG DDIM steps for ONE image (UNet batch
    2) + one VAE decode -- extrapolated to 50 steps: images/s = 1 / (50 * t_step + t_decode)."""
    if int(os.environ.get("RANK", "0")) != 0:
        return
    import torch
    from celebbasis_b200 import synth, workload
    from oracle import torch_ref
    info = pick_cpu_threads()
    params = workload.model_params("full")
    om = torch_ref.OracleModel(params, clip_layers=12)
    om.load_state_dict(synth.synth_state_dict(om, seed=0))
    om.eval()
    fs = params["first_stage_config"]["params"]
    dec = torch_ref.AutoencoderKLDecode(fs["ddconfig"], fs["embed_dim"]).eval()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 4, 64, 64, generator=g)
    ctx = torch.randn(1, 77, 768, generator=g)
    with torch.no_grad():
        t0 = time.perf_counter()
        x1 = torch_ref.ddim_sample(om.model.diffusion_model, om.sched, ctx, ctx * 0.5, x, 2, 10.0)
        t_step = (time.perf_counter() - t0) / 2
        t0 = time.perf_counter()
        dec(x1 / 0.18215)
        t_dec = time.perf_counter() - t0
    val = 1.0 / (50 * t_step + t_dec)
    sample = (f"2 CFG DDIM steps (UNet batch 2) + 1 VAE decode for one 512x512 image on {info['threads']} threads, fp32, "
              f"extrapolated to 50 steps: t_step {t_step:.2f} s, t_decode {t_dec:.2f} s")
    print(json.dumps({"impl": "reference", "metric": T2I_METRIC, "value": val, "unit": "images/s", "n_gpus": args.gpus,
                      "steps": args.steps, "warmup": args.warmup, "ms_per_step": 8e3 / val, "higher_is_better": True,
                      "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                      "config": t2i_config(args.gpus),
                      "cpu_baseline": {"value": val, "unit": "images/s", "cores": info["threads"], "kind": "port", "sample": sample},
                      "e2e": {"value": val, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--skip-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed as DIR/<name>.npy (float32)")
    ap.add_argument("--workload", default="train", choices=["train", "txt2img"],
                    help="train = BASELINE.json metric (configs[1]); txt2img = configs[3] (images/s)")
    args = ap.parse_args()
    if args.workload == "txt2img":
        (run_txt2img_reference if args.impl == "reference" else run_txt2img)(args)
    elif args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
