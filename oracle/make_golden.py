"""Generate tests/golden/*.pt by running the UNMODIFIED reference (through oracle/ref_shim.py) on CPU.

    python oracle/make_golden.py tiny        # seconds
    python oracle/make_golden.py full        # ~1-2 min, needs ~12 GB host RAM
    python oracle/make_golden.py infer       # DDIM txt2img + VAE decode on the tiny configuration

Fixtures hold the inputs' seeds (the inputs themselves are re-derivable from celebbasis_b200.workload +
celebbasis_b200.synth) and the reference's outputs: latent z, context, eps prediction, loss, and the gradient
of the two trainable tensors (full tensor for 'tiny'; norm + a fixed strided sample for 'full').
Also the integer known-answer of ldm/modules/id_embedding/helpers.py:44-54.
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

from celebbasis_b200 import synth, workload
from oracle import ref_shim

GOLD = os.path.join(ROOT, "tests", "golden")


def run(kind):
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    basis = synth.synth_celeb_basis(seed=0)
    t0 = time.time()
    model = ref_shim.build_reference(workload.model_params(kind), seed=0, clip_layers=workload.clip_layers(kind),
                                     celeb_basis=basis)
    print(f"[{kind}] reference built in {time.time() - t0:.1f}s")
    batch, draws = workload.synth_batch(kind, B=1, seed=1234)
    cap = {}
    # capture intermediate tensors without touching the arithmetic
    orig_apply = model.apply_model

    def apply_model(x_noisy, t, cond, *a, **k):
        out = orig_apply(x_noisy, t, cond, *a, **k)
        cap["x_noisy"], cap["context"], cap["eps"] = x_noisy.detach().clone(), cond.detach().clone(), out.detach().clone()
        return out
    model.apply_model = apply_model
    orig_fse = model.get_first_stage_encoding

    def fse(post):
        z = orig_fse(post)
        cap["z"] = z.detach().clone()
        cap["moments"] = post.parameters.detach().clone()
        return z
    model.get_first_stage_encoding = fse
    mlp = model.embedding_manager.meta_id_net
    orig_celebs = mlp._celebs_forward

    def celebs_forward(img, id_idx, celebs_embeds):
        z, cls, x = orig_celebs(img, id_idx, celebs_embeds)
        cap["celeb_z"], cap["celeb_coef"] = z.detach().clone(), x.detach().clone()
        return z, cls, x
    mlp._celebs_forward = celebs_forward
    orig_idm = mlp.id_model.forward

    def idm(x):
        y = orig_idm(x)
        cap["face_in"], cap["face_feat"] = x.detach().clone(), y.detach().clone()
        return y
    mlp.id_model.forward = idm

    em0 = model.embedding_manager
    ema_init = {"coef": em0.id_coefficients[0].detach().clone(), "emb": em0.id_embeddings[0].detach().clone()}
    t0 = time.time()
    with ref_shim.replay_randomness(draws["t"], draws["noise"], draws["posterior_eps"]):
        loss, loss_dict = model.shared_step(batch)
    print(f"[{kind}] forward {time.time() - t0:.1f}s loss={loss.item():.6f}")
    t0 = time.time()
    loss.backward()
    print(f"[{kind}] backward {time.time() - t0:.1f}s")
    W = mlp.stylegan_mlp.net[0].weight
    b = mlp.stylegan_mlp.net[0].bias
    graded = [n for n, p in model.named_parameters() if p.grad is not None]
    out = {
        "kind": kind, "loss": loss.detach().clone(), "z": cap["z"], "moments": cap["moments"],
        "context": cap["context"], "eps": cap["eps"], "x_noisy": cap["x_noisy"], "celeb_z": cap["celeb_z"],
        "celeb_coef": cap["celeb_coef"], "face_feat": cap["face_feat"],
        "graded": graded, "gW_norm": W.grad.norm().clone(), "gb": b.grad.detach().clone(),
        "ema_coef_id0": model.embedding_manager.id_coefficients[0].detach().clone(),
        "ema_emb_id0": model.embedding_manager.id_embeddings[0].detach().clone(),
        "ema_coef_id0_init": ema_init["coef"], "ema_emb_id0_init": ema_init["emb"],
        "momentum": float(model.embedding_manager.momentum),
    }
    if kind == "tiny":
        out["gW_rows8"] = W.grad.detach()[::8].clone()       # every 8th output row: the file stays under 1 MB
        out["face_in"] = cap["face_in"]
    else:
        out["gW_sample"] = W.grad.detach().flatten()[::131].clone()
    os.makedirs(GOLD, exist_ok=True)
    torch.save(out, os.path.join(GOLD, f"step_{kind}.pt"))
    print(f"[{kind}] graded params: {graded}; |gW|={W.grad.norm().item():.6e}")


def run_infer(kind="tiny", steps=4, scale=5.0):
    """scripts/stable_txt2img.py semantics on the UNMODIFIED reference (CPU): eval-mode conditioning from stored identity
    coefficients (embedding_manager.py eval branch), DDIMSampler.sample with classifier-free guidance, eta = 0
    (ddim.py:57-204), decode_first_stage (ddpm.py:761-819).  Pins oracle/torch_ref.py's ddim_sample / AutoencoderKLDecode /
    eval-branch inject."""
    import torch.nn.functional as F
    torch.manual_seed(0)
    basis = synth.synth_celeb_basis(seed=0)
    model = ref_shim.build_reference(workload.model_params(kind), seed=0, clip_layers=workload.clip_layers(kind),
                                     celeb_basis=basis)
    model.eval()
    from ldm.models.diffusion.ddim import DDIMSampler

    def register_buffer(self, name, attr):            # ddim.py:19-23 hard-codes .to("cuda"); same values on the CPU
        setattr(self, name, attr)
    DDIMSampler.register_buffer = register_buffer
    g = torch.Generator().manual_seed(3)
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    model.embedding_manager.id_coefficients = [c.clone() for c in coefs]
    prompts = ["a photo of sks person"]
    image_ori = {"faces": None, "ids": torch.tensor([[3, 3]]), "num_ids": torch.ones(1, dtype=torch.long)}
    hw = workload.model_params(kind)["image_size"]
    with torch.no_grad():
        uc = model.get_learned_conditioning([""])
        c = model.get_learned_conditioning(prompts, image_ori=image_ori)
        x_T = torch.randn(1, 4, hw, hw, generator=g)
        sampler = DDIMSampler(model)
        samples, _ = sampler.sample(S=steps, conditioning=c, batch_size=1, shape=[4, hw, hw], verbose=False,
                                    unconditional_guidance_scale=scale, unconditional_conditioning=uc, eta=0.0, x_T=x_T)
        img = model.decode_first_stage(samples)
        # two / three persons in one prompt (embedding_manager.py:323-345,362-392): conditioning only
        multi = []
        for prompt, pid in (("a photo of sks person and ks person", [3, 5]),
                            ("sks person , ks person and ata person", [1, 2, 7])):
            io = {"faces": None, "ids": torch.tensor([pid]), "num_ids": torch.tensor([len(pid)])}
            multi.append({"prompt": prompt, "ids": pid, "c": model.get_learned_conditioning([prompt], image_ori=io).clone()})
    # a32: the embedding checkpoint the reference writes every 200 steps / reads back in stable_txt2img.py:230
    # (embedding_manager.py:396-426): written by the reference's own save(), fp32 and fp16 variants
    import tempfile
    em = model.embedding_manager
    with tempfile.TemporaryDirectory() as td:
        em.save(os.path.join(td, "e32.pt"))
        ck32 = torch.load(os.path.join(td, "e32.pt"))
        em.save_fp16 = True
        em.save(os.path.join(td, "e16.pt"))
        ck16 = torch.load(os.path.join(td, "e16.pt"))
        em.save_fp16 = False
    torch.save({"fp32": ck32, "fp16": ck16, "coef_seed": 3}, os.path.join(GOLD, "embeddings_ref.pt"))
    out = {"kind": kind, "multi": multi, "steps": steps, "scale": scale, "coef_seed": 3, "prompts": prompts, "person_id": 3,
           "uc": uc.clone(), "c": c.clone(), "x_T": x_T.clone(), "samples": samples.clone(), "img": img.clone(),
           "ddim_timesteps": torch.as_tensor(np.asarray(sampler.ddim_timesteps).copy())}
    os.makedirs(GOLD, exist_ok=True)
    # non-zip serialization: no per-record zip padding, which keeps the file under 10^6 bytes
    torch.save(out, os.path.join(GOLD, f"infer_{kind}.pt"), _use_new_zipfile_serialization=False)
    print(f"[infer/{kind}] samples |x|={samples.norm().item():.6f} img |x|={img.norm().item():.6f} "
          f"timesteps={out['ddim_timesteps'].tolist()}")


def run_curve(kind="tiny", steps=50, lr=5e-3):
    """BASELINE config 1/2 in miniature: `steps` optimiser steps of the UNMODIFIED reference (shared_step -> backward ->
    torch.optim.AdamW as configure_optimizers builds it, ddpm.py:1442-1454) on the replayed per-step stream
    workload.synth_batch(kind, step=i): the loss curve, the trained tensors and the identity EMA the user's
    embeddings_gs-*.pt would hold."""
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    basis = synth.synth_celeb_basis(seed=0)
    model = ref_shim.build_reference(workload.model_params(kind), seed=0, clip_layers=workload.clip_layers(kind),
                                     celeb_basis=basis)
    model.learning_rate = lr
    opt = model.configure_optimizers()
    opt = opt[0] if isinstance(opt, (list, tuple)) else opt
    em = model.embedding_manager
    init = {"coef": em.id_coefficients[0].detach().clone(), "emb": em.id_embeddings[0].detach().clone()}
    losses, ts = [], []
    t0 = time.time()
    for i in range(steps):
        batch, draws = workload.synth_batch(kind, B=1, seed=1234, step=i)
        with ref_shim.replay_randomness(draws["t"], draws["noise"], draws["posterior_eps"]):
            loss, _ = model.shared_step(batch)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
        ts.append(int(draws["t"][0]))
    lin = em.meta_id_net.stylegan_mlp.net[0]
    out = {"kind": kind, "steps": steps, "lr": lr, "losses": torch.tensor(losses, dtype=torch.float64), "t": ts,
           "W_final_rows4": lin.weight.detach()[::4].clone(),   # every 4th output row
           "b_final": lin.bias.detach().clone(),
           "ema_coef_id0_init": init["coef"], "ema_emb_id0_init": init["emb"],
           "ema_coef_id0": em.id_coefficients[0].detach().clone(), "ema_emb_id0": em.id_embeddings[0].detach().clone(),
           "optimizer": type(opt).__name__, "opt_defaults": {k: v for k, v in opt.defaults.items() if isinstance(v, (int, float, tuple, bool))}}
    torch.save(out, os.path.join(GOLD, f"curve_{kind}.pt"))
    print(f"[curve/{kind}] {steps} steps in {time.time() - t0:.1f}s; loss[0]={losses[0]:.6f} loss[-1]={losses[-1]:.6f} "
          f"optimizer={out['optimizer']} {out['opt_defaults']}")


def _token_len_table():
    """infer_images/token_len.txt (written by modules.py:503-515 with the real CLIP BPE vocabulary): name -> real ids."""
    import re
    table = {}
    with open(os.path.join(ref_shim.REF_ROOT, "infer_images", "token_len.txt")) as f:
        for line in f:
            m = re.match(r"\d+ (.*): len=\d+, token=\[(.*)\]\s*$", line)
            if m:
                table[m.group(1)] = [int(t) for t in m.group(2).split(",") if t.strip()]
    return table


def run_basis():
    """f3: FrozenCLIPEmbedder._get_celeb_embeddings (modules.py:472-624) of the UNMODIFIED reference on its own name list
    (infer_images/wiki_names_v2.txt) with the REAL CLIP token ids of infer_images/token_len.txt (names that file does not
    list fall back to the synthetic per-word ids), a synthetic token-embedding table, three configurations."""
    table = _token_len_table()
    ref_shim.PHRASES.clear()
    ref_shim.PHRASES.update(table)
    ref_shim.install_stubs(2)
    from ldm.modules.encoders.modules import FrozenCLIPEmbedder
    names_path = os.path.join(ref_shim.REF_ROOT, "infer_images", "wiki_names_v2.txt")
    with open(names_path) as f:
        names = f.read().splitlines()
    out = {"names": names, "phrases": {n: table[n] for n in set(names) if n in table}, "cases": []}
    for cfg in (dict(use_flatten=False, use_sample_reduce=False), dict(use_flatten=True, use_sample_reduce=False),
                dict(use_flatten=False, use_sample_reduce=True)):
        torch.manual_seed(0)
        emb = FrozenCLIPEmbedder(device="cpu", celeb_txt=names_path, use_celeb=False, use_svd=True, n_components=512,
                                 rm_repeats=True, n_samples=513, num_embeds_per_token=2, **cfg)
        sd = synth.synth_state_dict(emb, seed=0, prefix="cond_stage_model.")
        emb.load_state_dict(sd, strict=False)
        emb.use_celeb = True
        emb._get_celeb_embeddings(512)
        ce = emb.celeb_embeddings.detach().float().cpu()
        out["cases"].append({"cfg": cfg, "shape": tuple(ce.shape), "mean_rows": ce[:, 0].clone(),
                             "head": ce[:, :33].clone(), "row_norms": ce.norm(dim=-1).clone(),
                             "gram_diag_err": float((ce[:, 1:] @ ce[:, 1:].transpose(1, 2)
                                                     - torch.eye(ce.shape[1] - 1)).abs().max())})
        print(f"[basis] {cfg}: shape {tuple(ce.shape)} |mean| {ce[:, 0].norm(dim=-1).tolist()}")
    torch.save(out, os.path.join(GOLD, "celeb_basis.pt"))


def run_ti():
    """f4: the vanilla Textual-Inversion EmbeddingManager.forward of the UNMODIFIED reference (embedding_manager.py:38-184)
    on CPU: one vector per token and three vectors per token (insertion with shifting), two placeholders, and the
    checkpoint its save() writes."""
    ref_shim.install_stubs(2)
    from ldm.modules.encoders.modules import FrozenCLIPEmbedder
    from ldm.modules.embedding_manager import EmbeddingManager
    torch.manual_seed(0)
    emb = FrozenCLIPEmbedder(device="cpu", use_celeb=False)
    emb.load_state_dict(synth.synth_state_dict(emb, seed=0, prefix="cond_stage_model."), strict=False)
    tok = emb.tokenizer
    prompts = ["a photo of * person", "* and ks with a * face", "no placeholder here"]
    cases = []
    import tempfile
    for nv in (1, 3):
        torch.manual_seed(1)
        em = EmbeddingManager(emb, placeholder_strings=["*", "ks"], initializer_words=None, num_vectors_per_token=nv)
        ids = tok(prompts, truncation=True, max_length=77, return_length=True, return_overflowing_tokens=False,
                  padding="max_length", return_tensors="pt")["input_ids"]
        g = torch.Generator().manual_seed(5)
        text = torch.randn(len(prompts), 77, 768, generator=g)
        ids_in, text_in = ids.clone(), text.clone()
        out = em(ids_in, text_in)
        out.sum().backward() if out.requires_grad else None
        with tempfile.TemporaryDirectory() as td:
            em.save(os.path.join(td, "ti.pt"))
            ck = torch.load(os.path.join(td, "ti.pt"), weights_only=False)
        cases.append({"nv": nv, "ids": ids, "text_seed": 5, "text_sum": float(text.double().sum()),
                      # only the rows of `out` that differ from the seeded input text (the rest is that text)
                      "out_rows": (out.detach() != text).any(-1).nonzero(),
                      "out_vals": out.detach()[(out.detach() != text).any(-1)].clone(), "ids_after": ids_in.clone(),
                      "params": {k: v.detach().clone() for k, v in em.string_to_param_dict.items()},
                      "tokens": {k: int(v) for k, v in em.string_to_token_dict.items()},
                      "grads": {k: (v.grad.detach().clone() if v.grad is not None else None)
                                for k, v in em.string_to_param_dict.items()},
                      "ckpt_keys": sorted(ck.keys()), "ckpt_types": {k: type(v).__name__ for k, v in ck.items()}})
        print(f"[ti] nv={nv}: out {tuple(out.shape)} ids_after[1][:12]={ids_in[1][:12].tolist()}")
    torch.save({"prompts": prompts, "cases": cases}, os.path.join(GOLD, "ti_manager.pt"))


def run_data():
    """f2: FaceIdDatasetOneShot.__getitem__ of the UNMODIFIED reference (PIL + torchvision transforms on the host) on
    synthetic images: captions, identity lists, the tensors it yields and the state of the three RNGs after each item (the
    device data path must consume exactly the same draws)."""
    import hashlib
    import pickle
    import random
    import tempfile
    ref_shim.install_stubs(2)
    from ldm.data.face_id import FaceIdDatasetOneShot
    hw = 64
    with tempfile.TemporaryDirectory() as td:
        pk, _ = workload.synth_face_files(td, n=4, hw=hw, seed=0)
        items = []
        for split, diff in (("train", 0), ("train", 1)):
            random.seed(11)
            np.random.seed(11)
            torch.manual_seed(11)
            ds = FaceIdDatasetOneShot(pk, num_ids=3, specific_ids=[0, 1, 3], image_size=hw, repeats=5, split=split,
                                      diff_cnt=diff)
            for i in (0, 4, 7):
                ex = ds[i]
                dig = hashlib.sha1(pickle.dumps((random.getstate(), np.random.get_state()[1].tobytes(),
                                                 np.random.get_state()[2], torch.get_rng_state().numpy().tobytes()))).hexdigest()
                items.append({"split": split, "diff_cnt": diff, "index": i, "caption": ex["caption"],
                              "ids": ex["image_ori"]["ids"].clone(), "num_ids": ex["image_ori"]["num_ids"],
                              "image": ex["image"].half(), "faces": ex["image_ori"]["faces"].half(), "rng_digest": dig,
                              "len": len(ds)})
    torch.save({"hw": hw, "items": items, "seed": 11}, os.path.join(GOLD, "data_path.pt"))
    print("[data]", [(it["index"], it["caption"], it["ids"].tolist()) for it in items])


def helpers_kat():
    """helpers.py:44-54 toy case, computed by the reference's own functions."""
    ref_shim.install_stubs()
    from ldm.modules.id_embedding.helpers import get_rep_pos, shift_tensor_dim0
    tok = torch.LongTensor([0, 1, 2, 2, 3, 4, 5, 6, 7, 99] + [99] * 20)
    pos = get_rep_pos(tok, [2, 6])
    res, fin = shift_tensor_dim0(tok.clone(), pos, 2)
    cases = [{"tokens": tok, "rep_tokens": [2, 6], "reps": 2, "rep_pos": [p.tolist() for p in pos],
              "result": res, "final_pos": [f.tolist() for f in fin]}]
    rng = np.random.RandomState(0)
    for _ in range(40):
        n = 77
        t = torch.from_numpy(rng.randint(1000, 2000, size=n)).long()
        toks = list(range(5, 5 + int(rng.randint(1, 4))))
        reps = int(rng.randint(1, 4))
        for tk in toks:  # each placeholder occurs 1-2 times, early in the prompt (as in real captions)
            for p_ in rng.choice(np.arange(1, 30), size=int(rng.randint(1, 3)), replace=False):
                if int(t[p_]) >= 1000:
                    t[p_] = tk
        pos = get_rep_pos(t, toks)
        emb = torch.arange(n).float()[:, None].repeat(1, 3)
        res, fin = shift_tensor_dim0(emb.clone(), pos, reps)
        cases.append({"tokens": t, "rep_tokens": toks, "reps": reps, "rep_pos": [p.tolist() for p in pos],
                      "result": res[:, 0].long(), "final_pos": [f.tolist() for f in fin]})
    torch.save(cases, os.path.join(GOLD, "helpers_kat.pt"))
    print(f"[helpers] {len(cases)} known-answer cases")


if __name__ == "__main__":
    which = sys.argv[1:] or ["helpers", "tiny"]
    for w in which:
        if w == "helpers":
            helpers_kat()
        elif w == "infer":
            run_infer("tiny")
        elif w == "curve":
            run_curve("tiny")
        elif w == "basis":
            run_basis()
        elif w == "data":
            run_data()
        elif w == "ti":
            run_ti()
        else:
            run(w)
