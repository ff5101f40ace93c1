"""CPU: pin the oracle restatement (oracle/torch_ref.py) against fixtures produced by the UNMODIFIED reference
(oracle/make_golden.py ran /root/reference's LatentDiffusion.shared_step + backward through oracle/ref_shim.py)."""
import os

import numpy as np
import pytest
import torch

from celebbasis_b200 import synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from oracle import torch_ref


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-30)).item()


def test_helpers_known_answers(golden_dir):
    """ldm/modules/id_embedding/helpers.py: integer path, bit-exact (incl. the reference's own __main__ toy case)."""
    cases = torch.load(os.path.join(golden_dir, "helpers_kat.pt"))
    assert len(cases) >= 20
    for c in cases:
        tok = c["tokens"].numpy()
        pos = torch_ref.get_rep_pos(tok, c["rep_tokens"])
        assert [p.tolist() for p in pos] == c["rep_pos"]
        src, fin = torch_ref.shift_index_map(tok.shape[0], pos, c["reps"])
        assert [f.tolist() for f in fin] == c["final_pos"]
        if c is cases[0]:
            got = tok[src]            # the toy case shifts the token vector itself
        else:
            got = src                 # the others shift arange(n)
        assert got.tolist() == c["result"].tolist()
    first = cases[0]
    assert first["rep_pos"] == [[2, 3], [7]] and first["final_pos"] == [[[2, 3], [4, 5]], [[9, 10]]]


def test_tiny_step_matches_reference(golden_dir):
    """Whole training-step forward + backward of the restatement == the reference's, fp32, same weights/inputs."""
    gold = torch.load(os.path.join(golden_dir, "step_tiny.pt"))
    torch.manual_seed(0)
    params = workload.model_params("tiny")
    model = torch_ref.OracleModel(params, clip_layers=workload.clip_layers("tiny"))
    sd = synth.synth_state_dict(model, seed=0)
    model.load_state_dict(sd, strict=True)
    model.eval()
    batch, draws = workload.synth_batch("tiny", B=1, seed=1234)
    ids = SyntheticCLIPTokenizer()(batch["caption"])["input_ids"]
    basis = synth.synth_celeb_basis(seed=0)
    W, b = model.trainable()
    W.requires_grad_(True)
    b.requires_grad_(True)
    out = model.step(batch, draws, ids, basis, placeholder_token=SyntheticCLIPTokenizer.word_id("sks"))
    out["loss"].backward()
    assert _rel(out["face_feat"], torch.nn.functional.normalize(gold["face_feat"], dim=-1)) < 1e-5
    assert _rel(out["z"], gold["z"]) < 1e-5
    assert _rel(out["coef"], gold["celeb_coef"]) < 1e-5
    assert _rel(out["celeb_z"], gold["celeb_z"]) < 1e-5
    assert _rel(out["context"], gold["context"]) < 1e-5
    assert _rel(out["x_noisy"], gold["x_noisy"]) < 1e-5
    assert _rel(out["eps"], gold["eps"]) < 1e-4
    assert abs(out["loss"].item() - gold["loss"].item()) / abs(gold["loss"].item()) < 1e-5
    assert _rel(W.grad[::8], gold["gW_rows8"]) < 1e-3 and abs(W.grad.norm().item() / gold["gW_norm"].item() - 1) < 1e-3
    assert _rel(b.grad, gold["gb"]) < 1e-3
    assert gold["graded"] == ["embedding_manager.meta_id_net.stylegan_mlp.net.0.weight",
                              "embedding_manager.meta_id_net.stylegan_mlp.net.0.bias"]
    # placeholder lands at positions 7,8 of "a photo of a face of sks person"
    assert [f.tolist() for f in out["positions"][0]] == [[[7, 8]]]


def test_tiny_inference_matches_reference(golden_dir):
    """DDIM txt2img + VAE decode (scripts/stable_txt2img.py semantics: eval-mode conditioning from stored coefficients,
    DDIMSampler.sample with CFG and eta 0, decode_first_stage): the restatement == the UNMODIFIED reference (fixture from
    `python oracle/make_golden.py infer`)."""
    import torch.nn.functional as F
    gold = torch.load(os.path.join(golden_dir, "infer_tiny.pt"))
    params = workload.model_params("tiny")
    om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers("tiny"))
    sd = synth.synth_state_dict(om, seed=0)
    om.load_state_dict(sd, strict=True)
    om.eval()
    basis = synth.synth_celeb_basis(seed=0)
    g = torch.Generator().manual_seed(gold["coef_seed"])
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    x_T = torch.randn(1, 4, params["image_size"], params["image_size"], generator=g)
    assert torch.equal(x_T, gold["x_T"])                                   # same draw order as the fixture generator
    tok = SyntheticCLIPTokenizer()
    tm = om.cond_stage_model.transformer.text_model
    with torch.no_grad():
        uc = tm.forward_embeds(tm.embed_tokens(tok([""])["input_ids"]))
        ids = tok(gold["prompts"])["input_ids"]
        z = torch_ref.celeb_basis(coefs[gold["person_id"]].view(1, 2, 1, 512), basis)
        emb, pos = torch_ref.inject_embeddings(ids, tm.embed_tokens(ids), z, tok.word_id("sks"), 2)
        c = tm.forward_embeds(emb)
        x = torch_ref.ddim_sample(om.model.diffusion_model, om.sched, c, uc, x_T, gold["steps"], gold["scale"])
        fs = params["first_stage_config"]["params"]
        dec = torch_ref.AutoencoderKLDecode(fs["ddconfig"], fs["embed_dim"])
        # decoder / post_quant_conv weights: the same deterministic function of (seed, reference key, shape) the
        # reference model was loaded with (keys first_stage_model.decoder.*, first_stage_model.post_quant_conv.*)
        dec.load_state_dict(synth.synth_state_dict(dec, seed=0, prefix="first_stage_model."), strict=True)
        img = dec(x / 0.18215)
    assert _rel(uc, gold["uc"]) < 1e-5 and _rel(c, gold["c"]) < 1e-5
    assert _rel(x, gold["samples"]) < 1e-4
    assert img.shape == gold["img"].shape and _rel(img, gold["img"]) < 1e-4



def test_multi_identity_conditioning_matches_reference(golden_dir):
    """Two / three persons in one prompt (embedding_manager.py:323-345,362-392, eval branch): the host row map
    (train_step.build_inject_map_multi: integer, bit-exact placeholder arithmetic) applied to the restatement's token
    embeddings, through the CLIP restatement == the UNMODIFIED reference's get_learned_conditioning."""
    import torch.nn.functional as F
    from celebbasis_b200.train_step import build_inject_map_multi
    gold = torch.load(os.path.join(golden_dir, "infer_tiny.pt"))
    params = workload.model_params("tiny")
    om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers("tiny"))
    om.load_state_dict(synth.synth_state_dict(om, seed=0), strict=True)
    om.eval()
    basis = synth.synth_celeb_basis(seed=0)
    g = torch.Generator().manual_seed(gold["coef_seed"])
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    tok = SyntheticCLIPTokenizer()
    tm = om.cond_stage_model.transformer.text_model
    words = params["personalization_config"]["params"]["placeholder_strings"]
    es = params["personalization_config"]["params"]["num_embeds_per_token"]
    assert len(gold["multi"]) == 2
    for case in gold["multi"]:
        pid = case["ids"]
        ids = tok([case["prompt"]])["input_ids"]
        ph = [tok.word_id(words[k]) for k in range(len(pid))]
        with torch.no_grad():
            z = torch.cat([torch_ref.celeb_basis(coefs[i].view(1, 2, 1, 512), basis)[0] for i in pid], 0)   # (persons*es, 768)
            m, pos = build_inject_map_multi(ids.numpy(), [(ph, [k * es for k in range(len(pid))])], es)
            e = tm.embed_tokens(ids)[0]
            rows = [e[int(j)] if j >= 0 else z[-int(j) - 1] for j in m[0]]
            c = tm.forward_embeds(torch.stack(rows, 0)[None])
        assert _rel(c, case["c"]) < 1e-5, case["prompt"]
        assert len(pos[0]) == len(pid) and all(len(p) >= 1 for p in pos[0])
