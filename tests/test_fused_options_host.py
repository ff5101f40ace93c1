"""CPU tests of the training-step options the fused CUDA-graph step accepts (loss weights, multi-person prompts, the
Textual Inversion coarse regulariser and progressive words):

  * which batches and configurations LatentDiffusion._fused_applicable sends to the fused step;
  * the eager p_losses gives a scalar loss with num_vectors_per_token 2 and embedding_reg_weight > 0, with the
    reference's weighted loss and gradient;
  * the multi-person EMA order list;
  * what ptxas made of the new kernels (sm_90a, no spills).
"""
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from celebbasis_b200 import build
from test_gemm_sass import _tool, spills

NEW_KERNELS = ("diffusion_loss_sample_kernel", "diffusion_loss_batch_kernel", "ti_coarse_reg_kernel",
               "ema_rows_sel_kernel")


def _model(ti=False, **over):
    from celebbasis_b200 import workload
    from ldm.models.diffusion.ddpm import LatentDiffusion
    torch.manual_seed(0)
    params = workload.ti_model_params("tiny", num_vectors_per_token=2) if ti else workload.model_params("tiny")
    params["cond_stage_config"]["params"].update(num_hidden_layers=1)
    if ti:
        params["personalization_config"]["params"].update(placeholder_strings=["*", "sks"],
                                                          initializer_words=["person"], progressive_words=True)
    params.update(over)
    model = LatentDiffusion(**params).train()
    if not ti:
        model.cond_stage_model.celeb_embeddings = torch.zeros(2, 513, 768)
    return model


def _on_gpu(model):
    """The gate's last question is whether the model's weights live on a CUDA device: answer yes without one."""
    model.model.parameters = lambda: iter([types.SimpleNamespace(is_cuda=True)])
    return model


def _cb_batch(num_ids, n_chunks=4, hw=64):
    B = len(num_ids)
    return {"image": torch.zeros(B, hw, hw, 3), "caption": ["a photo of sks"] * B,
            "image_ori": {"faces": torch.zeros(B, hw, hw, 3 * n_chunks), "ids": torch.zeros(B, n_chunks, dtype=torch.long),
                          "num_ids": torch.tensor(num_ids)}}


WEIGHTS = dict(l_simple_weight=0.5, original_elbo_weight=1e-2, logvar_init=0.1)


@pytest.mark.parametrize("weights", [{}, WEIGHTS, dict(embedding_reg_weight=1e-2), dict(WEIGHTS, embedding_reg_weight=1e-2)])
def test_fused_applicable_celebbasis(weights):
    model = _on_gpu(_model(**weights))
    for nid in ([1], [1, 1], [2, 1], [3, 2], [3, 3, 1]):
        assert model._fused_applicable(_cb_batch(nid)), nid
    assert model._fused_applicable(_cb_batch([1], n_chunks=2))
    assert model._fused_applicable(_cb_batch([2, 2], n_chunks=2))
    # a three-person prompt names a third identity: the batch must carry one (the eager route fails on it as well)
    assert not model._fused_applicable(_cb_batch([3], n_chunks=2))


@pytest.mark.parametrize("weights", [{}, WEIGHTS, dict(WEIGHTS, embedding_reg_weight=1e-2)])
def test_fused_applicable_textual_inversion(weights):
    model = _on_gpu(_model(ti=True, **weights))
    assert model.embedding_manager.progressive_words and model.embedding_manager.max_vectors_per_token == 2
    batch = {"image": torch.zeros(2, 64, 64, 3), "caption": ["a photo of *", "a photo of sks"]}
    assert model._fused_applicable(batch)


def test_fused_route_refused_only_for_unfreeze_env_and_cpu(monkeypatch):
    batch = _cb_batch([2, 3])
    assert not _model(**WEIGHTS)._fused_applicable(batch)                 # weights on the CPU
    assert not _on_gpu(_model(unfreeze_model=True))._fused_applicable(batch)
    monkeypatch.setenv("CB_FUSED_STEP", "0")
    assert not _on_gpu(_model(**WEIGHTS))._fused_applicable(batch)
    ti = _model(ti=True, embedding_reg_weight=1e-2)
    assert not ti._fused_applicable({"image": torch.zeros(1, 64, 64, 3), "caption": ["*"]})


def test_eager_p_losses_scalar_with_coarse_regulariser(monkeypatch):
    """num_vectors_per_token 2 makes embedding_to_coarse_loss a 2x2 matrix; the reference averages it (ddpm.py:1102).
    The loss is the reference's weighted sum, and its gradient reaches the prediction through loss_vlb too."""
    model = _model(ti=True, embedding_reg_weight=1e-2, **WEIGHTS)
    em = model.embedding_manager
    with torch.no_grad():
        em.string_to_param_dict["*"].add_(0.01 * torch.randn(2, 768))
    pred = torch.randn(2, 4, 8, 8, requires_grad=True)
    monkeypatch.setattr(model, "q_sample", lambda x_start, t, noise: x_start)
    monkeypatch.setattr(model, "apply_model", lambda x, t, c: pred)
    monkeypatch.setattr(model, "get_loss", lambda p, tgt, mean=True: ((p - tgt) ** 2).mean([1, 2, 3]))
    x0, noise, t = torch.zeros(2, 4, 8, 8), torch.randn(2, 4, 8, 8), torch.tensor([0, 999])
    loss, d = model.p_losses(x0, None, t, noise=noise)
    assert loss.dim() == 0
    loss.backward()
    ls = ((pred.detach() - noise) ** 2).mean([1, 2, 3])
    lv = model.logvar[t]
    delta = em.string_to_param_dict["*"].detach() - em.initial_embeddings["*"]
    reg = (delta @ delta.T / 1).mean()
    want = 0.5 * (ls / torch.exp(lv) + lv).mean() + 1e-2 * (model.lvlb_weights[t] * ls).mean() + 1e-2 * reg
    assert torch.allclose(loss.detach(), want, rtol=1e-6)
    f = (0.5 / torch.exp(lv) + 1e-2 * model.lvlb_weights[t]) / 2
    dpred = 2 * (pred.detach() - noise) / (4 * 8 * 8) * f.view(2, 1, 1, 1)
    assert torch.allclose(pred.grad, dpred, rtol=1e-5, atol=1e-12)
    g = em.string_to_param_dict["*"].grad
    assert torch.allclose(g, (2e-2 * delta.sum(0) / 4).expand(2, -1), rtol=1e-4, atol=1e-9)


def test_multi_person_ema_order():
    """Per sample, then its first, second, third person (embedding_manager.py:321-392); -1 pads the fixed-size list."""
    from celebbasis_b200.train_step import CelebBasisStep
    slot = CelebBasisStep.ema_slots([1, 3, 2], 4)
    assert slot.dtype == np.int32
    assert slot.tolist() == [0, -1, -1, 4, 5, 6, 8, 9, -1]
    assert CelebBasisStep.person_chunks(4) == ((0, 1, 2), (0, 1, 1))
    assert CelebBasisStep.person_chunks(2) == ((0, 1, 1), (0, 1, 1))


def test_new_kernels_compile_for_sm90a_without_spills(tmp_path):
    nvcc = _tool("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not available")
    obj = str(tmp_path / "cb_embed.o")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "cb_embed.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sp = spills(r.stdout + r.stderr)
    for k in NEW_KERNELS:
        found = {f: s for f, s in sp.items() if k in f}
        assert len(found) == 1, (k, found)
        assert list(found.values()) == [(0, 0)], found
    assert "sm_90a" in r.stdout + r.stderr
