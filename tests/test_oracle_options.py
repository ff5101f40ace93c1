"""CPU: the fp32 port of the training-step options (oracle/options_ref.py) and the host arithmetic of the fused step
against what the UNMODIFIED reference recorded in tests/golden/step_options_tiny.pt (oracle/make_golden_options.py):
8 shared_step -> backward -> AdamW steps of CelebBasis with 1/2/3-person prompts and loss weights, and of Textual
Inversion with two placeholders, 2 vectors per token, the coarse regulariser and progressive words."""
import os
import types

import numpy as np
import pytest
import torch

from celebbasis_b200 import synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from oracle import options_ref, torch_ref


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "step_options_tiny.pt"), weights_only=False)


def _oracle(params):
    torch.manual_seed(0)
    om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers("tiny"))
    om.load_state_dict(synth.synth_state_dict(om, seed=0), strict=False)
    return om.eval()


def _tables(params):
    T = params["timesteps"]
    return (torch.full((T,), float(params["logvar_init"])),
            options_ref.lvlb_weights(T, params["linear_start"], params["linear_end"]),
            (params["l_simple_weight"], params["original_elbo_weight"]))


def test_celebbasis_persons_and_weights_match_reference(gold):
    g = gold["cb"]
    p = g["params"]
    om = _oracle(p)
    tok = SyntheticCLIPTokenizer()
    ph = [tok.word_id(s) for s in p["personalization_config"]["params"]["placeholder_strings"][:3]]
    pc = p["personalization_config"]["params"]
    basis = synth.synth_celeb_basis(seed=0)
    logvar, lvlb, weights = _tables(p)
    W, b = om.trainable()
    opt = torch.optim.AdamW([W, b], lr=g["lr"])
    ema_coef, ema_emb = g["ema_coef0"].clone(), g["ema_emb0"].clone()
    losses = []
    for s in range(g["steps"]):
        batch, d = workload.synth_persons_batch(s), g["draws"][s]
        ids = tok(batch["caption"])["input_ids"]
        loss, vlb, positions, order = options_ref.cb_step(om, batch, d, ids, basis, ph, logvar, lvlb, weights, ema_coef,
                                                          ema_emb, pc["momentum"])
        assert positions == g["positions"][s], s
        assert order == g["ema_order"][s], s
        assert abs(vlb.item() - g["loss_vlb"][s].item()) <= 1e-5 * abs(g["loss_vlb"][s].item())
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    err = (torch.tensor(losses, dtype=torch.float64) - g["losses"]).abs() / g["losses"].abs()
    assert float(err.max()) <= 1e-5, (losses, g["losses"].tolist())
    assert _rel(W.detach()[::4], g["W_final_rows4"]) < 1e-4 and _rel(b.detach(), g["b_final"]) < 1e-4
    assert _rel(ema_coef, g["ema_coef"]) < 1e-5 and _rel(ema_emb, g["ema_emb"]) < 1e-5


def test_celebbasis_host_maps_and_ema_order_bit_exact(gold):
    """The fused step's host arithmetic: the row map's placeholder positions (build_inject_map_multi) and the EMA list
    (CelebBasisStep.ema_slots over the flat identity tensor) reproduce the reference's, step by step."""
    from celebbasis_b200.train_step import CelebBasisStep, build_inject_map_multi
    g = gold["cb"]
    tok = SyntheticCLIPTokenizer()
    ph = [tok.word_id(s) for s in g["params"]["personalization_config"]["params"]["placeholder_strings"][:3]]
    for s in range(g["steps"]):
        batch = workload.synth_persons_batch(s)
        io = batch["image_ori"]
        ids = tok(batch["caption"])["input_ids"].numpy()
        nid = [int(k) for k in io["num_ids"]]
        _, positions = build_inject_map_multi(ids, [(ph[:k], [0] * k) for k in nid], 2)
        assert [[f.tolist() for f in pos] for pos in positions] == g["positions"][s], s
        slot = CelebBasisStep.ema_slots(nid, io["ids"].shape[1])
        flat = io["ids"].reshape(-1).tolist()
        assert [flat[k] for k in slot.tolist() if k >= 0] == g["ema_order"][s], s


def test_textual_inversion_options_match_reference(gold):
    g = gold["ti"]
    p = g["params"]
    om = _oracle(p)
    tok = SyntheticCLIPTokenizer()
    logvar, lvlb, weights = _tables(p)
    params = {k: v.clone().requires_grad_(True) for k, v in g["params0"].items()}
    opt = torch.optim.AdamW(list(params.values()), lr=g["lr"])
    counter, losses = g["counter0"], []
    for s in range(g["steps"]):
        batch, d = workload.synth_ti_option_batch(s), g["draws"][s]
        ids = tok(batch["caption"])["input_ids"]
        loss, new_ids, counter = options_ref.ti_step(om, batch, d, ids, g["tokens"], params, g["initial"], True, counter,
                                                     logvar, lvlb, weights, p["embedding_reg_weight"])
        assert counter == g["counters"][s] and torch.equal(new_ids, g["rewritten_ids"][s]), s
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    err = (torch.tensor(losses, dtype=torch.float64) - g["losses"]).abs() / g["losses"].abs()
    assert float(err.max()) <= 1e-5, (losses, g["losses"].tolist())
    for k, v in params.items():
        assert _rel(v.detach(), g["params_final"][k]) < 1e-4, k


def test_textual_inversion_host_map_bit_exact(gold):
    """EmbeddingManager.ti_map (what the fused step injects from) rewrites the prompts as the reference did, with the
    progressive-words counter advanced once per placeholder per step, across the PROGRESSIVE_SCALE boundary."""
    from ldm.modules.embedding_manager import EmbeddingManager
    g = gold["ti"]
    tok = SyntheticCLIPTokenizer()
    em = types.SimpleNamespace(string_to_token_dict=dict(g["tokens"]), string_to_param_dict=g["params0"],
                               max_vectors_per_token=2, progressive_words=True, progressive_counter=g["counter0"])
    for s in range(g["steps"]):
        ids = tok(workload.synth_ti_option_batch(s)["caption"])["input_ids"].numpy()
        _, new_ids = EmbeddingManager.ti_map(em, ids)
        assert em.progressive_counter == g["counters"][s]
        assert np.array_equal(new_ids, g["rewritten_ids"][s].numpy()), s
    assert g["counters"][0] < options_ref.PROGRESSIVE_SCALE <= g["counters"][-1]
