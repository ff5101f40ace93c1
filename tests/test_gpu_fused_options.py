"""GPU tests of the training-step options the CUDA-graph step runs since it took over from the eager route:

  * cb_diffusion_loss_fwd_bwd (p_losses with l_simple_weight / logvar / original_elbo_weight, t read on the device),
    cb_ti_coarse_reg (the Textual Inversion coarse regulariser) and cb_ema_rows_sel (the multi-person EMA order) against
    fp64 / host references, with NaN-poisoned outputs and bit-identical repeat launches;
  * Trainer.fit on the fused route against the eager per-module route (CB_FUSED_STEP=0) at the same seeds: loss weights,
    mixed 1/2/3-person CelebBasis batches, and Textual Inversion with two placeholders (one without an initializer
    word), num_vectors_per_token 2, the coarse regulariser and progressive words crossing a step boundary;
  * one graph capture across steps whose person mix and progressive length change; two runs bit-identical.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.double().cpu().flatten(), b.double().cpu().flatten()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 8])
@pytest.mark.parametrize("t_kind", ["zero", "one", "last", "mixed"])
def test_diffusion_loss_vs_fp64(dev, B, t_kind):
    from celebbasis_b200 import lib, ops
    T, per = 1000, 4 * 8 * 8 + 3          # a per-sample length that is not a multiple of the block
    g = torch.Generator().manual_seed(B * 31 + len(t_kind))
    pred, target = torch.randn(B, per, generator=g), torch.randn(B, per, generator=g)
    t = {"zero": torch.zeros(B), "one": torch.ones(B), "last": torch.full((B,), T - 1),
         "mixed": torch.tensor([0, 1, T - 1, 500, 7, 999, 1, 0][:B])}[t_kind].long()
    logvar = 0.1 + 0.05 * torch.randn(T, generator=g)
    lvlb = torch.rand(T, generator=g) * 3 + 0.1
    lvlb[0] = lvlb[1]
    lsw, ew, gscale = 0.5, 1e-2, 4.0
    # fp64 reference: ddpm.py:1084-1099
    p64 = pred.double().requires_grad_(True)
    ls = ((p64 - target.double()) ** 2).mean(1)
    lv = logvar.double()[t]
    loss = lsw * (ls / torch.exp(lv) + lv).mean()
    vlb = (lvlb.double()[t] * ls).mean()
    loss = loss + ew * vlb
    loss.backward()
    outs = []
    d_pred, d_target, d_t, d_logvar, d_lvlb = (x.to(dev) for x in (pred, target, t, logvar, lvlb))   # alive past the call
    for _ in range(2):
        lsimple = torch.full((B,), float("nan"), device=dev)
        o = torch.full((2,), float("nan"), device=dev)
        grad = torch.full((B, per), float("nan"), device=dev)
        rc = lib.load().cb_diffusion_loss_fwd_bwd(
            ops._p(d_pred), ops._p(d_target), ops._p(d_t), ops._p(d_logvar), ops._p(d_lvlb),
            lsw, ew, ops._p(lsimple), ops._p(o[0:1]), ops._p(o[1:2]), ops._p(grad), B, per, gscale, ops._st())
        assert rc == 0, lib.last_error()
        torch.cuda.synchronize()
        outs.append((lsimple.cpu(), o.cpu(), grad.cpu()))
    lsimple, o, grad = outs[0]
    assert rel(lsimple, ls.detach()) < 1e-6
    assert abs(o[0].item() - loss.item()) <= 1e-6 * abs(loss.item())
    assert abs(o[1].item() - vlb.item()) <= 1e-6 * abs(vlb.item())
    assert rel(grad, p64.grad * gscale) < 1e-6
    for x, y in zip(outs[0], outs[1]):
        assert torch.equal(x, y)
    # the ops wrapper, with the gradient skipped
    ls2, l2, v2, g2 = ops.diffusion_loss_fwd_bwd(d_pred, d_target, d_t, d_logvar, d_lvlb, lsw, ew, gscale, want_grad=False)
    assert g2 is None and torch.equal(ls2.cpu(), lsimple) and torch.equal(l2.cpu(), o[0:1]) and torch.equal(v2.cpu(), o[1:2])


@pytest.mark.parametrize("nv", [1, 2, 3])
@pytest.mark.parametrize("n_init", [1, 2])
def test_ti_coarse_reg_vs_fp64(dev, nv, n_init):
    from celebbasis_b200 import ops
    D, w = 768, 1e-2
    g = torch.Generator().manual_seed(nv * 7 + n_init)
    p0 = torch.randn(nv, D, generator=g)
    p = p0 + 0.05 * torch.randn(nv, D, generator=g)
    grad0 = torch.randn(nv, D, generator=g)
    loss0 = torch.tensor([1.25])
    # fp64 reference: embedding_manager.py:170-180 for this placeholder, ddpm.py:1101-1107
    q = p.double().requires_grad_(True)
    d = q - p0.double()
    reg = w * (d @ d.T / n_init).mean()
    reg.backward()
    outs = []
    for _ in range(2):
        grad, loss = grad0.to(dev).clone(), loss0.to(dev).clone()
        ops.ti_coarse_reg(p.to(dev), p0.to(dev), grad, loss, n_init, w)
        torch.cuda.synchronize()
        outs.append((grad.cpu(), loss.cpu()))
    grad, loss = outs[0]
    assert abs(loss.item() - (1.25 + reg.item())) <= 1e-6 * (1.25 + reg.item())
    # the increment is ~1e-3 of the preset gradient: compare the sum (the increment alone would measure fp32 rounding)
    assert rel(grad, grad0.double() + q.grad) < 1e-6
    assert ((grad.double() - grad0.double()) - q.grad).abs().max().item() <= 2 ** -22 * grad0.abs().max().item()
    for x, y in zip(outs[0], outs[1]):
        assert torch.equal(x, y)


def test_ema_rows_sel_follows_list_order(dev):
    """Entries of one identity fold in list order; unused entries and identities outside the table are skipped."""
    from celebbasis_b200 import ops
    g = torch.Generator().manual_seed(3)
    n_rows, row, m = 10, 2 * 768, 0.9
    table = torch.randn(n_rows, row, generator=g)
    ids = torch.tensor([[1, 3, 5, 7], [2, 12, 3, 6], [3, 1, 1, 9]])        # identity 1 three times, 3 twice, 12 outside
    nid, n_chunks = [2, 3, 3], 4
    from celebbasis_b200.train_step import CelebBasisStep
    slot = CelebBasisStep.ema_slots(nid, n_chunks)
    src = torch.randn(12, row, generator=g)
    src_row = torch.tensor([(j * 2 + b) % 12 for b in range(3) for j in range(3)], dtype=torch.int32)
    want = table.clone()
    for k, s in enumerate(slot.tolist()):
        if s < 0:
            continue
        i = int(ids.view(-1)[s])
        if 0 <= i < n_rows:
            want[i] = m * want[i] + (1 - m) * src[int(src_row[k])]
    got = table.to(dev)
    ops.ema_rows_sel(got, ids.to(dev), torch.from_numpy(slot).to(dev), src_row.to(dev), src.to(dev), m)
    torch.cuda.synchronize()
    assert (got.cpu() - want).abs().max().item() < 1e-5
    assert torch.equal(got.cpu()[[0, 4, 8]], table[[0, 4, 8]])


# ---------------------------------------------------------------------------------------------------------------------
# Trainer.fit: fused route against the eager route
# ---------------------------------------------------------------------------------------------------------------------
CAPTIONS = {1: "a photo of a face of sks person", 2: "a photo of sks person and ks person",
            3: "a photo of sks and ks and ata together"}


def _cb_batches(n_steps, mix, B=2, id_cnt=4, seed=11):
    """Hand-built CelebBasis batches of `id_cnt` face crops per sample; mix[i][b] = num_ids of sample b at step i."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n_steps):
        image = torch.rand(B, 64, 64, 3, generator=g) * 2 - 1
        faces = torch.rand(B, 64, 64, 3 * id_cnt, generator=g) * 2 - 1
        ids = torch.stack([torch.randperm(10, generator=g)[:id_cnt] for _ in range(B)])
        ids[:, 1] = 3                                  # one identity shared by both samples: the EMA order matters
        nid = torch.tensor(mix[i % len(mix)][:B], dtype=torch.long)
        out.append({"image": image, "caption": [CAPTIONS[int(k)] for k in nid],
                    "image_ori": {"faces": faces, "ids": ids, "num_ids": nid}})
    return out


def _fit(dev, params, batches, fused, setup=None, seed=123):
    from celebbasis_b200 import synth
    from celebbasis_b200.compat import pytorch_lightning as pl
    from celebbasis_b200.step_graph import StepGraphs
    from ldm.models.diffusion.ddpm import LatentDiffusion

    class Rec(pl.Callback):
        def __init__(self):
            self.losses = []

        def on_train_batch_end(self, trainer, module, outputs, batch, batch_idx, dl=0):
            self.losses.append(float(outputs["loss"].item()))

    torch.manual_seed(seed)
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model.fused_step = fused
    model.learning_rate = 5e-3
    model = model.to(dev)
    if not model._textual_inversion():
        model.cond_stage_model.celeb_embeddings = synth.synth_celeb_basis(seed=0).to(dev)
    if setup is not None:
        setup(model)
    rec = Rec()
    captures = []
    orig = StepGraphs.capture

    def counting(self):
        captures.append(self)
        return orig(self)
    StepGraphs.capture = counting
    try:
        torch.manual_seed(7)
        pl.Trainer(gpus="0,", max_steps=len(batches), callbacks=[rec]).fit(model, train_dataloaders=batches)
    finally:
        StepGraphs.capture = orig
    return rec.losses, model, len(captures)


def _cb_params(**weights):
    from celebbasis_b200 import workload
    params = workload.model_params("tiny")
    params["cond_stage_config"]["params"].update(num_hidden_layers=2, device="cuda")
    params.update(weights)
    return params


def _cb_state(model):
    em = model.embedding_manager
    lin = em.meta_id_net.stylegan_mlp.net[0]
    return (lin.weight.detach().float().cpu().clone(), torch.stack([c.float().cpu() for c in em.id_coefficients]),
            torch.stack([e.float().cpu() for e in em.id_embeddings]))


WEIGHTS = dict(l_simple_weight=0.5, original_elbo_weight=1e-2, logvar_init=0.1)


@pytest.mark.parametrize("case", ["weights_B1", "mixed_persons", "mixed_persons_weights", "single_then_mixed"])
def test_trainer_fit_fused_equals_eager_celebbasis(dev, case):
    """single_then_mixed: a run that starts with single-person batches keeps the default launches until its first
    multi-person batch, then captures the multi-person graphs once more; the trained tensors, the EMA state and the
    optimiser state carry over, so the run still matches the eager route."""
    mix = [[1, 1], [1, 1], [2, 3], [1, 1], [3, 2], [2, 2]] if case == "single_then_mixed" else \
        [[1, 2], [3, 1], [2, 3], [1, 1], [3, 2], [2, 2]]
    if case == "weights_B1":
        from celebbasis_b200 import workload
        batches = [workload.synth_batch("tiny", B=1, seed=1234, step=i)[0] for i in range(5)]
    else:
        batches = _cb_batches(6, mix)
    params = _cb_params(**(WEIGHTS if "weights" in case else {}))
    l_f, m_f, n_cap = _fit(dev, params, batches, True)
    l_e, m_e, _ = _fit(dev, params, batches, False)
    assert m_f._fused is not None and m_e._fused is None
    assert n_cap == (2 if case == "single_then_mixed" else 1), n_cap
    assert m_f._fused.eng.multi is None if case == "weights_B1" else m_f._fused.eng.multi is not None
    assert (m_f._fused.eng.loss_weights is not None) == ("weights" in case)
    for a, b in zip(l_f, l_e):
        assert abs(a - b) / abs(b) < 1e-3, (l_f, l_e)
    (w_f, c_f, e_f), (w_e, c_e, e_e) = _cb_state(m_f), _cb_state(m_e)
    print(f"[fused-options] {case}: losses fused {l_f} eager {l_e}; rel(W) {rel(w_f, w_e):.2e} "
          f"rel(coef) {rel(c_f, c_e):.2e} rel(emb) {rel(e_f, e_e):.2e}")
    assert torch.isfinite(w_f).all() and rel(w_f, w_e) < 1e-2
    assert rel(c_f, c_e) < 1e-4 and rel(e_f, e_e) < 1e-4


def _ti_params(weights=True):
    from celebbasis_b200 import workload
    params = workload.ti_model_params("tiny", num_vectors_per_token=2)
    params["cond_stage_config"]["params"].update(num_hidden_layers=2, device="cuda")
    params["personalization_config"]["params"].update(placeholder_strings=["*", "sks"], initializer_words=["person"],
                                                      progressive_words=True)
    params["embedding_reg_weight"] = 1e-2
    if weights:
        params.update(WEIGHTS)
    return params


def _ti_batches(n_steps, B=2, seed=5):
    g = torch.Generator().manual_seed(seed)
    caps = ["a photo of *", "a photo of sks and *", "a sks photo", "* in a photo of sks"]
    return [{"image": torch.rand(B, 64, 64, 3, generator=g) * 2 - 1,
             "caption": [caps[(i + b) % len(caps)] for b in range(B)]} for i in range(n_steps)]


def _progressive_start(model):
    from ldm.modules.embedding_manager import PROGRESSIVE_SCALE
    model.embedding_manager.progressive_counter = PROGRESSIVE_SCALE - 5     # two increments per step: crosses at step 3


@pytest.mark.parametrize("weights", [True, False], ids=["weights", "reg_only"])
def test_trainer_fit_fused_equals_eager_textual_inversion(dev, weights):
    from ldm.modules.embedding_manager import PROGRESSIVE_SCALE
    batches = _ti_batches(6)
    params = _ti_params(weights)
    l_f, m_f, n_cap = _fit(dev, params, batches, True, setup=_progressive_start)
    l_e, m_e, _ = _fit(dev, params, batches, False, setup=_progressive_start)
    assert m_f._fused is not None and m_e._fused is None and n_cap == 1
    eng = m_f._fused.eng
    assert eng.coarse_reg is not None and eng.coarse_reg[1] == 1 and len(eng.coarse_reg[2]) == 1
    em_f, em_e = m_f.embedding_manager, m_e.embedding_manager
    # the counter advanced once per placeholder per step on both routes, past the boundary
    assert em_f.progressive_counter == em_e.progressive_counter == PROGRESSIVE_SCALE - 5 + 2 * len(batches)
    assert np.array_equal(em_f.last_map, em_e.last_map)
    for a, b in zip(l_f, l_e):
        assert abs(a - b) / abs(b) < 1e-3, (l_f, l_e)
    for k in em_f.string_to_param_dict:
        p_f, p_e = em_f.string_to_param_dict[k].detach(), em_e.string_to_param_dict[k].detach()
        print(f"[fused-options] ti {k}: losses fused {l_f} eager {l_e}; rel(rows) {rel(p_f, p_e):.2e}")
        assert torch.isfinite(p_f).all() and rel(p_f, p_e) < 1e-2
    # the logged loss_vlb is the reference's (lvlb_weights[t] * loss_simple).mean() on both routes, default weights included
    b = {"image": batches[0]["image"].to(dev), "caption": batches[0]["caption"]}
    logged = []
    for m in (m_f, m_e):
        torch.manual_seed(9)
        logged.append(m.shared_step(b)[1])
    assert m_f._fused.eng.loss_weights is not None
    vf, ve = float(logged[0]["train/loss_vlb"]), float(logged[1]["train/loss_vlb"])
    assert ve > 0 and abs(vf - ve) / ve < 1e-3, (vf, ve)


# ---------------------------------------------------------------------------------------------------------------------
# the fused route against the unmodified reference (tests/golden/step_options_tiny.pt, oracle/make_golden_options.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def options_gold(golden_dir):
    import os
    return torch.load(os.path.join(golden_dir, "step_options_tiny.pt"), weights_only=False)


def _golden_run(dev, g, make_batch, to_dev, setup, after_step=lambda model: None):
    """shared_step -> backward -> configure_optimizers' AdamW with the reference's draws replayed, on the fused route."""
    from celebbasis_b200 import synth
    from celebbasis_b200.step_graph import StepGraphs
    from ldm.models.diffusion.ddpm import LatentDiffusion
    from oracle import ref_shim
    params = dict(g["params"])
    params["cond_stage_config"] = {**params["cond_stage_config"],
                                   "params": {**params["cond_stage_config"]["params"], "num_hidden_layers": 2,
                                              "device": "cuda"}}
    torch.manual_seed(0)
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model = model.to(dev).train()
    setup(model)
    model.learning_rate = g["lr"]
    opt = model.configure_optimizers()
    captures, orig = [], StepGraphs.capture
    StepGraphs.capture = lambda self: (captures.append(self), orig(self))[1]
    losses = []
    try:
        for s in range(g["steps"]):
            d = g["draws"][s]
            with ref_shim.replay_randomness(d["t"], d["noise"], d["posterior_eps"]):
                loss, _ = model.shared_step(to_dev(make_batch(s)))
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(float(loss))
            after_step(model)
    finally:
        StepGraphs.capture = orig
    assert model._fused is not None and len(captures) == 1
    err = (torch.tensor(losses, dtype=torch.float64) - g["losses"]).abs() / g["losses"].abs()
    assert float(err.max()) <= 1e-3, (losses, g["losses"].tolist())
    return model, float(err.max())


def test_fused_celebbasis_options_vs_reference_golden(dev, options_gold):
    from celebbasis_b200 import synth, workload
    g = options_gold["cb"]
    positions = []

    def setup(model):
        model.cond_stage_model.celeb_embeddings = synth.synth_celeb_basis(seed=0).to(dev)
        em = model.embedding_manager
        em.id_coefficients = [c.clone() for c in g["ema_coef0"]]
        em.id_embeddings = [e.clone() for e in g["ema_emb0"]]

    def to_dev(b):
        io = b["image_ori"]
        return {"image": b["image"].to(dev), "caption": b["caption"],
                "image_ori": {"faces": io["faces"].to(dev), "ids": io["ids"], "num_ids": io["num_ids"]}}

    model, err = _golden_run(dev, g, workload.synth_persons_batch, to_dev, setup,
                             lambda m: positions.append(m.embedding_manager.last_positions))
    em = model.embedding_manager
    assert [[[f.tolist() for f in pos] for pos in step] for step in positions] == g["positions"]
    coef, emb = torch.stack([c.float().cpu() for c in em.id_coefficients]), torch.stack([e.float().cpu() for e in em.id_embeddings])
    W = em.meta_id_net.stylegan_mlp.net[0].weight.detach().float().cpu()
    print(f"[fused-options] cb golden: max |dL|/L {err:.2e} rel(coef) {rel(coef, g['ema_coef']):.2e} "
          f"rel(emb) {rel(emb, g['ema_emb']):.2e} rel(W) {rel(W[::4], g['W_final_rows4']):.2e}")
    assert rel(coef, g["ema_coef"]) < 1e-4 and rel(emb, g["ema_emb"]) < 1e-4
    assert rel(W[::4], g["W_final_rows4"]) < 1e-2


def test_fused_textual_inversion_options_vs_reference_golden(dev, options_gold):
    from celebbasis_b200 import workload
    g = options_gold["ti"]

    def setup(model):
        em = model.embedding_manager
        for k, v in g["params0"].items():
            em.string_to_param_dict[k].data.copy_(v)
        for k, v in g["initial"].items():
            em.initial_embeddings[k].data.copy_(v)
        em.progressive_counter = g["counter0"]

    model, err = _golden_run(dev, g, workload.synth_ti_option_batch,
                             lambda b: {"image": b["image"].to(dev), "caption": b["caption"]}, setup)
    em = model.embedding_manager
    assert em.progressive_counter == g["counters"][-1]
    for k, p in em.string_to_param_dict.items():
        r = rel(p.detach(), g["params_final"][k])
        print(f"[fused-options] ti golden {k}: max |dL|/L {err:.2e} rel(rows) {r:.2e}")
        assert r < 1e-2, (k, r)


def test_fused_options_runs_are_bit_identical(dev):
    batches = _cb_batches(4, [[1, 3], [2, 1], [3, 2], [1, 1]])
    params = _cb_params(**WEIGHTS)
    runs = [_fit(dev, params, batches, True) for _ in range(2)]
    assert runs[0][0] == runs[1][0]
    for x, y in zip(_cb_state(runs[0][1]), _cb_state(runs[1][1])):
        assert torch.equal(x, y)
    ti = [_fit(dev, _ti_params(), _ti_batches(4), True, setup=_progressive_start) for _ in range(2)]
    assert ti[0][0] == ti[1][0]
    for k, p in ti[0][1].embedding_manager.string_to_param_dict.items():
        assert torch.equal(p.detach(), ti[1][1].embedding_manager.string_to_param_dict[k].detach())
