"""GPU tests of the Textual Inversion training step (v1-finetune.yaml) on the fused CUDA-graph path:

  * against the UNMODIFIED reference (tests/golden/ti_train_tiny.pt, oracle/make_golden_ti.py): shared_step ->
    backward -> AdamW on batch-size-2 batches of PersonalizedBase, losses point-wise and the trained rows;
  * against the eager per-module path (CB_FUSED_STEP=0) through Trainer.fit, with look-ahead;
  * the step graphs: pipelined == serial, two runs bit-identical;
  * end to end: Trainer.fit over PersonalizedBase writes embeddings_gs-*.pt, a v1-inference model loads it and DDIM
    samples "a photo of *".
"""
import os
import random

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


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ti_train_tiny.pt"), weights_only=False)


def rel(a, b):
    a, b = a.float().cpu().flatten(), b.float().cpu().flatten()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cos(a, b):
    a, b = a.float().cpu().flatten(), b.float().cpu().flatten()
    return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-30))


def _model(dev, fused=True, seed=123):
    from celebbasis_b200 import synth, workload
    from ldm.models.diffusion.ddpm import LatentDiffusion
    torch.manual_seed(seed)
    params = workload.ti_model_params("tiny")
    params["cond_stage_config"]["params"].update(num_hidden_layers=2, device="cuda")
    model = LatentDiffusion(**params)
    model.load_state_dict(synth.synth_state_dict(model, seed=0), strict=False)
    model.fused_step = fused
    model.learning_rate = 5e-3
    return model.to(dev).train()


def _batches(tmp_path, gold, n_steps, B=2, seed=None):
    """Batch-size-B batches of the mirror's PersonalizedBase over the fixture's synthetic photos (its file order)."""
    from celebbasis_b200 import workload
    from ldm.data.personalized import PersonalizedBase
    root = str(tmp_path / "photos")
    workload.synth_photo_files(root, seed=gold["photo_seed"])
    tr = gold["train"]
    s = tr["seed"] if seed is None else seed
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)
    ds = PersonalizedBase(root, size=tr["size"], repeats=100, interpolation="bicubic", flip_p=0.5)
    ds.image_paths = [os.path.join(root, f) for f in gold["files"]]
    return [torch.utils.data.default_collate([ds[k * B + j] for j in range(B)]) for k in range(n_steps)]


def _to_dev(batch, dev):
    return {"image": batch["image"].to(dev), "caption": list(batch["caption"])}


# ---------------------------------------------------------------------------------------------------------------------
def test_ti_loss_curve_vs_reference_golden(dev, gold, tmp_path):
    """shared_step -> backward -> AdamW (configure_optimizers) on the fused path, with the reference's t / noise /
    posterior eps replayed: point-wise |dL|/L <= 1e-3 and the trained rows' update along the reference's."""
    from oracle import ref_shim
    tr = gold["train"]
    batches = _batches(tmp_path, gold, tr["steps"], tr["B"])
    assert [list(b["caption"]) for b in batches] == [list(c) for c in tr["captions"]]
    model = _model(dev)
    em = model.embedding_manager
    assert {k: int(v) for k, v in em.string_to_token_dict.items()} == tr["tokens"]
    for k, v in tr["params0"].items():
        em.string_to_param_dict[k].data.copy_(v)
    model.learning_rate = tr["lr"]
    opt = model.configure_optimizers()
    losses = []
    for b, d in zip(batches, tr["draws"]):
        with ref_shim.replay_randomness(d["t"], d["noise"], d["posterior_eps"]):
            loss, _ = model.shared_step(_to_dev(b, dev))
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert model._fused is not None and model._fused.g_pipe is not None
    losses = torch.tensor(losses, dtype=torch.float64)
    err = (losses - tr["losses"]).abs() / tr["losses"].abs()
    assert float(err.max()) <= 1e-3, (float(err.max()), losses.tolist(), tr["losses"].tolist())
    for k, p in em.string_to_param_dict.items():
        upd, upd_ref = p.detach().cpu() - tr["params0"][k], tr["params_final"][k] - tr["params0"][k]
        c, r = cos(upd, upd_ref), rel(p, tr["params_final"][k])
        print(f"[ti-golden] {k}: max |dL|/L {float(err.max()):.2e}  cos(update) {c:.5f}  rel(rows) {r:.2e}")
        # measured on an H100 80GB HBM3 at 700 W: max |dL|/L 4.4e-4, cos(update) 0.99995, rel(rows) 7.5e-3 (AdamW moves
        # every element by ~lr per step whatever its gradient's size, so elements with round-off sized gradients drift)
        assert c > 0.999 and r < 1e-2, (c, r)


def test_ti_trainer_fit_fused_equals_eager(dev, gold, tmp_path):
    """Trainer.fit on the fused path (look-ahead front end, G_pipe) gives the eager path's losses and trained rows, and
    the placeholder parameters alias the engine's flat buffer."""
    from celebbasis_b200.compat import pytorch_lightning as pl
    batches = _batches(tmp_path, gold, 5)

    class Rec(pl.Callback):
        def __init__(self):
            self.losses = []

        def on_train_batch_end(self, trainer, module, outputs, batch, batch_idx, dl=0):
            self.losses.append(float(outputs["loss"].item()))

    def fit(fused):
        model = _model(dev, fused)
        rec = Rec()
        torch.manual_seed(7)
        pl.Trainer(gpus="0,", max_steps=len(batches), callbacks=[rec]).fit(model, train_dataloaders=batches)
        p = model.embedding_manager.string_to_param_dict["*"]
        return rec.losses, p.detach().float().cpu().clone(), model
    l_f, p_f, m_f = fit(True)
    l_e, p_e, m_e = fit(False)
    assert m_f._fused is not None and m_e._fused is None
    G = m_f._fused
    assert G.g_pipe is not None and G.faces_n is None and G.v is None
    assert m_f.embedding_manager.string_to_param_dict["*"].data_ptr() == G.eng.flat.data_ptr()
    for a, b in zip(l_f, l_e):
        assert abs(a - b) / abs(b) < 1e-3, (l_f, l_e)
    p0 = _model(dev, seed=123).embedding_manager.string_to_param_dict["*"].detach().cpu()
    print(f"[ti-eager] losses fused {l_f} eager {l_e}; rel(rows) {rel(p_f, p_e):.2e} cos(update) {cos(p_f - p0, p_e - p0):.5f}")
    assert torch.isfinite(p_f).all() and rel(p_f, p_e) < 1e-2
    assert cos(p_f - p0, p_e - p0) > 0.98


def _engine_stream(dev, gold, tmp_path, n=4):
    from celebbasis_b200.step_graph import StepGraphs
    from celebbasis_b200.train_step import TextualInversionStep
    model = _model(dev)
    em = model.embedding_manager
    eng = TextualInversionStep(model._engine_params, model.state_dict(), [p.detach() for p in model._ti_params()], dev,
                               tokenizer=model.cond_stage_model.tokenizer)
    G = StepGraphs(eng, B=2, T=77, n_chunks=0, image_hw=64)
    g = torch.Generator().manual_seed(17)
    stream = []
    for b in _batches(tmp_path, gold, n):
        ids = eng.tokenize(list(b["caption"]))
        map_np, _ = em.ti_map(ids.numpy())
        stream.append((b["image"], ids, map_np, torch.randint(0, 1000, (2,), generator=g),
                       torch.randn(2, 4, 8, 8, generator=g), torch.randn(2, 4, 8, 8, generator=g)))
    img, ids, mp, t, noise, peps = stream[0]
    G.load_next(img, None, peps)
    G.load_step(ids, mp, t, noise)
    G.capture()
    return eng, G, stream


def test_ti_step_graphs_pipelined_equals_serial_and_reproducible(dev, gold, tmp_path):
    eng, G, stream = _engine_stream(dev, gold, tmp_path)
    assert G.g_pipe is not None and G.launches["pipe"] == G.launches["pre"] + G.launches["main"]

    def run(pipelined):
        # a graph's outputs live in the graphs' shared memory pool: read them before the next replay
        out = []
        G.load_next(stream[0][0], None, stream[0][5])
        G.prefetch()
        for i, (img, ids, mp, t, noise, peps) in enumerate(stream):
            G.load_step(ids, mp, t, noise)
            nxt = stream[i + 1] if i + 1 < len(stream) else None
            if pipelined and nxt is not None:
                G.load_next(nxt[0], None, nxt[5])
                out.append((G.step(lookahead=True).clone(), eng.grad.clone(), G.z.clone()))
            else:
                out.append((G.step(lookahead=False).clone(), eng.grad.clone(), G.z.clone()))
                if nxt is not None:
                    G.load_next(nxt[0], None, nxt[5])
                    G.prefetch()
        return out
    ser, pip, pip2 = run(False), run(True), run(True)
    for (ls, gs, zs), (lp, gp, zp) in zip(ser, pip):
        assert rel(zp, zs) < 2e-3
        assert abs(ls.item() - lp.item()) / abs(ls.item()) < 1e-3
        assert cos(gp, gs) > 0.99
    for a, b in zip(pip, pip2):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    # the gradient is the placeholder rows' gradient summed over both prompts of the batch
    assert float(eng.grad.abs().sum()) > 0 and torch.isfinite(eng.grad).all()


def test_ti_end_to_end_train_save_load_sample(dev, gold, tmp_path):
    """Trainer.fit over PersonalizedBase (DataLoader, batch size 2) writes embeddings_gs-*.pt; a v1-inference model loads
    it (EmbeddingManager.load) and DDIM samples "a photo of *" into finite images."""
    from celebbasis_b200 import workload
    from celebbasis_b200.compat import pytorch_lightning as pl
    from celebbasis_b200.compat.pytorch_lightning.callbacks import ModelCheckpoint
    from ldm.data.personalized import PersonalizedBase
    from ldm.models.diffusion.ddim import DDIMSampler
    root = str(tmp_path / "photos")
    workload.synth_photo_files(root, seed=0)
    ds = PersonalizedBase(root, size=64, repeats=10, set="train", placeholder_token="*")
    loader = torch.utils.data.DataLoader(ds, batch_size=2, shuffle=True, num_workers=0, drop_last=True)
    model = _model(dev)
    ckdir = str(tmp_path / "ckpt")
    ck = ModelCheckpoint(dirpath=ckdir, every_n_train_steps=3, save_weights_only=True)
    torch.manual_seed(5)
    pl.Trainer(gpus="0,", max_steps=3, callbacks=[ck], default_root_dir=str(tmp_path)).fit(model, train_dataloaders=loader)
    assert model._fused is not None
    files = [f for f in os.listdir(ckdir) if f.startswith("embeddings_gs-")]
    assert files, os.listdir(ckdir)
    trained = model.embedding_manager.string_to_param_dict["*"].detach().cpu().clone()
    inf = _model(dev, seed=9).eval()
    inf.embedding_manager.load(os.path.join(ckdir, sorted(files)[-1]))
    inf = inf.to(dev)
    assert torch.equal(inf.embedding_manager.string_to_param_dict["*"].detach().cpu(), trained)
    with torch.no_grad():
        uc = inf.get_learned_conditioning([""])
        c = inf.get_learned_conditioning(["a photo of *"])
        samples, _ = DDIMSampler(inf).sample(S=4, conditioning=c, batch_size=1, shape=[4, 8, 8], verbose=False,
                                             unconditional_guidance_scale=5.0, unconditional_conditioning=uc, eta=0.0)
        img = inf.decode_first_stage(samples)
    assert img.shape == (1, 3, 64, 64) and torch.isfinite(img).all()
