"""Generate tests/golden/step_options_tiny.pt by running the UNMODIFIED reference on the CPU with the training-step options
the fused step accepts besides the defaults.

    python oracle/make_golden_options.py

  * CelebBasis (EmbeddingManagerId) at l_simple_weight 0.5, original_elbo_weight 1e-2, logvar_init 0.1: STEPS x
    (shared_step -> backward -> torch.optim.AdamW) on batch-size-2 batches of 4 face crops whose prompts name 1, 2 or 3
    persons (workload.synth_persons_batch).  Recorded: the draws, the losses and loss_vlb, the trained (W, b), the whole
    identity EMA state (W: every 4th row), and per step the placeholder positions shift_tensor_dim0 returned and the order of the
    _momentum_update calls (sample, person, identity).
  * Textual Inversion (EmbeddingManager) with num_vectors_per_token 2, placeholders '*' (initializer 'person') and 'sks'
    (none), embedding_reg_weight 1e-2, progressive_words with progressive_counter preset 5 below PROGRESSIVE_SCALE, and
    the loss weights above.  Recorded: the draws, the losses, the initial and trained rows, and per step the counter
    and the token ids the manager rewrote in place.
t, noise and the posterior eps are replayed from workload.option_draws (step 0 draws t = 0 and T-1).
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

from celebbasis_b200 import synth, workload
from oracle import ref_shim

GOLD = os.path.join(ROOT, "tests", "golden")
STEPS, LR = 8, 5e-3
WEIGHTS = dict(l_simple_weight=0.5, original_elbo_weight=1e-2, logvar_init=0.1)
COUNTER0 = 2000 - 5


def cb_params():
    p = workload.model_params("tiny")
    p.update(WEIGHTS)
    return p


def ti_params():
    p = workload.ti_model_params("tiny", num_vectors_per_token=2)
    p["personalization_config"]["params"].update(placeholder_strings=["*", "sks"], initializer_words=["person"],
                                                 progressive_words=True)
    p["embedding_reg_weight"] = 1e-2
    p.update(WEIGHTS)
    return p


def _optimizer(model):
    model.learning_rate = LR
    opt = model.configure_optimizers()
    return opt[0] if isinstance(opt, (list, tuple)) else opt


def run_cb():
    torch.manual_seed(0)
    basis = synth.synth_celeb_basis(seed=0)
    model = ref_shim.build_reference(cb_params(), seed=0, clip_layers=workload.clip_layers("tiny"), celeb_basis=basis)
    import ldm.modules.embedding_manager as em_mod
    em = model.embedding_manager
    rec = {"positions": [], "ema": []}
    shift0, mom0 = em_mod.shift_tensor_dim0, em_mod.EmbeddingManagerId._momentum_update

    def shift(ori, r_pos, reps):
        out, fin = shift0(ori, r_pos, reps)
        rec["positions"][-1].append([f.tolist() if hasattr(f, "tolist") else [list(map(int, x)) for x in f] for f in fin])
        return out, fin

    def momentum(self, e, c, id_idx):
        rec["ema"][-1].append(int(id_idx))
        return mom0(self, e, c, id_idx)
    em_mod.shift_tensor_dim0, em_mod.EmbeddingManagerId._momentum_update = shift, momentum
    opt = _optimizer(model)
    lin = em.meta_id_net.stylegan_mlp.net[0]
    ema0 = (torch.stack([c.detach().clone() for c in em.id_coefficients]),
            torch.stack([e.detach().clone() for e in em.id_embeddings]))
    losses, vlbs, draws = [], [], []
    for s in range(STEPS):
        batch, d = workload.synth_persons_batch(s), workload.option_draws(s)
        rec["positions"].append([])
        rec["ema"].append([])
        with ref_shim.replay_randomness(d["t"], d["noise"], d["posterior_eps"]):
            loss, ld = model.shared_step(batch)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
        vlbs.append(float(ld["train/loss_vlb"]))
        draws.append(d)
    em_mod.shift_tensor_dim0, em_mod.EmbeddingManagerId._momentum_update = shift0, mom0
    print(f"[options/cb] losses {losses}")
    return {"params": cb_params(), "steps": STEPS, "lr": LR, "draws": draws,
            "losses": torch.tensor(losses, dtype=torch.float64), "loss_vlb": torch.tensor(vlbs, dtype=torch.float64),
            "W_final_rows4": lin.weight.detach()[::4].clone(), "b_final": lin.bias.detach().clone(),
            "ema_coef0": ema0[0], "ema_emb0": ema0[1],
            "ema_coef": torch.stack([c.detach().clone() for c in em.id_coefficients]),
            "ema_emb": torch.stack([e.detach().clone() for e in em.id_embeddings]),
            "positions": rec["positions"], "ema_order": rec["ema"]}


def run_ti():
    torch.manual_seed(0)
    model = ref_shim.build_reference(ti_params(), seed=0, clip_layers=workload.clip_layers("tiny"))
    em = model.embedding_manager
    em.progressive_counter = COUNTER0
    fwd0 = type(em).forward
    rec = []

    def forward(self, tokenized_text, *a, **k):
        out = fwd0(self, tokenized_text, *a, **k)
        rec.append((self.progressive_counter, tokenized_text.detach().clone()))
        return out
    type(em).forward = forward
    opt = _optimizer(model)
    params0 = {k: v.detach().clone() for k, v in em.string_to_param_dict.items()}
    losses, draws = [], []
    for s in range(STEPS):
        batch, d = workload.synth_ti_option_batch(s), workload.option_draws(s)
        with ref_shim.replay_randomness(d["t"], d["noise"], d["posterior_eps"]):
            loss, _ = model.shared_step(batch)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
        draws.append(d)
    type(em).forward = fwd0
    assert len(rec) == STEPS
    print(f"[options/ti] losses {losses}; counters {[c for c, _ in rec]}")
    return {"params": ti_params(), "steps": STEPS, "lr": LR, "counter0": COUNTER0, "draws": draws,
            "losses": torch.tensor(losses, dtype=torch.float64), "params0": params0,
            "params_final": {k: v.detach().clone() for k, v in em.string_to_param_dict.items()},
            "initial": {k: v.detach().clone() for k, v in em.initial_embeddings.items()},
            "tokens": {k: int(v) for k, v in em.string_to_token_dict.items()},
            "counters": [c for c, _ in rec], "rewritten_ids": torch.stack([t for _, t in rec])}


def main():
    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    out = {"cb": run_cb(), "ti": run_ti()}
    os.makedirs(GOLD, exist_ok=True)
    torch.save(out, os.path.join(GOLD, "step_options_tiny.pt"), _use_new_zipfile_serialization=False)
    print(f"[options] wrote step_options_tiny.pt in {time.time() - t0:.1f}s")


if __name__ == "__main__":
    main()
