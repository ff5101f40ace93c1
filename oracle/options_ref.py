"""fp32 port (plain PyTorch, CPU or GPU) of the training-step options beyond the defaults, on torch_ref's modules:
p_losses with l_simple_weight / logvar / original_elbo_weight (ddpm.py:1084-1099), two- and three-person CelebBasis
prompts with the identity EMA in the reference's order (embedding_manager.py:279-392,483-489), and the Textual Inversion
manager with several vectors per token, progressive words and the coarse regulariser (embedding_manager.py:97-151,170-180,
ddpm.py:1101-1107).  Pinned against tests/golden/step_options_tiny.pt (oracle/make_golden_options.py)."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import torch_ref

PROGRESSIVE_SCALE = 2000


def lvlb_weights(timesteps, linear_start, linear_end):
    """ddpm.py:126-178 (linear schedule, v_posterior 0, eps parameterisation): fp64 host schedule, fp32 buffers."""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
    alphas = 1. - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1., ac[:-1])
    pv = betas * (1. - ac_prev) / (1. - ac)
    f = lambda a: torch.tensor(a, dtype=torch.float32)
    w = f(betas) ** 2 / (2 * f(pv) * f(alphas) * (1 - f(ac)))
    w[0] = w[1]
    return w


def weighted_loss(eps, noise, t, logvar, lvlb, l_simple_weight, original_elbo_weight):
    """Returns (loss, loss_vlb, loss_simple)."""
    loss_simple = ((eps - noise) ** 2).mean(dim=[1, 2, 3])
    lv = logvar[t]
    loss = l_simple_weight * (loss_simple / torch.exp(lv) + lv).mean()
    vlb = (lvlb[t] * loss_simple).mean()
    return loss + original_elbo_weight * vlb, vlb, loss_simple


def _front(om, batch, draws):
    x = batch["image"].permute(0, 3, 1, 2).contiguous().float()
    with torch.no_grad():
        z = torch_ref.posterior_sample(om.first_stage_model(x), draws["posterior_eps"], om.scale_factor)
    return z


def _unet_loss(om, z, context, draws, logvar, lvlb, weights):
    t, noise = draws["t"], draws["noise"]
    x_noisy = torch_ref.q_sample(om.sched, z, t, noise)
    eps = om.model.diffusion_model(x_noisy, t, context)
    return weighted_loss(eps, noise, t, logvar, lvlb, *weights)


def persons(om, batch, basis, W, b):
    """The per-person rows and coefficients (embedding_manager.py:296-304): metas[j] (B, es, D) and cefs[j] (B, es, 1, K)
    of the first, second and third person: face chunks 0, 1, id_cnt // 2 (coefficients 0, 1, 1)."""
    faces, ids = batch["image_ori"]["faces"], batch["image_ori"]["ids"]
    B, n_id = ids.shape
    with torch.no_grad():
        mnet = om.embedding_manager.meta_id_net
        mnet.id_model.eval()
        cat = torch.cat(faces.chunk(n_id, -1), 0)
        v = F.normalize(mnet.id_model(torch_ref.face_preprocess(cat)), dim=-1, p=2)
    coef = torch_ref.celeb_mlp(v, W, b)
    zc = torch_ref.celeb_basis(coef, basis)
    meta, cef = zc.view(n_id, B, *zc.shape[1:]), coef.view(n_id, B, *coef.shape[1:])
    return [meta[0], meta[1], meta[n_id // 2]], [cef[0], cef[1], cef[1]]


def inject_persons(token_ids, tok_emb, metas, num_ids, ph_tokens, reps):
    """embedding_manager.py:321-392: sample b's j-th placeholder gets metas[j][b]; returns (emb, positions)."""
    out, positions = [], []
    for b in range(tok_emb.shape[0]):
        k = int(num_ids[b])
        pos = torch_ref.get_rep_pos(np.asarray(token_ids[b]), ph_tokens[:k])
        src, fin = torch_ref.shift_index_map(tok_emb.shape[1], pos, reps)
        rows = list(tok_emb[b][torch.as_tensor(src)].unbind(0))
        for j in range(k):
            for one_pos in fin[j]:
                for r, p in enumerate(one_pos):
                    rows[int(p)] = metas[j][b][r]
        out.append(torch.stack(rows, 0))
        positions.append([f.tolist() for f in fin])
    return torch.stack(out, 0), positions


def ema_persons(ema_coef, ema_emb, ids, num_ids, metas, cefs, momentum):
    """_momentum_update of every person in the reference's order (per sample, then person); returns the identity order."""
    order = []
    for b in range(ids.shape[0]):
        for j in range(int(num_ids[b])):
            i = int(ids[b][j])
            order.append(i)
            if i < ema_emb.shape[0]:
                ema_emb[i] = momentum * ema_emb[i] + (1 - momentum) * metas[j][b].detach()
                ema_coef[i] = momentum * ema_coef[i] + (1 - momentum) * cefs[j][b].detach()
    return order


def cb_step(om, batch, draws, token_ids, basis, ph_tokens, logvar, lvlb, weights, ema_coef, ema_emb, momentum):
    """shared_step of a CelebBasis batch with 1/2/3-person prompts; updates the EMA tables in place."""
    W, b = om.trainable()
    z = _front(om, batch, draws)
    metas, cefs = persons(om, batch, basis, W, b)
    io = batch["image_ori"]
    order = ema_persons(ema_coef, ema_emb, io["ids"], io["num_ids"], metas, cefs, momentum)
    tm = om.cond_stage_model.transformer.text_model
    emb, positions = inject_persons(token_ids, tm.embed_tokens(token_ids), metas, io["num_ids"], ph_tokens,
                                    metas[0].shape[1])
    loss, vlb, _ = _unet_loss(om, z, tm.forward_embeds(emb), draws, logvar, lvlb, weights)
    return loss, vlb, positions, order


def ti_inject(token_ids, tok_emb, placeholders, progressive, counter):
    """EmbeddingManager.forward with several vectors per token (embedding_manager.py:108-151).  placeholders: [(token,
    (nv, D) parameter)] in the dict's order.  Returns (emb, rewritten token ids, counter)."""
    ids, emb = token_ids.clone(), tok_emb.clone()
    n = ids.shape[1]
    for ptoken, P in placeholders:
        if progressive:
            counter += 1
            steps = 1 + counter // PROGRESSIVE_SCALE
        else:
            steps = P.shape[0]
        nv = min(P.shape[0], steps)
        rows, cols = torch.where(ids == ptoken)
        if rows.numel() == 0:
            continue
        sc, si = torch.sort(cols, descending=True)
        for row, col in zip(rows[si].tolist(), sc.tolist()):
            ids[row] = torch.cat([ids[row][:col], torch.full((nv,), ptoken, dtype=ids.dtype), ids[row][col + 1:]])[:n]
            emb[row] = torch.cat([emb[row][:col], P[:nv], emb[row][col + 1:]], 0)[:n]
    return emb, ids, counter


def coarse_reg(placeholders, initial):
    """embedding_to_coarse_loss().mean(): sum over the placeholders with an initializer of (P-P0)(P-P0)^T / n."""
    loss = 0.
    for key, P in placeholders.items():
        if key in initial:
            d = P - initial[key]
            loss = loss + d @ d.T / len(initial)
    return loss.mean()


def ti_step(om, batch, draws, token_ids, tokens, params, initial, progressive, counter, logvar, lvlb, weights, reg_w):
    """shared_step of a Textual Inversion batch; returns (loss, rewritten ids, counter)."""
    z = _front(om, batch, draws)
    tm = om.cond_stage_model.transformer.text_model
    emb, ids, counter = ti_inject(token_ids, tm.embed_tokens(token_ids), [(tokens[k], params[k]) for k in params],
                                  progressive, counter)
    loss, _, _ = _unet_loss(om, z, tm.forward_embeds(emb), draws, logvar, lvlb, weights)
    return loss + reg_w * coarse_reg(params, initial), ids, counter
