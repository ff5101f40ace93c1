"""Host mirror of ldm/modules/embedding_manager.py:187-532 (EmbeddingManagerId).

Same constructor keywords, attributes (`string_to_token_dict`, `id_coefficients`, `id_embeddings`, `meta_id_net`,
`test_mode`), `forward(tokenized_text, embedded_text, face_image, img_ori, celeb_embeddings)` contract and
`save/load` file format as the reference.  The per-sample Python loop of in-place row writes becomes one gather
kernel driven by an integer row map computed on the host with the bit-exact mirror of helpers.py.
"""
from functools import partial

import numpy as np
import torch
from torch import nn

from celebbasis_b200 import ops
from celebbasis_b200.train_step import build_inject_map_multi
from ldm.modules.id_embedding.meta_net import MetaIdNet


def get_clip_token_for_string(tokenizer, string):
    batch_encoding = tokenizer(string, truncation=True, max_length=77, return_length=True,
                               return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
    tokens = batch_encoding["input_ids"]
    assert torch.count_nonzero(tokens - 49407) == 2, \
        f"String '{string}' maps to more than a single token. Please use another string"
    return tokens[0, 1]


def get_embedding_for_clip_token(embedder, token):
    return embedder(token.unsqueeze(0))[0, 0]


class _InjectFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tok_emb, z_rows, map_dev, zero_pos):
        B, T, D = tok_emb.shape
        out = ops.embed_inject_fwd(tok_emb.reshape(B * T, D).float().contiguous(), z_rows.float().contiguous(),
                                   map_dev.view(-1), zero_pos, B, T)
        ctx.save_for_backward(map_dev)
        ctx.dims = (B, T, D, z_rows.shape[0])
        return out.view(B, T, D)

    @staticmethod
    def backward(ctx, dout):
        (map_dev,) = ctx.saved_tensors
        B, T, D, R = ctx.dims
        dz = ops.embed_inject_bwd(dout.reshape(B * T, D).float().contiguous(), map_dev.view(-1), R, B, T)
        return None, dz, None, None


class EmbeddingManagerId(nn.Module):
    def __init__(self, embedder, placeholder_strings=None, initializer_words=None, max_ids: int = 10,
                 num_embeds_per_token=1, momentum: float = 0.9, meta_mlp_depth: int = 2, loss_type: str = None,
                 meta_inner_dim: int = 512, meta_heads: int = 1, use_rm_mlp: bool = False,
                 test_mode: str = 'coefficient', save_fp16: bool = True, **kwargs):
        super().__init__()
        self.string_to_token_dict = {}
        self.placeholder_strings = list(placeholder_strings)
        self.max_ids = max_ids
        self.num_es = num_embeds_per_token
        self.meta_heads = meta_heads
        self.use_rm_mlp = use_rm_mlp
        assert hasattr(embedder, 'tokenizer'), "the CelebBasis path uses the CLIP text encoder"
        self.is_clip = True
        get_token_for_string = partial(get_clip_token_for_string, embedder.tokenizer)
        token_dim = 768
        self.id_embeddings = [torch.zeros(num_embeds_per_token, token_dim)] * self.max_ids
        self.id_coefficients = [torch.randn(num_embeds_per_token, meta_heads, meta_inner_dim)] * self.max_ids
        self.celeb_embeddings = None
        for placeholder_string in self.placeholder_strings:
            self.string_to_token_dict[placeholder_string] = get_token_for_string(placeholder_string)
        if initializer_words:
            tok = get_token_for_string(initializer_words[0])
            with torch.no_grad():
                init = embedder.transformer.text_model.embeddings.token_embedding.weight[int(tok)].detach().cpu().clone()
            for idx in range(self.max_ids):
                self.id_embeddings[idx] = init.unsqueeze(0).repeat(self.num_es * self.meta_heads, 1)
        else:
            for idx in range(self.max_ids):
                self.id_embeddings[idx] = torch.rand(self.num_es * self.meta_heads, token_dim)
        self.meta_id_net = MetaIdNet(use_expert=False, mlp_depth=meta_mlp_depth, use_header=False,
                                     inner_dim=meta_inner_dim, meta_dim=token_dim, use_celebs=True,
                                     num_embeds_per_token=self.num_es, heads=self.meta_heads, use_rm_mlp=use_rm_mlp)
        self.momentum = momentum
        self.id_neg_loss = 0.
        self.moved_to_device = False
        self.loss_type = loss_type
        assert loss_type in (None, 'none'), "aigc_id.yaml: loss_type 'none' (other heads are never executed)"
        self.test_mode = test_mode
        assert self.test_mode in ['coefficient', 'embedding', 'image']
        self.save_fp16 = save_fp16
        self._zero_pos = None
        self.last_positions = None

    # ---- forward -------------------------------------------------------------------------------------------
    def forward(self, tokenized_text, embedded_text, face_image=None, img_ori=None, celeb_embeddings=None):
        b, n = tokenized_text.shape
        device = embedded_text.device
        self.celeb_embeddings = celeb_embeddings.to(device)
        if img_ori is None:
            return embedded_text
        faces, ids, num_ids = img_ori["faces"], img_ori["ids"], img_ori["num_ids"]
        ids_host = np.asarray(ids.cpu() if isinstance(ids, torch.Tensor) else ids)
        nid_host = np.asarray(num_ids.cpu() if isinstance(num_ids, torch.Tensor) else num_ids).astype(np.int64)
        self._embedding_to_device(device)
        if self.training or (faces is not None and self.test_mode == 'image'):
            meta, _, cef = self.meta_id_net.forward_multi_faces(faces.to(device), torch.as_tensor(ids_host),
                                                                self.celeb_embeddings)
            metas = [meta[0], meta[1] if len(meta) > 1 else meta[0], meta[ids_host.shape[1] // 2]]
            cefs = [cef[0], cef[1] if len(cef) > 1 else cef[0], cef[1] if len(cef) > 1 else cef[0]]
        else:
            metas = cefs = None
            print(f'[Embedding Manager] test_mode: {self.test_mode}')
        z_list, per_sample, base = [], [], 0
        for b_idx in range(b):
            k = int(nid_host[b_idx])
            assert k in (1, 2, 3)
            toks, bases = [], []
            for j in range(k):
                pred_e = metas[j][b_idx] if metas is not None else None
                pred_c = cefs[j][b_idx] if cefs is not None else None
                memo = self._momentum_update(pred_e, pred_c, int(ids_host[b_idx][j]))
                z_list.append(memo.to(device))
                toks.append(int(self.string_to_token_dict[self.placeholder_strings[j]]))
                bases.append(base)
                base += self.num_es * self.meta_heads
            per_sample.append((toks, bases))
        tok_host = tokenized_text.detach().cpu().numpy()
        map_np, positions = build_inject_map_multi(tok_host, per_sample, self.num_es * self.meta_heads)
        self.last_positions = positions
        map_dev = torch.from_numpy(map_np).to(device)
        z_rows = torch.cat(z_list, 0)
        if self._zero_pos is None or self._zero_pos.device != device or self._zero_pos.shape[0] < n:
            self._zero_pos = torch.zeros(n, embedded_text.shape[-1], dtype=torch.float32, device=device)
        return _InjectFn.apply(embedded_text, z_rows, map_dev, self._zero_pos)

    # ---- side state ------------------------------------------------------------------------------------------
    def _momentum_update(self, one_pred_embedding, one_pred_coefficient, id_idx: int):
        if not self.training:
            if self.test_mode == 'coefficient':
                if self.celeb_embeddings is None or self.id_coefficients is None:
                    print('[Warning] celeb_embeddings is None or id_coefficients is None.')
                    return one_pred_embedding.float()
                x = self.id_coefficients[id_idx].to(self.celeb_embeddings.device).float()       # (es,h,inner)
                z = ops.celeb_basis_fwd(x.reshape(1, x.shape[0], -1).contiguous(), self.celeb_embeddings.float().contiguous())
                return z[0]
            elif self.test_mode == 'embedding':
                return self.id_embeddings[id_idx].float()
            return one_pred_embedding.float()
        if id_idx < len(self.id_embeddings):
            m = self.momentum
            with torch.no_grad():
                e_old = self.id_embeddings[id_idx].to(one_pred_embedding.device).float().contiguous()
                c_old = self.id_coefficients[id_idx].to(one_pred_embedding.device).float().contiguous()
                self.id_embeddings[id_idx] = ops.axpby(e_old, m, one_pred_embedding.detach().contiguous(), 1.0 - m)
                pc = one_pred_coefficient.detach().reshape(c_old.shape[0], -1).contiguous()
                self.id_coefficients[id_idx] = ops.axpby(c_old.view(c_old.shape[0], -1), m, pc, 1.0 - m).view(c_old.shape)
        return one_pred_embedding

    def _embedding_to_device(self, device):
        if self.moved_to_device:
            return
        # a checkpoint written in test_mode 'coefficient' carries no id_embeddings (load() leaves None), and vice versa
        if self.id_embeddings is not None:
            self.id_embeddings = [x.to(device) for x in self.id_embeddings]
        if self.id_coefficients is not None:
            self.id_coefficients = [x.to(device) for x in self.id_coefficients]
        self.moved_to_device = True

    # ---- checkpoint format (embedding_manager.py:396-426) -------------------------------------------------------
    def save(self, ckpt_path):
        save_dict = {}
        cast = (lambda x: x.detach().cpu().half()) if self.save_fp16 else (lambda x: x.detach().cpu())
        if self.test_mode == 'coefficient':
            save_dict["id_coefficients"] = [cast(x) for x in self.id_coefficients]
        if self.test_mode == 'embedding':
            save_dict["id_embeddings"] = [cast(x) for x in self.id_embeddings]
        if self.test_mode == 'image':
            save_dict["meta_id_net"] = self.meta_id_net.trainable_state_dict(verbose=True)
        torch.save(save_dict, ckpt_path)

    def load(self, ckpt_path):
        ckpt = torch.load(ckpt_path, map_location='cpu')
        self.id_coefficients = ckpt.get("id_coefficients")
        self.id_embeddings = ckpt.get("id_embeddings")
        if self.id_coefficients is not None:
            self.id_coefficients = [x.float() for x in self.id_coefficients]
        if self.id_embeddings is not None:
            self.id_embeddings = [x.float() for x in self.id_embeddings]
        if ckpt.get("meta_id_net") is not None:
            self.meta_id_net.load_trainable_state_dict(ckpt["meta_id_net"], verbose=True)
            self.meta_id_net.eval()
        self.moved_to_device = False
        print('[Embedding Manager] weights loaded.')

    def embedding_parameters(self):
        return []

    def trainable_parameters(self):
        return list(self.meta_id_net.parameters())

    def embedding_to_coarse_loss(self):
        return 0.

    def embedding_neg_loss(self):
        return self.id_neg_loss


# =====================================================================================================================
# vanilla Textual-Inversion manager (embedding_manager.py:38-184; configs/stable-diffusion/v1-finetune.yaml:23-30)
# =====================================================================================================================
DEFAULT_PLACEHOLDER_TOKEN = ["*"]
PROGRESSIVE_SCALE = 2000


def build_ti_map(tokens, placeholders, max_vectors_per_token, n_active):
    """Host mirror of EmbeddingManager.forward's index arithmetic (embedding_manager.py:108-151) as a gather map.

    tokens: (B, n) int64 host array; placeholders: [(token id, z_row_base, rows of that placeholder's parameter)] in the
    dict's insertion order; max_vectors_per_token / n_active as in the reference (n_active = max_step_tokens).
    Returns (map (B, n) int32: >= 0 original row of the same prompt, < 0: z row -(m+1)), new_tokens).  One vector per
    token: every occurrence is replaced in place.  Several vectors: occurrences are expanded right-to-left, later tokens
    shift right and the row is truncated to n -- and the token row is rewritten with the repeated placeholder id, which a
    later placeholder's search sees, exactly like the reference's in-place update."""
    tok = np.array(tokens, dtype=np.int64, copy=True)
    B, n = tok.shape
    src = np.tile(np.arange(n, dtype=np.int64), (B, 1))
    for ptoken, base, rows in placeholders:
        if max_vectors_per_token == 1:
            hit = tok == int(ptoken)
            src[hit] = -(int(base) + 1)
            continue
        nv = min(int(rows), int(n_active))
        r_idx, c_idx = np.where(tok == int(ptoken))
        if r_idx.size == 0:
            continue
        order = np.argsort(-c_idx, kind="stable")
        for k in order:
            row, col = int(r_idx[k]), int(c_idx[k])
            tok[row] = np.concatenate([tok[row][:col], np.full(nv, int(ptoken), dtype=np.int64), tok[row][col + 1:]])[:n]
            zrows = -(int(base) + np.arange(nv, dtype=np.int64) + 1)
            src[row] = np.concatenate([src[row][:col], zrows, src[row][col + 1:]])[:n]
    return src.astype(np.int32), tok


class EmbeddingManager(nn.Module):
    """Textual Inversion: one learnable (num_vectors_per_token, 768) embedding per placeholder string, written over /
    inserted at the placeholder's position(s) of the token embeddings.  Same constructor keywords, attributes
    (`string_to_token_dict`, `string_to_param_dict`, `initial_embeddings`), `forward` contract and `save/load` file format
    as the reference; the row writes are the same gather kernel EmbeddingManagerId uses (cb_embed_inject_fwd/bwd)."""

    def __init__(self, embedder, placeholder_strings=None, initializer_words=None, per_image_tokens=False,
                 num_vectors_per_token=1, progressive_words=False, **kwargs):
        super().__init__()
        self.string_to_token_dict = {}
        self.string_to_param_dict = nn.ParameterDict()
        self.initial_embeddings = nn.ParameterDict()          # these are not optimised
        self.progressive_words = progressive_words
        self.progressive_counter = 0
        self.max_vectors_per_token = num_vectors_per_token
        assert hasattr(embedder, 'tokenizer'), "the SD-v1 path uses the CLIP text encoder (the BERT branch is LDM-only)"
        self.is_clip = True
        assert not per_image_tokens, "per_image_tokens is false in v1-finetune.yaml (ldm/data/personalized.py list)"
        placeholder_strings = list(placeholder_strings or DEFAULT_PLACEHOLDER_TOKEN)
        table = embedder.transformer.text_model.embeddings.token_embedding.weight
        token_dim = table.shape[1]
        for idx, placeholder_string in enumerate(placeholder_strings):
            token = get_clip_token_for_string(embedder.tokenizer, placeholder_string)
            if initializer_words and idx < len(initializer_words):
                init_tok = get_clip_token_for_string(embedder.tokenizer, initializer_words[idx])
                with torch.no_grad():
                    init = table[int(init_tok)].detach().float().cpu().clone()
                token_params = torch.nn.Parameter(init.unsqueeze(0).repeat(num_vectors_per_token, 1), requires_grad=True)
                self.initial_embeddings[placeholder_string] = torch.nn.Parameter(
                    init.unsqueeze(0).repeat(num_vectors_per_token, 1), requires_grad=False)
            else:
                token_params = torch.nn.Parameter(torch.rand(size=(num_vectors_per_token, token_dim), requires_grad=True))
            self.string_to_token_dict[placeholder_string] = token
            self.string_to_param_dict[placeholder_string] = token_params
        self._zero_pos = None
        self.last_map = None

    def ti_map(self, tok_host):
        """The inject map of (B, n) host token ids: (map (B, n) int32 over the original rows / -(z row + 1), rewritten
        token ids).  z rows are the placeholders' parameters concatenated in the dict's order."""
        b, n = tok_host.shape
        placeholders, base, steps = [], 0, []
        for key, ptoken in self.string_to_token_dict.items():
            p = self.string_to_param_dict[key]
            if self.max_vectors_per_token > 1 and self.progressive_words:
                self.progressive_counter += 1
                steps.append(1 + self.progressive_counter // PROGRESSIVE_SCALE)
            else:
                steps.append(self.max_vectors_per_token)
            placeholders.append((int(ptoken), base, p.shape[0]))
            base += p.shape[0]
        # per-placeholder active length: apply them one at a time so each sees its own max_step_tokens
        cur_tok = tok_host
        maps = np.tile(np.arange(n, dtype=np.int32), (b, 1))
        for (ph, st) in zip(placeholders, steps):
            m, cur_tok = build_ti_map(cur_tok, [ph], self.max_vectors_per_token, st)
            # compose: rows of `m` index the CURRENT row order
            sel = m >= 0
            new = np.where(sel, np.take_along_axis(maps, np.clip(m, 0, n - 1), axis=1), m)
            maps = new.astype(np.int32)
        return maps, cur_tok

    def forward(self, tokenized_text, embedded_text, face_image=None, img_ori=None, celeb_embeddings=None):
        b, n = tokenized_text.shape
        device = embedded_text.device
        maps, cur_tok = self.ti_map(tokenized_text.detach().cpu().numpy())
        if self.max_vectors_per_token > 1:
            tokenized_text.copy_(torch.from_numpy(cur_tok).to(tokenized_text.device))     # in-place, like the reference
        self.last_map = maps
        map_dev = torch.from_numpy(maps).to(device)
        z_rows = torch.cat([self.string_to_param_dict[k].to(device) for k in self.string_to_token_dict], 0).float()
        if self._zero_pos is None or self._zero_pos.device != device or self._zero_pos.shape[0] < n:
            self._zero_pos = torch.zeros(n, embedded_text.shape[-1], dtype=torch.float32, device=device)
        return _InjectFn.apply(embedded_text, z_rows, map_dev, self._zero_pos)

    def save(self, ckpt_path):
        torch.save({"string_to_token": self.string_to_token_dict, "string_to_param": self.string_to_param_dict}, ckpt_path)

    def load(self, ckpt_path):
        ckpt = torch.load(ckpt_path, map_location='cpu', weights_only=False)
        self.string_to_token_dict = ckpt["string_to_token"]
        self.string_to_param_dict = ckpt["string_to_param"]

    def get_embedding_norms_squared(self):
        all_params = torch.cat(list(self.string_to_param_dict.values()), axis=0)
        return (all_params * all_params).sum(axis=-1)

    def embedding_parameters(self):
        return self.string_to_param_dict.parameters()

    def trainable_parameters(self):
        return []

    def embedding_to_coarse_loss(self):
        loss = 0.
        num_embeddings = len(self.initial_embeddings)
        for key in self.initial_embeddings:
            optimized = self.string_to_param_dict[key]
            coarse = self.initial_embeddings[key].clone().to(optimized.device)
            loss = loss + (optimized - coarse) @ (optimized - coarse).T / num_embeddings
        return loss

    def embedding_neg_loss(self):
        return 0.
