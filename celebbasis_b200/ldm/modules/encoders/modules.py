"""Host mirror of ldm/modules/encoders/modules.py:157-631 (FrozenCLIPEmbedder).

Same constructor keywords; `.tokenizer`, `.transformer.text_model.embeddings` (callable on token ids),
`.celeb_embeddings`, `.save_celeb_embeddings`, `forward/encode(text, embedding_manager=, face_img=, image_ori=)`.
The text transformer's parameters keep the Hugging Face names (`transformer.text_model.encoder.layers.N...`) so the
`cond_stage_model.*` keys of an SD-v1 checkpoint load unchanged; the 12-layer forward and the activation-gradient
backward (needed because the trainable signal enters at the input embeddings, modules.py:290-296) run in
celebbasis_b200.clip_engine.CLIPTextEngine.
"""
import torch
from torch import nn

from celebbasis_b200 import ops
from celebbasis_b200.clip_engine import CLIPTextEngine
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer


def _reset_engines(module, incompatible_keys):
    """load_state_dict post-hook: packed device weights are rebuilt lazily after a checkpoint load."""
    for name in ("_engine", "_face_engine", "_enc", "_dec"):
        if hasattr(module, name):
            setattr(module, name, None)


class AbstractEncoder(nn.Module):
    def encode(self, *args, **kwargs):
        raise NotImplementedError


class _CLIPAttn(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (nn.Linear(d, d) for _ in range(4))


class _CLIPMLP(nn.Module):
    def __init__(self, d, inter):
        super().__init__()
        self.fc1, self.fc2 = nn.Linear(d, inter), nn.Linear(inter, d)


class _CLIPLayer(nn.Module):
    def __init__(self, d, inter, eps):
        super().__init__()
        self.self_attn = _CLIPAttn(d)
        self.layer_norm1 = nn.LayerNorm(d, eps=eps)
        self.mlp = _CLIPMLP(d, inter)
        self.layer_norm2 = nn.LayerNorm(d, eps=eps)


class _CLIPEncoder(nn.Module):
    def __init__(self, n, d, inter, eps):
        super().__init__()
        self.layers = nn.ModuleList([_CLIPLayer(d, inter, eps) for _ in range(n)])


class _CLIPEmbeddings(nn.Module):
    def __init__(self, vocab, d, max_pos):
        super().__init__()
        self.token_embedding = nn.Embedding(vocab, d)
        self.position_embedding = nn.Embedding(max_pos, d)
        self.register_buffer("position_ids", torch.arange(max_pos).expand((1, -1)), persistent=False)

    def forward(self, input_ids=None, position_ids=None, inputs_embeds=None, only_embedding=False, **kw):
        """modules.py:176-298 without an embedding manager: token rows (+ positions unless only_embedding)."""
        ids = input_ids.reshape(1, -1) if input_ids.dim() == 1 else input_ids
        tok = ops.embedding_gather(ids.reshape(-1).to(self.token_embedding.weight.device).long().contiguous(),
                                   self.token_embedding.weight.detach().float().contiguous())
        tok = tok.view(ids.shape[0], ids.shape[1], -1)
        if only_embedding:
            return tok
        pos = self.position_embedding.weight[: ids.shape[1]].detach().float().contiguous()
        out = torch.empty_like(tok)
        for b in range(tok.shape[0]):
            ops.axpby(tok[b], 1.0, pos, 1.0, out=out[b])
        return out


class _CLIPTextTransformer(nn.Module):
    def __init__(self, vocab=49408, d=768, layers=12, heads=12, inter=3072, max_pos=77, eps=1e-5):
        super().__init__()
        self.embeddings = _CLIPEmbeddings(vocab, d, max_pos)
        self.encoder = _CLIPEncoder(layers, d, inter, eps)
        self.final_layer_norm = nn.LayerNorm(d, eps=eps)
        self.heads, self.eps = heads, eps


class _CLIPTextModel(nn.Module):
    def __init__(self, **kw):
        super().__init__()
        self.text_model = _CLIPTextTransformer(**kw)


class _CLIPFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb, engine, batch):
        need = ctx.needs_input_grad[0]
        ctx.engine, ctx.need, ctx.shape = engine, need, emb.shape
        out = engine.forward(emb.reshape(-1, emb.shape[-1]).float().contiguous(), batch, need_grad=need)
        return out.view(emb.shape)

    @staticmethod
    def backward(ctx, dctx):
        if not ctx.need:
            return None, None, None
        d = ctx.engine.backward(dctx.reshape(-1, dctx.shape[-1]).float().contiguous())
        return d.view(ctx.shape), None, None


class _AddPosFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, pos):
        out = torch.empty_like(x)
        for b in range(x.shape[0]):
            ops.axpby(x[b].contiguous(), 1.0, pos, 1.0, out=out[b])
        return out

    @staticmethod
    def backward(ctx, g):
        return g, None


class FrozenCLIPEmbedder(AbstractEncoder):
    """Uses the CLIP transformer encoder for text (Hugging Face layout), H100-native arithmetic."""

    def __init__(self, version="openai/clip-vit-large-patch14", device="cuda", max_length=77,
                 celeb_txt="./infer_images/wiki_names_v2.txt", use_celeb=False, use_svd=False, n_components: int = 512,
                 rm_repeats: bool = True, use_sample_reduce=False, n_samples: int = 513, use_flatten: bool = True,
                 num_embeds_per_token: int = 2, num_hidden_layers: int = 12):
        super().__init__()
        self.tokenizer = self._make_tokenizer(version)
        self.transformer = _CLIPTextModel(layers=num_hidden_layers)
        self._try_load_pretrained(version)
        self.device = device
        self.max_length = max_length
        self.celeb_txt, self.celeb_embeddings = celeb_txt, None
        self.use_celeb, self.use_svd, self.rm_repeats = use_celeb, use_svd, rm_repeats
        self.use_sample_reduce, self.n_samples, self.use_flatten = use_sample_reduce, n_samples, use_flatten
        self.num_embeds_per_token = num_embeds_per_token
        self.n_components = n_components
        self._engine = None
        self.register_load_state_dict_post_hook(_reset_engines)
        if use_celeb:
            self._get_celeb_embeddings(n_components)

    @staticmethod
    def _make_tokenizer(version):
        try:
            from transformers import CLIPTokenizer
            tok = CLIPTokenizer.from_pretrained(version, local_files_only=True)
            probe = tok("sks", truncation=True, max_length=77, padding="max_length", return_tensors="pt")["input_ids"]
            if int(probe[0, 0]) == 49406 and int(probe[0, 1]) == 48136:   # a real CLIP BPE vocabulary is present
                return tok
        except Exception:
            pass
        return SyntheticCLIPTokenizer()   # no CLIP vocabulary on disk and no network (see tokenizer.py)

    def _try_load_pretrained(self, version):
        try:
            from transformers import CLIPTextModel
            hf = CLIPTextModel.from_pretrained(version, local_files_only=True)
            self.transformer.load_state_dict(hf.state_dict(), strict=False)
        except Exception:
            pass   # weights arrive with the SD checkpoint (cond_stage_model.* keys) or stay at their random init

    def freeze(self):
        self.transformer = self.transformer.eval()
        for p in self.parameters():
            p.requires_grad = False

    def engine(self, dtype=torch.float16):
        tm = self.transformer.text_model
        dev = tm.final_layer_norm.weight.device
        if dev.type != "cuda":
            raise RuntimeError("celebbasis_b200 FrozenCLIPEmbedder runs on sm_90a only (no CPU fallback)")
        if self._engine is None or self._engine.dev != dev or self._engine.dt != dtype:
            self._engine = CLIPTextEngine(self.transformer.state_dict(), dev, dtype=dtype, heads=tm.heads, eps=tm.eps)
        return self._engine

    def forward(self, text, embedding_manager=None, face_img=None, image_ori=None, only_embedding=False, **kwargs):
        eng = self.engine()
        dev = eng.dev
        enc = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                             return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        tokens = enc["input_ids"]
        B, T = tokens.shape
        tok = ops.embedding_gather(tokens.to(dev).reshape(-1).contiguous(), eng.tok_table).view(B, T, -1)
        if only_embedding:
            return tok
        if embedding_manager is not None:
            celeb = self.celeb_embeddings
            tok = embedding_manager(tokens, tok, face_img, image_ori, celeb)
        emb = _AddPosFn.apply(tok, eng.pos_table[:T].contiguous())
        return _CLIPFn.apply(emb, eng, B)

    def encode(self, text, **kwargs):
        return self(text, **kwargs)

    @torch.no_grad()
    def _get_celeb_embeddings(self, n_components: int = 0):
        """modules.py:472-624: the celeb basis -- per token column (use_flatten=False, aigc_id.yaml) or over all name
        tokens (use_flatten=True, the constructor default) the mean + n_components right-singular vectors of the CLIP
        token embeddings of the ~650 celebrity names, optionally after the sample reduction of :575-584.  Init-time,
        host-side linear algebra (torch.svd on CPU, like the reference); the hot path only consumes the resulting
        (num_embeds_per_token, 1+n_components, 768) tensor.

        Faithful to two quirks of the reference: names are sorted after de-duplication (:479-487), and the `tok in
        set_of_tensors` tests (:521-533) compare 0-dim tensors by identity and therefore never remove a repeated token."""
        with open(self.celeb_txt, "r") as f:
            names = f.read().splitlines()
        names = sorted(set(names)) if self.rm_repeats else sorted(names)
        table = self.transformer.text_model.embeddings.token_embedding.weight.detach().float().cpu()
        ids = [self.tokenizer(n, truncation=True, max_length=self.max_length, return_length=True,
                              return_overflowing_tokens=False, padding="max_length",
                              return_tensors="pt")["input_ids"][0] for n in names]
        all_tokens = torch.stack(ids, 0)                                  # (M, 77)
        keep = all_tokens < 49406
        if not self.use_flatten:
            cols = [table[all_tokens[:, j][keep[:, j]]] for j in range(all_tokens.shape[1])]
            cols = [c for c in cols if c.shape[0] > 0]
        else:
            cols = [table[all_tokens[keep]]]                              # row-major over (name, position), :535-544
        self.celeb_cols_len = [int(c.shape[0]) for c in cols]
        out = []
        for j, x in enumerate(cols[: self.num_embeds_per_token]):
            if self.use_sample_reduce:                                    # :575-584
                e = x.t()                                                 # (768, m)
                u, s_, v = torch.svd(e - e.mean(dim=0, keepdims=True), some=False)
                x = torch.matmul(e, v[:, : self.n_samples]).t()           # (r, 768)
            if self.use_svd:                                              # :598-607 ("3dmm/pca-based svd")
                c_mean = x.mean(dim=0, keepdims=True)
                u, s_, v = torch.svd(x - c_mean, some=False)
                x = torch.cat([c_mean, v.t()[:n_components]], dim=0)
            out.append(x.unsqueeze(0))
        if self.use_flatten:
            out = out * self.num_embeds_per_token                         # :617-618: the one flat basis, repeated
        self.celeb_embeddings = torch.cat(out, 0).to(self.device if torch.cuda.is_available() else "cpu")

    @torch.no_grad()
    def save_celeb_embeddings(self, pth_path: str):
        assert isinstance(self.celeb_embeddings, torch.Tensor), "No celeb_embeddings!"
        torch.save(self.celeb_embeddings.cpu(), pth_path)
