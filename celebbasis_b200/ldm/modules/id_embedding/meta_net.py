"""Host mirror of ldm/modules/id_embedding/meta_net.py (MetaIdNet, :100-355) for the CelebBasis configuration
(use_celebs=True, mlp_depth=1, use_expert=False, use_header=False, use_rm_mlp=False).

    faces (N,H,W,3k) -> chunk/cat -> affine warp + resize 112 -> CosFace iresnet100 -> L2 norm        [no grad]
          -> EqualLinear(512 -> es*inner, lr_mul 1) + LeakyReLU(0.2) -> (N,es,1,inner) -> L2 norm       [trainable]
          -> einsum with the celeb basis + mean -> (N, es, 768)
The trainable part is differentiable with respect to stylegan_mlp.net.0.{weight,bias}; all arithmetic runs in the
fp32 side kernels of celebbasis_b200/csrc/cb_embed.cu.
"""
import torch
from torch import nn

from celebbasis_b200 import ops
from celebbasis_b200.iresnet_engine import IResNetEngine
from celebbasis_b200.train_step import TRANS_MATRIX
from ldm.modules.id_embedding.iresnet import iresnet100


def _reset_engines(module, incompatible_keys):
    """load_state_dict post-hook: packed device weights are rebuilt lazily after a checkpoint load."""
    for name in ("_engine", "_face_engine", "_enc", "_dec"):
        if hasattr(module, name):
            setattr(module, name, None)


class EqualLinear(nn.Module):
    def __init__(self, in_dim, out_dim, lr_mul=1, bias=True, pre_norm=False):
        super().__init__()
        assert not pre_norm
        self.weight = nn.Parameter(torch.randn(out_dim, in_dim))
        self.bias = nn.Parameter(torch.zeros(out_dim))
        self.lr_mul = lr_mul


class StyleVectorizer(nn.Module):
    def __init__(self, dim_in, dim_out, depth, lr_mul=0.1):
        super().__init__()
        assert depth == 1, "aigc_id.yaml: meta_mlp_depth 1"
        self.net = nn.Sequential(EqualLinear(dim_in, dim_out, lr_mul))


class _CelebFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, W, b, v, basis, es):
        pre, coef, nrm = ops.celeb_mlp_fwd(v, W.detach().contiguous(), b.detach().contiguous(), es)
        z = ops.celeb_basis_fwd(coef, basis)
        ctx.save_for_backward(pre, coef, nrm, v, basis)
        ctx.shapes = (W.shape, b.shape)
        return z, coef

    @staticmethod
    def backward(ctx, dz, dcoef_unused):
        pre, coef, nrm, v, basis = ctx.saved_tensors
        dcoef = ops.celeb_basis_bwd(dz.contiguous().float(), basis)
        dW = torch.empty(ctx.shapes[0], dtype=torch.float32, device=v.device)
        db = torch.empty(ctx.shapes[1], dtype=torch.float32, device=v.device)
        ops.celeb_mlp_bwd(dcoef, coef, nrm, pre, v, dW, db)
        return dW, db, None, None, None


class MetaIdNet(nn.Module):
    def __init__(self, fr_dim=512, meta_dim=768, inner_dim=512, mlp_depth=1, use_expert=False, num_ids=10,
                 expert_dim=128, use_header=False, use_celebs=False, num_embeds_per_token=2, heads=1,
                 use_rm_mlp=False, vis_mean=False, vis_mean_params=None):
        super().__init__()
        assert use_celebs and not use_expert and not use_header and not use_rm_mlp and heads == 1
        self.fr_dim, self.meta_dim = fr_dim, meta_dim
        self.num_es, self.heads = num_embeds_per_token, heads
        self.id_model = None
        self.load_fr_net()
        self.register_buffer("trans_matrix", torch.tensor([[list(TRANS_MATRIX[:3]), list(TRANS_MATRIX[3:])]]).float())
        self.stylegan_mlp = StyleVectorizer(fr_dim, inner_dim * self.num_es * self.heads, depth=mlp_depth, lr_mul=1.0)
        self._face_engine = None
        self.register_load_state_dict_post_hook(_reset_engines)

    def load_fr_net(self):
        """meta_net.py:348-355 loads ./weights/glint360k_cosface_r100_fp16_0.1/backbone.pth when it exists."""
        import os
        self.id_model = iresnet100()
        path = './weights/glint360k_cosface_r100_fp16_0.1/backbone.pth'
        if os.path.exists(path):
            self.id_model.load_state_dict(torch.load(path, map_location="cpu"))
        for p in self.id_model.parameters():
            p.requires_grad = False
        self.id_model.eval()

    def face_engine(self):
        dev = self.stylegan_mlp.net[0].weight.device
        if dev.type != "cuda":
            raise RuntimeError("celebbasis_b200 MetaIdNet runs on sm_90a only (no CPU fallback)")
        if self._face_engine is None or self._face_engine.dev != dev:
            self._face_engine = IResNetEngine(self.id_model.state_dict(), dev)
        return self._face_engine

    @torch.no_grad()
    def face_features(self, faces, n_chunks):
        eng = self.face_engine()
        tm = [float(v) for v in self.trans_matrix.flatten().tolist()]
        x, geo = ops.face_warp_resize(faces.float().contiguous(), n_chunks, tm, out_hw=112, cpad=8, dtype=eng.dt)
        return ops.l2norm_rows(eng.forward(x, geo))

    def forward_multi_faces(self, img_multi, id_multi, celeb_embeds=None):
        """(N,H,W,3k) faces, (N,k) ids -> tuples of k chunks: vec (N,es,768), None, cef (N,es,1,inner)."""
        b, num = id_multi.shape
        v = self.face_features(img_multi, num)                                      # (k*N, 512), chunk-major
        lin = self.stylegan_mlp.net[0]
        z, coef = _CelebFn.apply(lin.weight, lin.bias, v, celeb_embeds.float().contiguous(), self.num_es)
        cef = coef.view(coef.shape[0], self.num_es, self.heads, -1)
        return z.chunk(num, 0), None, cef.chunk(num, 0)

    def trainable_state_dict(self, verbose=False):
        return {k: v for k, v in self.state_dict().items() if 'stylegan_mlp' in k}

    def load_trainable_state_dict(self, sd, verbose=False):
        self.load_state_dict(sd, strict=False)
