"""Host mirror of ldm/modules/attention.py (reference :37-64 GEGLU/FeedForward, :152-193 CrossAttention,
:196-215 BasicTransformerBlock, :218-261 SpatialTransformer).

The classes keep the reference's constructor arguments and parameter names (so SD-v1 checkpoints load by key).
Inside a UNetModel they are parameter containers: the UNet engine (celebbasis_b200/unet_engine.py) reads their
weights and runs the fused kernels.  CrossAttention.forward is also usable stand-alone (inference, no grad): it
runs q/k/v projection, scaled-dot-product softmax and out-projection on the wgmma GEMM + softmax kernels.
"""
import torch
from torch import nn

from celebbasis_b200 import ops
from celebbasis_b200.unet_engine import _Attn


def exists(val):
    return val is not None


def default(val, d):
    return val if exists(val) else d


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


def Normalize(in_channels):
    return torch.nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    def __init__(self, dim, dim_out=None, mult=4, glu=False, dropout=0.):
        super().__init__()
        inner_dim = int(dim * mult)
        dim_out = default(dim_out, dim)
        assert glu, "SD-v1 uses the GEGLU feed-forward (attention.py:205)"
        self.net = nn.Sequential(GEGLU(dim, inner_dim), nn.Dropout(dropout), nn.Linear(inner_dim, dim_out))


class CrossAttention(nn.Module):
    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.):
        super().__init__()
        inner_dim = dim_head * heads
        context_dim = default(context_dim, query_dim)
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.dim_head = dim_head
        self.to_q = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_k = nn.Linear(context_dim, inner_dim, bias=False)
        self.to_v = nn.Linear(context_dim, inner_dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, query_dim), nn.Dropout(dropout))
        self._packed = None

    def _pack(self, dtype):
        dev = self.to_q.weight.device
        if self._packed is None or self._packed[0] != (dev, dtype):
            w = lambda m: m.weight.detach().to(dev, torch.float32).to(dtype).contiguous()
            self._packed = ((dev, dtype), w(self.to_q), w(self.to_k), w(self.to_v), w(self.to_out[0]),
                            self.to_out[0].bias.detach().float().contiguous())
        return self._packed[1:]

    @torch.no_grad()
    def forward(self, x, context=None, mask=None):
        """x: (B, N, query_dim); context: (B, M, context_dim) or None (self-attention).  Returns (B, N, query_dim)."""
        assert mask is None, "the mask path of attention.py:182-186 is unused by CelebBasis"
        if not x.is_cuda:
            raise RuntimeError("celebbasis_b200 CrossAttention runs on sm_90a only (no CPU fallback)")
        dt = torch.float16
        wq, wk, wv, wo, bo = self._pack(dt)
        B, N, _ = x.shape
        ctx = x if context is None else context
        M = ctx.shape[1]
        x16 = ops.cast(x.reshape(B * N, -1).float().contiguous(), dt)
        c16 = x16 if context is None else ops.cast(ctx.reshape(B * M, -1).float().contiguous(), dt)
        q, k, v = ops.linear(x16, wq), ops.linear(c16, wk), ops.linear(c16, wv)
        o = torch.empty_like(q)
        _Attn.fwd(q, k, v, images=B, heads=self.heads, dh=self.dim_head, nq=N, nk=M, scale=self.scale, out=o)
        y = ops.linear(o, wo, bo, out_dtype=torch.float32)
        return y.view(B, N, -1).to(x.dtype)


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, n_heads, d_head, dropout=0., context_dim=None, gated_ff=True, checkpoint=True):
        super().__init__()
        self.attn1 = CrossAttention(query_dim=dim, heads=n_heads, dim_head=d_head, dropout=dropout)
        self.ff = FeedForward(dim, dropout=dropout, glu=gated_ff)
        self.attn2 = CrossAttention(query_dim=dim, context_dim=context_dim, heads=n_heads, dim_head=d_head,
                                    dropout=dropout)
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.norm3 = nn.LayerNorm(dim)
        self.checkpoint = checkpoint  # a no-op in the reference as well (diffusionmodules/util.py:112-116)


class SpatialTransformer(nn.Module):
    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0., context_dim=None):
        super().__init__()
        self.in_channels = in_channels
        inner_dim = n_heads * d_head
        self.norm = Normalize(in_channels)
        self.proj_in = nn.Conv2d(in_channels, inner_dim, kernel_size=1, stride=1, padding=0)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner_dim, n_heads, d_head, dropout=dropout, context_dim=context_dim)
             for _ in range(depth)])
        self.proj_out = zero_module(nn.Conv2d(inner_dim, in_channels, kernel_size=1, stride=1, padding=0))
