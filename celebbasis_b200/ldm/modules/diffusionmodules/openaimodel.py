"""Host mirror of ldm/modules/diffusionmodules/openaimodel.py:413-742 (UNetModel) for the SD-v1 configuration.

Same constructor keywords and the same parameter names (686 tensors, `input_blocks.N.0.in_layers.0.weight`, ...)
as the reference so `load_state_dict(sd-v1-4.ckpt)` works by key.  forward(x, timesteps, context) keeps the
reference's NCHW fp32 contract and is differentiable with respect to `context` (the only upstream tensor that needs
a gradient when all UNet weights are frozen): the arithmetic runs in celebbasis_b200.unet_engine.UNetEngine.
"""
import torch
from torch import nn

from celebbasis_b200.unet_engine import UNetEngine
from ldm.modules.attention import SpatialTransformer
from ldm.modules.diffusionmodules.util import conv_nd, linear, normalization, zero_module


def _reset_engines(module, incompatible_keys):
    """load_state_dict post-hook: packed device weights are rebuilt lazily after a checkpoint load."""
    for name in ("_engine", "_face_engine", "_enc", "_dec"):
        if hasattr(module, name):
            setattr(module, name, None)
    module.__dict__.pop("_graphs", None)          # captured inference graphs point at the old packed weights


class TimestepEmbedSequential(nn.Sequential):
    pass


class Upsample(nn.Module):
    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels, self.out_channels = channels, out_channels or channels
        assert use_conv and dims == 2
        self.conv = conv_nd(dims, self.channels, self.out_channels, 3, padding=padding)


class Downsample(nn.Module):
    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels, self.out_channels = channels, out_channels or channels
        assert use_conv and dims == 2
        self.op = conv_nd(dims, self.channels, self.out_channels, 3, stride=2, padding=padding)


class ResBlock(nn.Module):
    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False,
                 use_scale_shift_norm=False, dims=2, use_checkpoint=False, up=False, down=False):
        super().__init__()
        assert not (up or down or use_scale_shift_norm), "not used by SD-v1 (aigc_id.yaml:40-54)"
        self.channels, self.out_channels = channels, out_channels or channels
        self.in_layers = nn.Sequential(normalization(channels), nn.SiLU(),
                                       conv_nd(dims, channels, self.out_channels, 3, padding=1))
        self.emb_layers = nn.Sequential(nn.SiLU(), linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(normalization(self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        zero_module(conv_nd(dims, self.out_channels, self.out_channels, 3, padding=1)))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = conv_nd(dims, channels, self.out_channels, 1)


class _UNetFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, timesteps, context, engine):
        need = ctx.needs_input_grad[2]
        ctx.engine = engine
        ctx.need = need
        return engine.forward(x.float().contiguous(), timesteps.long().contiguous(), context.float().contiguous(),
                              need_grad=need)

    @staticmethod
    def backward(ctx, d_eps):
        if not ctx.need:
            return None, None, None, None
        return None, None, ctx.engine.backward(d_eps.float().contiguous()), None


class UNetModel(nn.Module):
    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None,
                 use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1, num_heads_upsample=-1,
                 use_scale_shift_norm=False, resblock_updown=False, use_new_attention_order=False,
                 use_spatial_transformer=False, transformer_depth=1, context_dim=None, n_embed=None, legacy=True):
        super().__init__()
        assert use_spatial_transformer and context_dim is not None, "only the SD-v1 cross-attention UNet is mirrored"
        assert num_classes is None and not resblock_updown and n_embed is None and transformer_depth == 1
        assert num_head_channels == -1 and num_heads != -1, "SD-v1 fixes num_heads=8 (aigc_id.yaml:49)"
        if not isinstance(context_dim, int):
            context_dim = list(context_dim)[0] if len(list(context_dim)) == 1 else context_dim
        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels, self.num_res_blocks = out_channels, num_res_blocks
        self.attention_resolutions = list(attention_resolutions)
        self.channel_mult = list(channel_mult)
        self.num_heads, self.context_dim = num_heads, context_dim
        self.dtype = torch.float32
        ted = model_channels * 4
        self.time_embed = nn.Sequential(linear(model_channels, ted), nn.SiLU(), linear(ted, ted))
        self.input_blocks = nn.ModuleList(
            [TimestepEmbedSequential(conv_nd(dims, in_channels, model_channels, 3, padding=1))])
        chans = [model_channels]
        ch, ds = model_channels, 1
        mk_xf = lambda c: SpatialTransformer(c, num_heads, c // num_heads, depth=transformer_depth, context_dim=context_dim)
        for level, mult in enumerate(channel_mult):
            for _ in range(num_res_blocks):
                layers = [ResBlock(ch, ted, dropout, out_channels=mult * model_channels, dims=dims,
                                   use_checkpoint=use_checkpoint)]
                ch = mult * model_channels
                if ds in attention_resolutions:
                    layers.append(mk_xf(ch))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(Downsample(ch, conv_resample, dims=dims, out_channels=ch)))
                chans.append(ch)
                ds *= 2
        self.middle_block = TimestepEmbedSequential(
            ResBlock(ch, ted, dropout, dims=dims, use_checkpoint=use_checkpoint), mk_xf(ch),
            ResBlock(ch, ted, dropout, dims=dims, use_checkpoint=use_checkpoint))
        self.output_blocks = nn.ModuleList([])
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                ich = chans.pop()
                layers = [ResBlock(ch + ich, ted, dropout, out_channels=model_channels * mult, dims=dims,
                                   use_checkpoint=use_checkpoint)]
                ch = model_channels * mult
                if ds in attention_resolutions:
                    layers.append(mk_xf(ch))
                if level and i == num_res_blocks:
                    layers.append(Upsample(ch, conv_resample, dims=dims, out_channels=ch))
                    ds //= 2
                self.output_blocks.append(TimestepEmbedSequential(*layers))
        self.out = nn.Sequential(normalization(ch), nn.SiLU(),
                                 zero_module(conv_nd(dims, model_channels, out_channels, 3, padding=1)))
        self._engine = None
        self.register_load_state_dict_post_hook(_reset_engines)

    def engine_config(self):
        return dict(in_channels=self.in_channels, out_channels=self.out_channels, model_channels=self.model_channels,
                    attention_resolutions=self.attention_resolutions, num_res_blocks=self.num_res_blocks,
                    channel_mult=self.channel_mult, num_heads=self.num_heads, context_dim=self.context_dim)

    def engine(self, dtype=torch.float16):
        dev = self.time_embed[0].weight.device
        if dev.type != "cuda":
            raise RuntimeError("celebbasis_b200 UNetModel runs on sm_90a only (no CPU fallback): move it to cuda")
        if self._engine is None or self._engine.dev != dev or self._engine.dt != dtype:
            self._engine = UNetEngine(self.engine_config(), self.state_dict(), dev, dtype=dtype)
            self.__dict__.pop("_graphs", None)
        return self._engine

    GRAPH_INFERENCE = True     # no-grad forwards (the DDIM loop) replay one CUDA graph per input shape
    CAPTURE_GEMM_SINK = None   # optional list receiving (GemmDesc bytes, flops) of the launches captured into those graphs

    def forward(self, x, timesteps=None, context=None, y=None, **kwargs):
        assert y is None, "class-conditional UNets are not on the CelebBasis path"
        if (self.GRAPH_INFERENCE and not torch.is_grad_enabled() and x.is_cuda
                and not torch.cuda.is_current_stream_capturing()):
            return self._forward_graphed(x, timesteps, context)
        return _UNetFn.apply(x, timesteps, context, self.engine())

    def _forward_graphed(self, x, timesteps, context):
        """The sampler calls the UNet 50 times with the same shapes (ddim.py:166-204): the ~500 launches of one forward
        are captured once per (shape) and replayed; inputs are copied into the graph's static buffers.  The returned
        tensor is the graph's output buffer -- valid until the next call with the same shapes (the DDIM update consumes
        it immediately)."""
        eng = self.engine()
        key = (tuple(x.shape), tuple(context.shape), eng.dt)
        cache = self.__dict__.setdefault("_graphs", {})
        ent = cache.get(key)
        if ent is None:
            xs = x.detach().float().contiguous().clone()
            ts = timesteps.detach().long().contiguous().clone()
            cs = context.detach().float().contiguous().clone()
            from celebbasis_b200 import ops as _ops
            for _ in range(2):                                   # eager: GEMM autotune + lazily created workspaces
                eng.forward(xs, ts, cs, need_grad=False)
            torch.cuda.synchronize()
            from celebbasis_b200 import lib as _lib
            n0 = _lib.launch_count()
            g = torch.cuda.CUDAGraph()
            prev, _ops.GEMM_RECORD = _ops.GEMM_RECORD, self.CAPTURE_GEMM_SINK   # bench.py: the captured launches only
            try:                                                                 # (their buffers live in the graph's pool)
                with torch.cuda.graph(g):
                    out = eng.forward(xs, ts, cs, need_grad=False)
            finally:
                _ops.GEMM_RECORD = prev
            self.__dict__.setdefault("_graph_launches", {})[key] = _lib.launch_count() - n0
            ent = cache[key] = (g, xs, ts, cs, out)
        g, xs, ts, cs, out = ent
        xs.copy_(x)
        ts.copy_(timesteps)
        cs.copy_(context)
        g.replay()
        self.__dict__["_replayed_launches"] = self.__dict__.get("_replayed_launches", 0) + self._graph_launches[key]
        return out
