"""AutoencoderKL.encode (first-stage encoder + quant_conv) on the sm_90a kernels, forward only / no grad.

Mirrors ldm/models/autoencoder.py:324-328 -> ldm/modules/diffusionmodules/model.py:434-459 (Encoder.forward),
:82-141 (ResnetBlock), :150-202 (AttnBlock: 1 head over all pixels), :60-79 (Downsample: pad (0,1,0,1) + stride 2).
The largest single item of a training step (1.1 TFLOP at 512x512): every conv is the same TMA-shifted implicit
GEMM as the UNet's, GroupNorm(eps 1e-6)+swish is one cb_groupnorm_fwd call with the SiLU fused, the 4096-token
attention reuses the batched GEMM + softmax path with head_dim = 512.
"""
import torch

from . import ops
from .ops import Geo
from .unet_engine import _Attn, _round_up


class VAEEncoderEngine:
    def __init__(self, ddconfig, embed_dim, state_dict, device, *, prefix="", dtype=torch.float16,
                 res_dtype=torch.float32):
        self.dev = torch.device(device)
        self.dt = dtype
        self.rt = res_dtype
        sd, p = state_dict, prefix
        f32 = lambda t: ops.to_device(t, self.dev)
        w16 = lambda t: ops.to_device(t, self.dev, self.dt)
        pack = lambda k, **kw: ops.pack_conv_weight(sd[p + k], self.dt, device=self.dev, **kw)
        ch, mult, nres = ddconfig["ch"], ddconfig["ch_mult"], ddconfig["num_res_blocks"]
        self.in_ch = ddconfig["in_channels"]
        self.in_pad = _round_up(self.in_ch, 8)
        self.zc2 = 2 * ddconfig["z_channels"] if ddconfig.get("double_z", True) else ddconfig["z_channels"]
        self.conv_in_w, self.conv_in_b = pack("encoder.conv_in.weight", cin_pad=self.in_pad), f32(sd[p + "encoder.conv_in.bias"])
        self.ch0 = ch

        def res(pre, cin, cout):
            w = {"cin": cin, "cout": cout,
                 "g1": f32(sd[pre + "norm1.weight"]), "b1": f32(sd[pre + "norm1.bias"]),
                 "w1": ops.pack_conv_weight(sd[pre + "conv1.weight"], self.dt, device=self.dev), "c1b": f32(sd[pre + "conv1.bias"]),
                 "g2": f32(sd[pre + "norm2.weight"]), "b2": f32(sd[pre + "norm2.bias"]),
                 "w2": ops.pack_conv_weight(sd[pre + "conv2.weight"], self.dt, device=self.dev), "c2b": f32(sd[pre + "conv2.bias"])}
            if cin != cout:
                w["ws"] = w16(sd[pre + "nin_shortcut.weight"].reshape(cout, cin))
                w["bs"] = f32(sd[pre + "nin_shortcut.bias"])
            else:
                w["ws"] = None
            return w

        in_mult = (1,) + tuple(mult)
        self.levels = []
        bin_ = ch
        for i in range(len(mult)):
            bin_, bout = ch * in_mult[i], ch * mult[i]
            blocks = []
            for j in range(nres):
                blocks.append(res(p + f"encoder.down.{i}.block.{j}.", bin_, bout))
                bin_ = bout
            down = None
            if i != len(mult) - 1:
                dk = p + f"encoder.down.{i}.downsample.conv."
                down = {"w": ops.pack_conv_weight(sd[dk + "weight"], self.dt, device=self.dev), "b": f32(sd[dk + "bias"]), "c": bin_}
            self.levels.append((blocks, down))
        self.mid1 = res(p + "encoder.mid.block_1.", bin_, bin_)
        self.mid2 = res(p + "encoder.mid.block_2.", bin_, bin_)
        ak = p + "encoder.mid.attn_1."
        c = bin_
        self.attn = {"c": c, "gn": f32(sd[ak + "norm.weight"]), "bn": f32(sd[ak + "norm.bias"]),
                     "wqkv": w16(torch.cat([sd[ak + "q.weight"].reshape(c, c), sd[ak + "k.weight"].reshape(c, c),
                                            sd[ak + "v.weight"].reshape(c, c)], 0)),
                     "bqkv": f32(torch.cat([sd[ak + "q.bias"], sd[ak + "k.bias"], sd[ak + "v.bias"]], 0)),
                     "wo": w16(sd[ak + "proj_out.weight"].reshape(c, c)), "bo": f32(sd[ak + "proj_out.bias"])}
        self.no_g, self.no_b = f32(sd[p + "encoder.norm_out.weight"]), f32(sd[p + "encoder.norm_out.bias"])
        self.c_last = bin_
        self.out_rows = _round_up(self.zc2, 16)
        self.conv_out_w = pack("encoder.conv_out.weight", cout_pad=self.out_rows)
        cb = torch.zeros(self.out_rows, dtype=torch.float32, device=self.dev)
        cb[: self.zc2] = f32(sd[p + "encoder.conv_out.bias"])
        self.conv_out_b = cb
        qw = sd[p + "quant_conv.weight"]
        self.q_out = qw.shape[0]
        qpad = torch.zeros(self.q_out, _round_up(self.zc2, 8), dtype=torch.float32)
        qpad[:, : self.zc2] = qw.reshape(self.q_out, self.zc2)
        self.quant_w, self.quant_b = w16(qpad), f32(sd[p + "quant_conv.bias"])
        self.mid_pad = _round_up(self.zc2, 8)

    def _res(self, w, x, geo):
        a, _ = ops.groupnorm(x, geo, w["g1"], w["b1"], eps=1e-6, silu=True, out_dtype=self.dt)
        h, _ = ops.conv2d(a, geo, w["w1"], w["cout"], bias=w["c1b"], out_dtype=self.dt)
        b, _ = ops.groupnorm(h, geo, w["g2"], w["b2"], eps=1e-6, silu=True, out_dtype=self.dt)
        if w["ws"] is None:
            resid = x
        else:
            x16 = x if x.dtype == self.dt else ops.cast(x, self.dt)
            resid = ops.linear(x16, w["ws"], w["bs"], out_dtype=self.rt)
        out, _ = ops.conv2d(b, geo, w["w2"], w["cout"], bias=w["c2b"], out_dtype=self.rt, residual=resid)
        return out

    def _attn(self, x, geo):
        w = self.attn
        c = w["c"]
        n, _ = ops.groupnorm(x, geo, w["gn"], w["bn"], eps=1e-6, silu=False, out_dtype=self.dt)
        qkv = ops.linear(n, w["wqkv"], w["bqkv"])
        o = torch.empty(geo.rows, c, dtype=self.dt, device=self.dev)
        _Attn.fwd(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], images=geo.n, heads=1, dh=c, nq=geo.hw, nk=geo.hw,
                  scale=float(c) ** -0.5, out=o)
        return ops.linear(o, w["wo"], w["bo"], out_dtype=self.rt, residual=x)

    @torch.no_grad()
    def encode_moments(self, x):
        """x: (B,3,H,W) fp32 NCHW in [-1,1] -> moments (B, 2*z, H/8, W/8) fp32 NCHW (the posterior parameters)."""
        x16, geo = ops.nchw_to_nhwc(x.contiguous().float(), self.in_pad, self.dt)
        h, _ = ops.conv2d(x16, geo, self.conv_in_w, self.ch0, bias=self.conv_in_b, out_dtype=self.rt)
        for blocks, down in self.levels:
            for w in blocks:
                h = self._res(w, h, geo)
            if down is not None:
                h16 = h if h.dtype == self.dt else ops.cast(h, self.dt)
                h, geo = ops.conv2d(h16, geo, down["w"], down["c"], bias=down["b"], stride=2, pad=(0, 1, 0, 1),
                                    out_dtype=self.rt)
        h = self._res(self.mid1, h, geo)
        h = self._attn(h, geo)
        h = self._res(self.mid2, h, geo)
        a, _ = ops.groupnorm(h, geo, self.no_g, self.no_b, eps=1e-6, silu=True, out_dtype=self.dt)
        m = torch.zeros(geo.rows, self.mid_pad, dtype=self.dt, device=self.dev) if self.mid_pad != self.zc2 else \
            torch.empty(geo.rows, self.mid_pad, dtype=self.dt, device=self.dev)
        ops.conv2d(a, geo, self.conv_out_w, self.zc2, bias=self.conv_out_b, out=m, cout_rows=self.out_rows)
        q = ops.linear(m, self.quant_w, self.quant_b, out_dtype=torch.float32)
        return ops.nhwc_to_nchw(q, geo, self.q_out)


class VAEDecoderEngine:
    """AutoencoderKL.decode: post_quant_conv + Decoder (ldm/models/autoencoder.py:330-333, model.py:462-568), no grad.

    The decoder's 512x512x128 activations are the largest tensors of the txt2img path, so its residual stream is
    fp16 (the reference runs it under fp16 autocast as well, scripts/stable_txt2img.py:320-322)."""

    def __init__(self, ddconfig, embed_dim, state_dict, device, *, prefix="", dtype=torch.float16, res_dtype=None):
        self.dev = torch.device(device)
        self.dt = dtype
        self.rt = res_dtype or dtype
        sd, p = state_dict, prefix
        f32 = lambda t: ops.to_device(t, self.dev)
        w16 = lambda t: ops.to_device(t, self.dev, self.dt)
        ch, mult, nres = ddconfig["ch"], ddconfig["ch_mult"], ddconfig["num_res_blocks"]
        zc = ddconfig["z_channels"]
        self.zc, self.zpad = zc, _round_up(zc, 8)
        self.out_ch = ddconfig["out_ch"]
        pq = torch.zeros(self.zpad, self.zpad, dtype=torch.float32)
        pq[:zc, :embed_dim] = sd[p + "post_quant_conv.weight"].reshape(zc, embed_dim)
        self.pq_w = w16(pq)
        pqb = torch.zeros(self.zpad, dtype=torch.float32)
        pqb[:zc] = sd[p + "post_quant_conv.bias"]
        self.pq_b = f32(pqb)
        self.embed_dim = embed_dim

        def res(pre, cin, cout):
            w = {"cin": cin, "cout": cout,
                 "g1": f32(sd[pre + "norm1.weight"]), "b1": f32(sd[pre + "norm1.bias"]),
                 "w1": ops.pack_conv_weight(sd[pre + "conv1.weight"], self.dt, device=self.dev), "c1b": f32(sd[pre + "conv1.bias"]),
                 "g2": f32(sd[pre + "norm2.weight"]), "b2": f32(sd[pre + "norm2.bias"]),
                 "w2": ops.pack_conv_weight(sd[pre + "conv2.weight"], self.dt, device=self.dev), "c2b": f32(sd[pre + "conv2.bias"])}
            if cin != cout:
                w["ws"] = w16(sd[pre + "nin_shortcut.weight"].reshape(cout, cin))
                w["bs"] = f32(sd[pre + "nin_shortcut.bias"])
            else:
                w["ws"] = None
            return w

        bin_ = ch * mult[-1]
        self.c_in = bin_
        self.conv_in_w = ops.pack_conv_weight(sd[p + "decoder.conv_in.weight"], self.dt, device=self.dev, cin_pad=self.zpad)
        self.conv_in_b = f32(sd[p + "decoder.conv_in.bias"])
        self.mid1 = res(p + "decoder.mid.block_1.", bin_, bin_)
        self.mid2 = res(p + "decoder.mid.block_2.", bin_, bin_)
        ak = p + "decoder.mid.attn_1."
        c = bin_
        self.attn = {"c": c, "gn": f32(sd[ak + "norm.weight"]), "bn": f32(sd[ak + "norm.bias"]),
                     "wqkv": w16(torch.cat([sd[ak + "q.weight"].reshape(c, c), sd[ak + "k.weight"].reshape(c, c),
                                            sd[ak + "v.weight"].reshape(c, c)], 0)),
                     "bqkv": f32(torch.cat([sd[ak + "q.bias"], sd[ak + "k.bias"], sd[ak + "v.bias"]], 0)),
                     "wo": w16(sd[ak + "proj_out.weight"].reshape(c, c)), "bo": f32(sd[ak + "proj_out.bias"])}
        self.levels = []   # executed order: highest level index first
        for i in reversed(range(len(mult))):
            bout = ch * mult[i]
            blocks = []
            for j in range(nres + 1):
                blocks.append(res(p + f"decoder.up.{i}.block.{j}.", bin_, bout))
                bin_ = bout
            up = None
            if i != 0:
                uk = p + f"decoder.up.{i}.upsample.conv."
                up = {"w": ops.pack_conv_weight(sd[uk + "weight"], self.dt, device=self.dev), "b": f32(sd[uk + "bias"]), "c": bin_}
            self.levels.append((blocks, up))
        self.no_g, self.no_b = f32(sd[p + "decoder.norm_out.weight"]), f32(sd[p + "decoder.norm_out.bias"])
        self.out_rows = 16
        self.conv_out_w = ops.pack_conv_weight(sd[p + "decoder.conv_out.weight"], self.dt, device=self.dev, cout_pad=self.out_rows)
        cb = torch.zeros(self.out_rows, dtype=torch.float32, device=self.dev)
        cb[: self.out_ch] = f32(sd[p + "decoder.conv_out.bias"])
        self.conv_out_b = cb

    _res = VAEEncoderEngine._res
    _attn = VAEEncoderEngine._attn

    @torch.no_grad()
    def decode(self, z):
        """z: (B, z_channels, h, w) fp32 NCHW -> image (B, out_ch, 8h, 8w) fp32 NCHW."""
        z16, geo = ops.nchw_to_nhwc(z.contiguous().float(), self.zpad, self.dt)
        h0 = ops.linear(z16, self.pq_w, self.pq_b)                                       # post_quant_conv (1x1)
        h, _ = ops.conv2d(h0, geo, self.conv_in_w, self.c_in, bias=self.conv_in_b, out_dtype=self.rt)
        h = self._res(self.mid1, h, geo)
        h = self._attn(h, geo)
        h = self._res(self.mid2, h, geo)
        for blocks, up in self.levels:
            for w in blocks:
                h = self._res(w, h, geo)
            if up is not None:
                h16 = h if h.dtype == self.dt else ops.cast(h, self.dt)
                u, geo = ops.upsample2x(h16, geo)
                h, _ = ops.conv2d(u, geo, up["w"], up["c"], bias=up["b"], out_dtype=self.rt)
        a, _ = ops.groupnorm(h, geo, self.no_g, self.no_b, eps=1e-6, silu=True, out_dtype=self.dt)
        y, _ = ops.conv2d(a, geo, self.conv_out_w, self.out_ch, bias=self.conv_out_b, out_dtype=torch.float32,
                          cout_rows=self.out_rows)
        return ops.nhwc_to_nchw(y, geo, self.out_ch)
