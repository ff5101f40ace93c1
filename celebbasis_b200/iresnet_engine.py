"""CosFace iresnet100 forward (eval, no grad) on the sm_90a kernels.

Mirrors ldm/modules/id_embedding/iresnet.py:166-181 (IResNet.forward) and :26-64 (IBasicBlock):
    bn1 -> conv3x3 -> bn2 -> PReLU -> conv3x3(stride) -> bn3  (+ identity | conv1x1(stride)+bn)
Eval-mode BatchNorms that FOLLOW a conv are folded into its weights/bias at load time (exact); the bn1 that
precedes a zero-padded conv is applied as a per-channel affine kernel (folding it would change the border).
The final BatchNorm2d -> flatten(NCHW) -> fc -> BatchNorm1d collapses into one GEMM whose weight columns are
permuted to the NHWC flatten order.
"""
import torch

from . import ops
from .ops import Geo


def _bn_fold(sd, pre, eps=1e-5):
    s = sd[pre + "weight"].float() / torch.sqrt(sd[pre + "running_var"].float() + eps)
    return s, sd[pre + "bias"].float() - sd[pre + "running_mean"].float() * s


class IResNetEngine:
    def __init__(self, state_dict, device, *, prefix="", layers=(3, 13, 30, 3), dtype=torch.float16):
        self.dev = torch.device(device)
        self.dt = dtype
        sd, p = state_dict, prefix
        f32 = lambda t: ops.to_device(t, self.dev)

        def conv_bn(wkey, bnpre, cin_pad=None):
            s, b = _bn_fold(sd, bnpre)
            return ops.pack_conv_weight(sd[wkey], self.dt, device=self.dev, cin_pad=cin_pad, out_scale=s), f32(b)

        self.stem_w, self.stem_b = conv_bn(p + "conv1.weight", p + "bn1.", cin_pad=8)
        self.stem_slope = f32(sd[p + "prelu.weight"])
        self.blocks = []
        inpl = 64
        for li, (planes, n) in enumerate(zip((64, 128, 256, 512), layers), start=1):
            for j in range(n):
                bp = p + f"layer{li}.{j}."
                s1, sh1 = _bn_fold(sd, bp + "bn1.")
                w1, b1 = conv_bn(bp + "conv1.weight", bp + "bn2.")
                w2, b2 = conv_bn(bp + "conv2.weight", bp + "bn3.")
                blk = {"cin": inpl, "cout": planes, "stride": 2 if j == 0 else 1, "s1": f32(s1), "sh1": f32(sh1),
                       "w1": w1, "b1": b1, "slope": f32(sd[bp + "prelu.weight"]), "w2": w2, "b2": b2}
                if j == 0:
                    wd, bd = conv_bn(bp + "downsample.0.weight", bp + "downsample.1.")
                    blk["wd"], blk["bd"] = wd, bd
                self.blocks.append(blk)
                inpl = planes
        # bn2 -> flatten (c*49+p) -> fc -> features(BN1d)
        s2, sh2 = _bn_fold(sd, p + "bn2.")
        Wfc = sd[p + "fc.weight"].float()                      # [512][512*49], column = c*49 + pix
        nf = Wfc.shape[0]
        Wr = Wfc.view(nf, 512, 49)
        bias = sd[p + "fc.bias"].float() + (Wr * sh2.view(1, 512, 1)).sum(dim=(1, 2))
        Wr = Wr * s2.view(1, 512, 1)
        sf, shf = _bn_fold(sd, p + "features.")
        Wr = Wr * sf.view(nf, 1, 1)
        bias = bias * sf + shf
        self.fc_w = ops.to_device(Wr.permute(0, 2, 1).reshape(nf, 49 * 512), self.dev, self.dt)  # column = pix*512 + c
        self.fc_b = f32(bias)

    FUSE_EPILOGUES = True    # PReLU and the next block's bn1 inside the conv epilogues (no channel_affine_act launches)

    @torch.no_grad()
    def forward(self, x, geo):
        """x: [F*112*112][8] channels-last (RGB + zero pad), geo=(F,112,112) -> features [F][512] fp32."""
        if not self.FUSE_EPILOGUES:
            return self._forward_unfused(x, geo)
        from .lib import CB_ACT_PRELU
        # The residual stream is fp32 (100 blocks deep); tensor-core operands are fp16.  Every IBasicBlock
        # (iresnet.py:26-64) is two launches: conv1 (+bn2 folded, PReLU in the epilogue) and conv2 (+bn3 folded, + shortcut)
        # whose epilogue ALSO writes bn1 of the NEXT block applied to the result as the 16-bit operand that block reads.
        blocks = self.blocks
        nb = len(blocks)

        def t_buf(g, c):
            return torch.empty(g.rows, c, dtype=self.dt, device=self.dev)
        t = t_buf(geo, 64)
        h, _ = ops.conv2d(x, geo, self.stem_w, 64, bias=self.stem_b, out_dtype=torch.float32, act=CB_ACT_PRELU,
                          act_param=self.stem_slope, out2=t, out2_affine=(blocks[0]["s1"], blocks[0]["sh1"]))
        for i, b in enumerate(blocks):
            u, _ = ops.conv2d(t, geo, b["w1"], b["cout"], bias=b["b1"], out_dtype=self.dt, act=CB_ACT_PRELU,
                              act_param=b["slope"])
            if "wd" in b:
                idn, ogeo = ops.conv2d(ops.cast(h, self.dt), geo, b["wd"], b["cout"], bias=b["bd"], ksize=1, stride=2,
                                       pad=(0, 0, 0, 0), out_dtype=torch.float32)
            else:
                idn, ogeo = h, geo
            t = t_buf(ogeo, b["cout"])
            aff = (blocks[i + 1]["s1"], blocks[i + 1]["sh1"]) if i + 1 < nb else None     # last block: plain 16-bit copy
            h, geo = ops.conv2d(u, geo, b["w2"], b["cout"], bias=b["b2"], stride=b["stride"], out_dtype=torch.float32,
                                residual=idn, out2=t, out2_affine=aff)
            assert (geo.h, geo.w) == (ogeo.h, ogeo.w)
        flat = t.view(geo.n, geo.hw * t.shape[1])
        return ops.linear(flat, self.fc_w, self.fc_b, out_dtype=torch.float32)

    @torch.no_grad()
    def _forward_unfused(self, x, geo):
        # the residual stream is fp32 (100 blocks deep); tensor-core operands are fp16
        h, _ = ops.conv2d(x, geo, self.stem_w, 64, bias=self.stem_b, out_dtype=torch.float32)
        ops.channel_affine_act(h, slope=self.stem_slope, out=h)
        for b in self.blocks:
            t = ops.channel_affine_act(h, scale=b["s1"], shift=b["sh1"], out_dtype=self.dt)
            u, _ = ops.conv2d(t, geo, b["w1"], b["cout"], bias=b["b1"], out_dtype=self.dt)
            ops.channel_affine_act(u, slope=b["slope"], out=u)
            if "wd" in b:
                idn, ogeo = ops.conv2d(ops.cast(h, self.dt), geo, b["wd"], b["cout"], bias=b["bd"], ksize=1, stride=2,
                                       pad=(0, 0, 0, 0), out_dtype=torch.float32)
            else:
                idn, ogeo = h, geo
            h, geo = ops.conv2d(u, geo, b["w2"], b["cout"], bias=b["b2"], stride=b["stride"],
                                out_dtype=torch.float32, residual=idn)
            assert (geo.h, geo.w) == (ogeo.h, ogeo.w)
        flat = ops.cast(h, self.dt).view(geo.n, geo.hw * h.shape[1])
        return ops.linear(flat, self.fc_w, self.fc_b, out_dtype=torch.float32)
