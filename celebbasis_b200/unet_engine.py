"""SD-v1 UNet forward + activation-gradient backward on the sm_90a kernels.

This is the executor behind ldm.modules.diffusionmodules.openaimodel.UNetModel in the host mirror.
It follows the reference's module graph exactly (openaimodel.py:413-742 UNetModel, :163-275 ResBlock,
:91-160 Up/Downsample; attention.py:152-261 CrossAttention/BasicTransformerBlock/SpatialTransformer)
but runs it as an explicit tape of kernel launches:

  * activations are channels-last matrices [N*H*W][C]; the residual stream, norm inputs and block
    outputs stay fp32, every tensor-core operand is fp16 (or bf16), accumulation is fp32 in registers;
  * all 22 ResBlock `emb_layers` linears are one GEMM per step whose output slice is the per-image
    bias of that block's first conv (fused in the conv epilogue together with the conv bias);
  * q/k/v (self) and k/v (cross) projections are single GEMMs over concatenated weights;
  * backward computes only what the reference's autograd needs with frozen weights
    (SURVEY.md §8 a29): activation gradients down to d(context); no weight gradients, no d(emb).
    Gradients are carried fp16 with a static loss scale; residual-stream gradients are fp32.
"""
import os

import torch

from . import ops
from .lib import CB_ACT_SILU, CB_MAJOR_MN


def _round_up(a, b):
    return (a + b - 1) // b * b


class _Attn:
    """softmax(q k^T * scale) v for (image, head) batches.  What is kept for the backward pass is either the
    log-sum-exp + output (flash backward, nothing quadratic in HBM) or the probabilities (materialised path)."""

    FLASH = True       # fused wgmma flash kernel for head dims <= 128 (set False to force the materialised path)
    FLASH_BWD = True   # recompute-in-registers backward (cb_attention_bwd) instead of P / dP / dS round trips through HBM
    FLASH_BWD_MIN_NK = 256   # short key sequences (cross attention on 77 tokens): the materialised path has more CTAs

    @staticmethod
    def fwd(q, k, v, *, images, heads, dh, nq, nk, scale, out, causal=False, need_p=True):
        """Returns the state the backward pass needs: ("lse", lse, out) or the probabilities
        [images*heads*nq][round_up(nk,8)] (None when not need_p)."""
        if _Attn.FLASH and dh <= 128 and dh % 8 == 0:
            if need_p and _Attn.FLASH_BWD and nk >= _Attn.FLASH_BWD_MIN_NK:
                _, lse = ops.attention_fwd(q, k, v, out, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale,
                                           causal=causal, want_lse=True)
                return ("lse", lse, out, causal)
            if need_p and _Attn.FLASH_BWD:
                # short key sequence (cross attention): keep P and lse; the backward rebuilds dS in registers (dQ kernel) and
                # exports it, dK / dV are two small GEMMs over P and dS
                P, lse = ops.attention_fwd(q, k, v, out, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale,
                                           causal=causal, want_p=True, want_lse=True)
                return ("p+lse", P, lse, out, causal)
            P, _ = ops.attention_fwd(q, k, v, out, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale,
                                     causal=causal, want_p=need_p)
            return P
        ldp = _round_up(nk, 8)
        P = torch.empty(images * heads * nq, ldp, dtype=q.dtype, device=q.device)
        ops.bmm(q, k, P, M=nq, N=nk, K=dh, heads=heads, images=images, lda=q.stride(0), ldb=k.stride(0), ldd=ldp,
                a_hs=dh, b_hs=dh, d_hs=nq * ldp, a_is=nq * q.stride(0), b_is=nk * k.stride(0),
                d_is=heads * nq * ldp, alpha=scale)
        ops.softmax_(P, images * heads * nq, nk, ldp, nq if causal else 0)
        ops.bmm(P, v, out, M=nq, N=dh, K=nk, heads=heads, images=images, lda=ldp, ldb=v.stride(0),
                ldd=out.stride(0), a_hs=nq * ldp, b_hs=dh, d_hs=dh, a_is=heads * nq * ldp, b_is=nk * v.stride(0),
                d_is=nq * out.stride(0), b_major=CB_MAJOR_MN)
        return P

    @staticmethod
    def bwd(dO, q, k, v, P, *, images, heads, dh, nq, nk, scale, dq, dk, dv, offload=None):
        """offload: optional _SideQueue -- the dK / dV GEMMs of a cross-attention block only feed the context gradient
        that is assembled at the very end of the backward pass, so they leave the critical path."""
        if isinstance(P, tuple) and P[0] == "p+lse":
            _, Pm, lse, out, causal = P
            ldp = Pm.shape[1]
            dS = torch.empty_like(Pm)
            ops.attention_bwd_dq(q, k, v, out, dO, lse, dq, dS, images=images, heads=heads, dh=dh, nq=nq, nk=nk,
                                 scale=scale, causal=causal)

            def dkdv():
                # dV = P^T dO ; dK = dS^T Q (dS already carries the softmax scale)
                ops.bmm(Pm, dO, dv, M=nk, N=dh, K=nq, heads=heads, images=images, lda=ldp, ldb=dO.stride(0),
                        ldd=dv.stride(0), a_hs=nq * ldp, b_hs=dh, d_hs=dh, a_is=heads * nq * ldp, b_is=nq * dO.stride(0),
                        d_is=nk * dv.stride(0), a_major=CB_MAJOR_MN, b_major=CB_MAJOR_MN)
                ops.bmm(dS, q, dk, M=nk, N=dh, K=nq, heads=heads, images=images, lda=ldp, ldb=q.stride(0),
                        ldd=dk.stride(0), a_hs=nq * ldp, b_hs=dh, d_hs=dh, a_is=heads * nq * ldp, b_is=nq * q.stride(0),
                        d_is=nk * dk.stride(0), a_major=CB_MAJOR_MN, b_major=CB_MAJOR_MN)
            if offload is not None:
                offload.submit(dkdv, keep=(Pm, dO, dS, q, dv, dk))
            else:
                dkdv()
            return
        if isinstance(P, tuple):
            _, lse, out, causal = P
            if dq is None:
                dq = torch.empty_like(q)
            ops.attention_bwd(q, k, v, out, dO, lse, dq, dk, dv, images=images, heads=heads, dh=dh, nq=nq, nk=nk,
                              scale=scale, causal=causal)
            return
        ldp = P.shape[1]
        dP = torch.empty_like(P)
        # dP = dO V^T
        ops.bmm(dO, v, dP, M=nq, N=nk, K=dh, heads=heads, images=images, lda=dO.stride(0), ldb=v.stride(0), ldd=ldp,
                a_hs=dh, b_hs=dh, d_hs=nq * ldp, a_is=nq * dO.stride(0), b_is=nk * v.stride(0),
                d_is=heads * nq * ldp)
        # dV = P^T dO   (both operands read MN-major straight from their forward layouts)
        ops.bmm(P, dO, dv, M=nk, N=dh, K=nq, heads=heads, images=images, lda=ldp, ldb=dO.stride(0),
                ldd=dv.stride(0), a_hs=nq * ldp, b_hs=dh, d_hs=dh, a_is=heads * nq * ldp, b_is=nq * dO.stride(0),
                d_is=nk * dv.stride(0), a_major=CB_MAJOR_MN, b_major=CB_MAJOR_MN)
        ops.softmax_bwd_(dP, P, images * heads * nq, nk, ldp)  # dP <- dS
        # dK = scale * dS^T Q
        ops.bmm(dP, q, dk, M=nk, N=dh, K=nq, heads=heads, images=images, lda=ldp, ldb=q.stride(0),
                ldd=dk.stride(0), a_hs=nq * ldp, b_hs=dh, d_hs=dh, a_is=heads * nq * ldp, b_is=nq * q.stride(0),
                d_is=nk * dk.stride(0), a_major=CB_MAJOR_MN, b_major=CB_MAJOR_MN, alpha=scale)
        if dq is None:
            return
        # dQ = scale * dS K
        ops.bmm(dP, k, dq, M=nq, N=dh, K=nk, heads=heads, images=images, lda=ldp, ldb=k.stride(0),
                ldd=dq.stride(0), a_hs=nq * ldp, b_hs=dh, d_hs=dh, a_is=heads * nq * ldp, b_is=nk * k.stride(0),
                d_is=nq * dq.stride(0), b_major=CB_MAJOR_MN, alpha=scale)


class _SideQueue:
    """Runs small launches that are off the critical path on a second stream (own workspace lane), ordered after the point
    of submission; join() makes the current stream wait for all of them.  Operand tensors are kept alive until join()
    (their memory must not be recycled by the submitting stream while the side stream still reads it)."""

    def __init__(self, device, lane):
        self.stream = torch.cuda.Stream(device=device, priority=-1)
        self.lane = lane
        self.keep = []
        self.pending = False

    def submit(self, fn, keep=()):
        cur = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(cur)
        self.stream.wait_event(ev)
        with torch.cuda.stream(self.stream), ops.lane(self.lane):
            fn()
        self.keep.append(keep)
        self.pending = True

    def join(self):
        if self.pending:
            ev = torch.cuda.Event()
            ev.record(self.stream)
            torch.cuda.current_stream().wait_event(ev)
            self.pending = False
        self.keep.clear()


class UNetEngine:
    SIDE_DKDV = True     # cross-attention dK / dV GEMMs on a side stream (they only feed d(context), assembled last)
    CAT_INPLACE = os.environ.get("CB_UNET_CAT_INPLACE", "1") != "0"   # skip-connection concat through GEMM epilogues

    def __init__(self, cfg, state_dict, device, dtype=torch.float16, loss_scale=1024.0):
        self.cfg = dict(cfg)
        self.dev = torch.device(device)
        self.dt = dtype
        self.loss_scale = float(loss_scale)
        self.mc = cfg["model_channels"]
        self.heads = cfg["num_heads"]
        self.ctx_dim = cfg["context_dim"]
        self.in_ch = cfg["in_channels"]
        self.out_ch = cfg["out_channels"]
        self.in_pad = _round_up(self.in_ch, 8)
        self.out_pad = 16
        self._build(state_dict)
        self.tape = None
        self._sideq = None

    # ------------------------------------------------------------------------------------------
    # weight preparation
    # ------------------------------------------------------------------------------------------
    def _w16(self, t):
        return ops.to_device(t, self.dev, self.dt)

    def _f32(self, t):
        return ops.to_device(t, self.dev)

    def _build(self, sd):
        cfg = self.cfg
        mc, mult = self.mc, cfg["channel_mult"]
        nres = cfg["num_res_blocks"]
        attn_res = set(cfg["attention_resolutions"])
        g = lambda k: sd[k]

        self.te0_w, self.te0_b = self._w16(g("time_embed.0.weight")), self._f32(g("time_embed.0.bias"))
        self.te2_w, self.te2_b = self._w16(g("time_embed.2.weight")), self._f32(g("time_embed.2.bias"))

        emb_ws, emb_bs = [], []
        self._emb_off = 0
        kvw = []              # cross-attention to_k / to_v of every transformer block: ONE [sum 2C][768] GEMM per step
        self._kv_off = 0

        def res(prefix, cin, cout):
            w = {"kind": "res", "cin": cin, "cout": cout}
            w["g1"], w["b1"] = self._f32(g(prefix + "in_layers.0.weight")), self._f32(g(prefix + "in_layers.0.bias"))
            w["w1"] = ops.pack_conv_weight(g(prefix + "in_layers.2.weight"), self.dt, device=self.dev)
            emb_ws.append(g(prefix + "emb_layers.1.weight"))
            emb_bs.append(g(prefix + "emb_layers.1.bias") + g(prefix + "in_layers.2.bias"))
            w["emb_off"] = self._emb_off
            self._emb_off += cout
            w["g2"], w["b2"] = self._f32(g(prefix + "out_layers.0.weight")), self._f32(g(prefix + "out_layers.0.bias"))
            w["w2"] = ops.pack_conv_weight(g(prefix + "out_layers.3.weight"), self.dt, device=self.dev)
            w["bias2"] = self._f32(g(prefix + "out_layers.3.bias"))
            if cin != cout:
                w["ws"] = self._w16(g(prefix + "skip_connection.weight").reshape(cout, cin))
                w["bs"] = self._f32(g(prefix + "skip_connection.bias"))
            else:
                w["ws"] = None
            return w

        def xf(prefix, c):
            w = {"kind": "xf", "c": c, "dh": c // self.heads}
            w["gn"], w["bn"] = self._f32(g(prefix + "norm.weight")), self._f32(g(prefix + "norm.bias"))
            w["wpi"], w["bpi"] = self._w16(g(prefix + "proj_in.weight").reshape(c, c)), self._f32(g(prefix + "proj_in.bias"))
            tb = prefix + "transformer_blocks.0."
            for i in (1, 2, 3):
                w[f"ln{i}g"], w[f"ln{i}b"] = self._f32(g(tb + f"norm{i}.weight")), self._f32(g(tb + f"norm{i}.bias"))
            w["wqkv"] = self._w16(torch.cat([g(tb + "attn1.to_q.weight"), g(tb + "attn1.to_k.weight"),
                                             g(tb + "attn1.to_v.weight")], 0))
            w["wo1"], w["bo1"] = self._w16(g(tb + "attn1.to_out.0.weight")), self._f32(g(tb + "attn1.to_out.0.bias"))
            w["wq2"] = self._w16(g(tb + "attn2.to_q.weight"))
            kvw.append(torch.cat([g(tb + "attn2.to_k.weight"), g(tb + "attn2.to_v.weight")], 0))
            w["kv_off"] = self._kv_off          # this block's [K | V] columns in the batched context projection
            self._kv_off += 2 * c
            w["wo2"], w["bo2"] = self._w16(g(tb + "attn2.to_out.0.weight")), self._f32(g(tb + "attn2.to_out.0.bias"))
            # GEGLU in the FF-in GEMM's epilogue: rows interleaved into (32 values, 32 gates) groups (ops.linear_geglu)
            w["wff1"] = self._w16(ops.glu_interleave_rows(g(tb + "ff.net.0.proj.weight")))
            w["bff1"] = self._f32(ops.glu_interleave_rows(g(tb + "ff.net.0.proj.bias")))
            w["wff2"], w["bff2"] = self._w16(g(tb + "ff.net.2.weight")), self._f32(g(tb + "ff.net.2.bias"))
            w["wpo"], w["bpo"] = self._w16(g(prefix + "proj_out.weight").reshape(c, c)), self._f32(g(prefix + "proj_out.bias"))
            return w

        def resample(kind, prefix, c):
            key = prefix + ("op." if kind == "down" else "conv.")
            return {"kind": kind, "c": c, "w": ops.pack_conv_weight(g(key + "weight"), self.dt, device=self.dev),
                    "b": self._f32(g(key + "bias"))}

        # stem
        self.stem_w = ops.pack_conv_weight(g("input_blocks.0.0.weight"), self.dt, device=self.dev, cin_pad=self.in_pad)
        self.stem_b = self._f32(g("input_blocks.0.0.bias"))

        self.input_blocks = []   # list of layer lists (block 0 = stem handled separately)
        chans = [mc]
        ch, ds, idx = mc, 1, 1
        for level, m in enumerate(mult):
            for _ in range(nres):
                layers = [res(f"input_blocks.{idx}.0.", ch, m * mc)]
                ch = m * mc
                if ds in attn_res:
                    layers.append(xf(f"input_blocks.{idx}.1.", ch))
                self.input_blocks.append(layers)
                chans.append(ch)
                idx += 1
            if level != len(mult) - 1:
                self.input_blocks.append([resample("down", f"input_blocks.{idx}.0.", ch)])
                chans.append(ch)
                idx += 1
                ds *= 2
        self.middle = [res("middle_block.0.", ch, ch), xf("middle_block.1.", ch), res("middle_block.2.", ch, ch)]
        self.output_blocks = []
        self.cat_split = []      # (channels of h, channels of the popped skip) per output block
        idx = 0
        for level, m in list(enumerate(mult))[::-1]:
            for i in range(nres + 1):
                ich = chans.pop()
                self.cat_split.append((ch, ich))
                layers = [res(f"output_blocks.{idx}.0.", ch + ich, mc * m)]
                ch = mc * m
                if ds in attn_res:
                    layers.append(xf(f"output_blocks.{idx}.1.", ch))
                if level and i == nres:
                    layers.append(resample("up", f"output_blocks.{idx}.{len(layers)}.", ch))
                    ds //= 2
                self.output_blocks.append(layers)
                idx += 1
        self.wkv_all = self._w16(torch.cat(kvw, 0)) if kvw else None
        del kvw
        # head
        self.out_g, self.out_b = self._f32(g("out.0.weight")), self._f32(g("out.0.bias"))
        self.out_w = ops.pack_conv_weight(g("out.2.weight"), self.dt, device=self.dev, cout_pad=self.out_pad)
        ob = torch.zeros(self.out_pad, dtype=torch.float32, device=self.dev)
        ob[: self.out_ch] = self._f32(g("out.2.bias"))
        self.out_bias = ob
        # all ResBlock timestep projections as one GEMM
        self.emb_w = self._w16(torch.cat(emb_ws, 0))
        self.emb_b = self._f32(torch.cat(emb_bs, 0))
        self.emb_total = self._emb_off

    # ------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------
    def _res_fwd(self, w, x, geo, emb_all, tape, out=None, out2=None):
        cout = w["cout"]
        a16, st1 = ops.groupnorm(x, geo, w["g1"], w["b1"], eps=1e-5, silu=True, out_dtype=self.dt)
        bias1 = emb_all[:, w["emb_off"]: w["emb_off"] + cout]
        h16, _ = ops.conv2d(a16, geo, w["w1"], cout, bias=bias1, bias_per_image=True, ldbias=emb_all.stride(0),
                            out_dtype=self.dt)
        b16, st2 = ops.groupnorm(h16, geo, w["g2"], w["b2"], eps=1e-5, silu=True, out_dtype=self.dt)
        if w["ws"] is None:
            resid = x
        else:
            resid = ops.linear(ops.cast(x, self.dt), w["ws"], w["bs"], out_dtype=torch.float32)
        out, _ = ops.conv2d(b16, geo, w["w2"], cout, bias=w["bias2"], out_dtype=torch.float32, residual=resid, out=out,
                            out2=out2)
        if tape is not None:
            tape.append(("res", w, geo, x, st1, h16, st2))
        return out

    def _res_bwd(self, rec, dout, dout16=None):
        """dout16: 16-bit copy of dout when the producing GroupNorm-backward kernel emitted one (else cast here)."""
        _, w, geo, x, st1, h16, st2 = rec
        if dout16 is None:
            dout16 = ops.cast(dout, self.dt)
        db16, _ = ops.conv2d_dgrad(dout16, geo, w["w2"], w["cout"])
        dh16 = ops.groupnorm_bwd(db16, h16, geo, w["g2"], w["b2"], st2, silu=True, dx_dtype=self.dt)
        da16, _ = ops.conv2d_dgrad(dh16, geo, w["w1"], w["cin"])
        if w["ws"] is None:
            dx = dout
        else:
            dx = ops.linear_dgrad(dout16, w["ws"], out_dtype=torch.float32)
        ops.groupnorm_bwd(da16, x, geo, w["g1"], w["b1"], st1, silu=True, dx=dx, accumulate=True)
        return dx

    def _xf_fwd(self, w, x, geo, kv_all, tape, out=None, out2=None):
        c, dh, H = w["c"], w["dh"], self.heads
        B, nq = geo.n, geo.hw
        scale = dh ** -0.5
        n16, stn = ops.groupnorm(x, geo, w["gn"], w["bn"], eps=1e-6, silu=False, out_dtype=self.dt)
        h0 = ops.linear(n16, w["wpi"], w["bpi"], out_dtype=torch.float32)
        # self attention
        l1, s1 = ops.layernorm(h0, w["ln1g"], w["ln1b"], out_dtype=self.dt)
        qkv = ops.linear(l1, w["wqkv"])
        o1 = torch.empty(geo.rows, c, dtype=self.dt, device=self.dev)
        P1 = _Attn.fwd(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], images=B, heads=H, dh=dh, nq=nq, nk=nq,
                       scale=scale, out=o1)
        h1 = ops.linear(o1, w["wo1"], w["bo1"], out_dtype=torch.float32, residual=h0)
        # cross attention
        l2, s2 = ops.layernorm(h1, w["ln2g"], w["ln2b"], out_dtype=self.dt)
        q2 = ops.linear(l2, w["wq2"])
        kv_all = kv_all()                                        # first use waits for the text encoder (see forward)
        nk = kv_all.shape[0] // geo.n
        kv2 = kv_all[:, w["kv_off"]:w["kv_off"] + 2 * c]       # K | V of this block (projected once for all blocks)
        o2 = torch.empty(geo.rows, c, dtype=self.dt, device=self.dev)
        P2 = _Attn.fwd(q2, kv2[:, :c], kv2[:, c:], images=B, heads=H, dh=dh, nq=nq, nk=nk, scale=scale, out=o2)
        h2 = ops.linear(o2, w["wo2"], w["bo2"], out_dtype=torch.float32, residual=h1)
        # GEGLU feed-forward
        l3, s3 = ops.layernorm(h2, w["ln3g"], w["ln3b"], out_dtype=self.dt)
        u16, g16 = ops.linear_geglu(l3, w["wff1"], w["bff1"], keep_preact=tape is not None)
        h3 = ops.linear(u16, w["wff2"], w["bff2"], out_dtype=self.dt, residual=h2)
        out = ops.linear(h3, w["wpo"], w["bpo"], out_dtype=torch.float32, residual=x, out=out, out2=out2)
        if tape is not None:
            tape.append(("xf", w, geo, x, stn, h0, s1, qkv, P1, h1, s2, q2, kv2, P2, h2, s3, g16, nk))
        return out

    def _xf_bwd(self, rec, dout, dkv_all, to_input=True):
        """to_input=False: this is the first transformer block of the network -- only the context gradient is wanted, so
        the chain stops after the cross-attention K/V gradients (what autograd prunes in the reference: x_noisy, the
        timestep embedding and every weight before this point do not require grad)."""
        _, w, geo, x, stn, h0, s1, qkv, P1, h1, s2, q2, kv2, P2, h2, s3, g16, nk = rec
        c, dh, H = w["c"], w["dh"], self.heads
        B, nq = geo.n, geo.hw
        scale = dh ** -0.5
        dx = dout
        dr = ops.linear_dgrad(ops.cast(dout, self.dt), w["wpo"], out_dtype=torch.float32)  # d h3 (fp32 running)
        dx16 = torch.empty(dout.shape, dtype=self.dt, device=self.dev) if to_input else None
        # feed-forward
        du = ops.linear_dgrad(ops.cast(dr, self.dt), w["wff2"])
        dg = ops.geglu_bwd(du, g16, interleaved=True)
        dl3 = ops.linear_dgrad(dg, w["wff1"])
        dr16 = torch.empty(dr.shape, dtype=self.dt, device=self.dev)      # 16-bit copy of the running gradient, written
        ops.layernorm_bwd(dl3, h2, w["ln3g"], s3, dx=dr, accumulate=True, dx_lp=dr16)   # by the kernel that updates it
        # cross attention
        dO = ops.linear_dgrad(dr16, w["wo2"])
        dq2 = torch.empty_like(q2) if to_input else None
        dkv2 = dkv_all[:, w["kv_off"]:w["kv_off"] + 2 * c]     # gradient slice of the batched context projection
        _Attn.bwd(dO, q2, kv2[:, :c], kv2[:, c:], P2, images=B, heads=H, dh=dh, nq=nq, nk=nk, scale=scale,
                  dq=dq2, dk=dkv2[:, :c], dv=dkv2[:, c:], offload=self._sideq_get())
        if not to_input:
            return None
        dl2 = ops.linear_dgrad(dq2, w["wq2"])
        ops.layernorm_bwd(dl2, h1, w["ln2g"], s2, dx=dr, accumulate=True, dx_lp=dr16)
        # self attention
        dO = ops.linear_dgrad(dr16, w["wo1"])
        dqkv = torch.empty_like(qkv)
        _Attn.bwd(dO, qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], P1, images=B, heads=H, dh=dh, nq=nq, nk=nq,
                  scale=scale, dq=dqkv[:, :c], dk=dqkv[:, c:2 * c], dv=dqkv[:, 2 * c:])
        dl1 = ops.linear_dgrad(dqkv, w["wqkv"])
        ops.layernorm_bwd(dl1, h0, w["ln1g"], s1, dx=dr, accumulate=True, dx_lp=dr16)
        # proj_in + group norm
        dn = ops.linear_dgrad(dr16, w["wpi"])
        ops.groupnorm_bwd(dn, x, geo, w["gn"], w["bn"], stn, silu=False, dx=dx, accumulate=True, dx_lp=dx16)
        self._last_dx16 = dx16      # 16-bit copy of the returned gradient (the next ResBlock's dgrad operand)
        return dx

    def _sideq_get(self):
        if not self.SIDE_DKDV:
            return None
        if self._sideq is None:
            self._sideq = _SideQueue(self.dev, lane=4)
        return self._sideq

    def _down_fwd(self, w, x, geo, tape, out=None, out2=None):
        out, ogeo = ops.conv2d(ops.cast(x, self.dt), geo, w["w"], w["c"], bias=w["b"], stride=2,
                               out_dtype=torch.float32, out=out, out2=out2)
        if tape is not None:
            tape.append(("down", w, geo, ogeo))
        return out, ogeo

    def _down_bwd(self, rec, dout):
        _, w, geo, ogeo = rec
        z, zgeo = ops.zero_insert2x(ops.cast(dout, self.dt), ogeo)
        dx, _ = ops.conv2d_dgrad(z, zgeo, w["w"], w["c"], out_dtype=torch.float32)
        return dx

    def _up_fwd(self, w, x, geo, tape, out=None, out2=None):
        u, ugeo = ops.upsample2x(ops.cast(x, self.dt), geo)
        out, _ = ops.conv2d(u, ugeo, w["w"], w["c"], bias=w["b"], out_dtype=torch.float32, out=out, out2=out2)
        if tape is not None:
            tape.append(("up", w, geo, ugeo))
        return out, ugeo

    def _up_bwd(self, rec, dout):
        _, w, geo, ugeo = rec
        du, _ = ops.conv2d_dgrad(ops.cast(dout, self.dt), ugeo, w["w"], w["c"])
        return ops.upsample2x_bwd(du, geo, dx_dtype=torch.float32)

    def _run_layers(self, layers, h, geo, emb_all, kv_all, tape, out=None, out2=None):
        """out / out2: destinations of the LAST layer's result (see forward: skip-connection concat without copies);
        they are callables geo -> 2-D view because the geometry of an up / down layer's output is only known here."""
        for i, w in enumerate(layers):
            k = w["kind"]
            last = i == len(layers) - 1
            if k in ("down", "up"):
                ogeo = ops.Geo(geo.n, geo.h // 2, geo.w // 2) if k == "down" else ops.Geo(geo.n, 2 * geo.h, 2 * geo.w)
            else:
                ogeo = geo
            o = out(ogeo) if (last and out is not None) else None
            o2 = out2(ogeo) if (last and out2 is not None) else None
            if k == "res":
                h = self._res_fwd(w, h, geo, emb_all, tape, out=o, out2=o2)
            elif k == "xf":
                h = self._xf_fwd(w, h, geo, kv_all, tape, out=o, out2=o2)
            elif k == "down":
                h, geo = self._down_fwd(w, h, geo, tape, out=o, out2=o2)
            else:
                h, geo = self._up_fwd(w, h, geo, tape, out=o, out2=o2)
        return h, geo

    def forward(self, x, t, context, need_grad=True, context_ready=None):
        """x: (B,in_ch,H,W) fp32 NCHW; t: (B,) int64; context: (B,T,ctx_dim) fp32.  Returns eps (B,out_ch,H,W) fp32.
        context_ready: optional CUDA event after which `context` holds the text encoder's output (it may still be being
        computed on another stream: nothing before the first cross-attention -- timestep MLP, stem, first ResBlock, the
        first block's self-attention -- needs it)."""
        assert x.dtype == torch.float32 and context.dtype == torch.float32
        B = x.shape[0]
        tape = [] if need_grad else None
        # timestep embedding MLP + all ResBlock projections
        temb = ops.timestep_embedding(t, self.mc, dtype=self.dt)
        e1 = ops.linear(temb, self.te0_w, self.te0_b, act=CB_ACT_SILU)
        # SiLU(emb) is what every ResBlock consumes (openaimodel.py:222-226): fuse it into the 2nd linear
        e2 = ops.linear(e1, self.te2_w, self.te2_b, act=CB_ACT_SILU)
        emb_all = ops.linear(e2, self.emb_w, self.emb_b, out_dtype=torch.float32)
        kv_state = {}

        def kv_all():
            # the context is the same for all 16 transformer blocks: project it to every block's K and V in one GEMM
            if "kv" not in kv_state:
                if context_ready is not None:
                    torch.cuda.current_stream().wait_event(context_ready)
                ctx16 = ops.cast(context.reshape(-1, self.ctx_dim), self.dt)
                kv_state["kv"] = ops.linear(ctx16, self.wkv_all)
            return kv_state["kv"]
        x16, geo = ops.nchw_to_nhwc(x.contiguous(), self.in_pad, self.dt)
        # Skip connections without copies (torch.cat([h, hs.pop()], dim=1), openaimodel.py:737-739): the concat buffer of
        # every output block is allocated up front; the GEMM epilogue that produces a skip activation also stores it into
        # columns [c1, c1+c2) of the block that will pop it (second destination), and the epilogue that produces the
        # previous block's result writes columns [0, c1) directly.
        n_out = len(self.output_blocks)
        cats = [None] * n_out

        def cat_buf(k, g):
            if cats[k] is None:
                c1, c2 = self.cat_split[k]
                cats[k] = torch.empty(g.rows, c1 + c2, dtype=torch.float32, device=self.dev)
            return cats[k]

        def skip_dst(m):          # hs[m] is popped by output block n_out-1-m
            k = n_out - 1 - m
            return lambda g: cat_buf(k, g)[:, self.cat_split[k][0]:]

        def head_dst(k):          # the tensor entering output block k lands in columns [0, c1) of its concat buffer
            return lambda g: cat_buf(k, g)[:, : self.cat_split[k][0]]

        inplace = self.CAT_INPLACE
        h, _ = ops.conv2d(x16, geo, self.stem_w, self.mc, bias=self.stem_b, out_dtype=torch.float32,
                          out2=skip_dst(0)(geo) if inplace else None)
        hs = [h]
        for m, layers in enumerate(self.input_blocks, start=1):
            h, geo = self._run_layers(layers, h, geo, emb_all, kv_all, tape, out2=skip_dst(m) if inplace else None)
            if tape is not None:
                tape.append(("push",))
            hs.append(h)
        h, geo = self._run_layers(self.middle, h, geo, emb_all, kv_all, tape, out=head_dst(0) if inplace else None)
        for k, layers in enumerate(self.output_blocks):
            c1, c2 = self.cat_split[k]
            skip = hs.pop()
            if inplace:
                cat = cats[k]
                assert cat is not None and cat.shape[0] == geo.rows
            else:
                cat = torch.empty(geo.rows, c1 + c2, dtype=torch.float32, device=self.dev)
                ops.axpby(h, 1.0, out=cat[:, :c1])
                ops.axpby(skip, 1.0, out=cat[:, c1:])
            if tape is not None:
                tape.append(("cat", c1, c2))
            h, geo = self._run_layers(layers, cat, geo, emb_all, kv_all, tape,
                                      out=head_dst(k + 1) if (inplace and k + 1 < n_out) else None)
        a16, sto = ops.groupnorm(h, geo, self.out_g, self.out_b, eps=1e-5, silu=True, out_dtype=self.dt)
        y, _ = ops.conv2d(a16, geo, self.out_w, self.out_ch, bias=self.out_bias, out_dtype=torch.float32,
                          cout_rows=self.out_pad)
        eps = ops.nhwc_to_nchw(y, geo, self.out_ch)
        if tape is not None:
            tape.append(("head", geo, h, sto))
            self.tape = (tape, context.shape)
        return eps

    # ------------------------------------------------------------------------------------------
    # backward: d(eps) -> d(context)
    # ------------------------------------------------------------------------------------------
    def backward(self, d_eps):
        """d_eps: (B,out_ch,H,W) fp32 (unscaled).  Returns d_context (B,T,ctx_dim) fp32 (unscaled)."""
        assert self.tape is not None, "UNetEngine.backward without a recorded forward"
        tape, ctx_shape = self.tape
        self.tape = None
        S = self.loss_scale
        dkv_all = torch.empty(ctx_shape[0] * ctx_shape[1], self._kv_off, dtype=self.dt, device=self.dev)
        rec = tape.pop()
        _, geo, h_head, sto = rec
        d32, _ = ops.nchw_to_nhwc(d_eps.contiguous(), self.out_pad, torch.float32)
        dy16 = ops.cast(d32, self.dt, scale=S)
        da16, _ = ops.conv2d_dgrad(dy16, geo, self.out_w, self.mc, cout_rows=self.out_pad)
        dh16 = torch.empty(h_head.shape, dtype=self.dt, device=self.dev)
        dh = ops.groupnorm_bwd(da16, h_head, geo, self.out_g, self.out_b, sto, silu=True, dx_dtype=torch.float32, dx_lp=dh16)
        dskips = []
        first_xf = next((i for i, r in enumerate(tape) if r[0] == "xf"), -1)
        while tape:
            rec = tape.pop()
            k = rec[0]
            if k == "res":
                dh = self._res_bwd(rec, dh, dh16)
                dh16 = None
            elif k == "xf":
                if len(tape) == first_xf:
                    # first transformer block in forward order: nothing before it (stem, ResBlock, its own self-attention)
                    # depends on the context, so the backward pass ends with its cross-attention K/V gradients
                    self._xf_bwd(rec, dh, dkv_all, to_input=False)
                    tape.clear()
                    break
                dh = self._xf_bwd(rec, dh, dkv_all)
                dh16 = self._last_dx16
            elif k == "down":
                dh, dh16 = self._down_bwd(rec, dh), None
            elif k == "up":
                dh, dh16 = self._up_bwd(rec, dh), None
            elif k == "cat":
                _, c1, c2 = rec
                dskips.append(dh[:, c1:])
                dh, dh16 = ops.axpby(dh[:, :c1], 1.0), None
            elif k == "push":
                # this activation also fed a skip connection: add that branch's gradient
                dsk = dskips.pop()
                ops.axpby(dh, 1.0, dsk, 1.0, out=dh)
                dh16 = None
        if self._sideq is not None:
            self._sideq.join()
        # d(context) = [dK | dV of every block] . [W_k ; W_v of every block]: one GEMM with K = sum 2C
        dctx = ops.linear_dgrad(dkv_all, self.wkv_all, out_dtype=torch.float32)
        out = ops.axpby(dctx, 1.0 / S)
        return out.view(ctx_shape)
