"""CLIP ViT-L/14 text transformer (12 pre-LN layers, 12 heads x 64, quick-GELU MLP, causal mask) forward and
activation-gradient backward on the sm_90a kernels.

Mirrors what the reference runs through its patched HF forwards: ldm/modules/encoders/modules.py:345-406
(text_encoder_forward: causal mask, encoder, final_layer_norm) and :302-342 (encoder_forward over
transformers==4.18.0 CLIPEncoderLayer: LN1 -> CLIPAttention(q*scale, +mask, softmax, out_proj) -> +res ->
LN2 -> fc1 -> quick_gelu -> fc2 -> +res).  The backward is needed because the trainable signal enters at
the input embeddings (modules.py:290-296, ddpm.py:930-931).
"""
import torch

from . import ops
from .lib import CB_ACT_QUICK_GELU
from .unet_engine import _Attn


class CLIPTextEngine:
    def __init__(self, state_dict, device, *, prefix="text_model.", dtype=torch.float16, loss_scale=1024.0,
                 heads=12, eps=1e-5):
        self.dev = torch.device(device)
        self.dt = dtype
        self.heads = heads
        self.eps = eps
        self.loss_scale = float(loss_scale)
        sd, p = state_dict, prefix
        f32 = lambda t: ops.to_device(t, self.dev)
        w16 = lambda t: ops.to_device(t, self.dev, self.dt)
        self.tok_table = f32(sd[p + "embeddings.token_embedding.weight"])
        self.pos_table = f32(sd[p + "embeddings.position_embedding.weight"])
        self.hidden = self.tok_table.shape[1]
        self.dh = self.hidden // heads
        self.layers = []
        i = 0
        while (p + f"encoder.layers.{i}.layer_norm1.weight") in sd:
            lp = p + f"encoder.layers.{i}."
            L = {
                "ln1g": f32(sd[lp + "layer_norm1.weight"]), "ln1b": f32(sd[lp + "layer_norm1.bias"]),
                "ln2g": f32(sd[lp + "layer_norm2.weight"]), "ln2b": f32(sd[lp + "layer_norm2.bias"]),
                "wqkv": w16(torch.cat([sd[lp + "self_attn.q_proj.weight"], sd[lp + "self_attn.k_proj.weight"],
                                       sd[lp + "self_attn.v_proj.weight"]], 0)),
                "bqkv": f32(torch.cat([sd[lp + "self_attn.q_proj.bias"], sd[lp + "self_attn.k_proj.bias"],
                                       sd[lp + "self_attn.v_proj.bias"]], 0)),
                "wo": w16(sd[lp + "self_attn.out_proj.weight"]), "bo": f32(sd[lp + "self_attn.out_proj.bias"]),
                "w1": w16(sd[lp + "mlp.fc1.weight"]), "b1": f32(sd[lp + "mlp.fc1.bias"]),
                "w2": w16(sd[lp + "mlp.fc2.weight"]), "b2": f32(sd[lp + "mlp.fc2.bias"]),
            }
            self.layers.append(L)
            i += 1
        self.fg, self.fb = f32(sd[p + "final_layer_norm.weight"]), f32(sd[p + "final_layer_norm.bias"])
        self.tape = None

    def forward(self, emb, batch, need_grad=True):
        """emb: [batch*T][hidden] fp32 (token + position embeddings).  Returns [batch*T][hidden] fp32."""
        T = emb.shape[0] // batch
        c, H, dh = self.hidden, self.heads, self.dh
        scale = dh ** -0.5
        tape = [] if need_grad else None
        h = emb
        for L in self.layers:
            l1, s1 = ops.layernorm(h, L["ln1g"], L["ln1b"], eps=self.eps, out_dtype=self.dt)
            qkv = ops.linear(l1, L["wqkv"], L["bqkv"])
            o = torch.empty(h.shape[0], c, dtype=self.dt, device=self.dev)
            P = _Attn.fwd(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], images=batch, heads=H, dh=dh, nq=T, nk=T,
                          scale=scale, out=o, causal=True)
            h1 = ops.linear(o, L["wo"], L["bo"], out_dtype=torch.float32, residual=h)
            l2, s2 = ops.layernorm(h1, L["ln2g"], L["ln2b"], eps=self.eps, out_dtype=self.dt)
            f = ops.linear(l2, L["w1"], L["b1"])
            a = ops.act_fwd(f, CB_ACT_QUICK_GELU)
            h2 = ops.linear(a, L["w2"], L["b2"], out_dtype=torch.float32, residual=h1)
            if tape is not None:
                tape.append((L, h, s1, qkv, P, h1, s2, f))
            h = h2
        out, sf = ops.layernorm(h, self.fg, self.fb, eps=self.eps, out_dtype=torch.float32)
        if tape is not None:
            self.tape = (tape, h, sf, batch, T)
        return out

    def backward(self, dctx):
        """dctx: [batch*T][hidden] fp32 (unscaled).  Returns d(emb) fp32 (unscaled)."""
        assert self.tape is not None, "CLIPTextEngine.backward without a recorded forward"
        tape, h_last, sf, batch, T = self.tape
        self.tape = None
        S = self.loss_scale
        c, H, dh = self.hidden, self.heads, self.dh
        scale = dh ** -0.5
        dys = ops.axpby(dctx, S)
        dh_ = ops.layernorm_bwd(dys, h_last, self.fg, sf, dx_dtype=torch.float32)
        dh16 = ops.cast(dh_, self.dt)     # 16-bit copy of the running gradient; the LayerNorm-backward kernels keep it current
        while tape:
            L, h, s1, qkv, P, h1, s2, f = tape.pop()
            da = ops.linear_dgrad(dh16, L["w2"])
            df = ops.act_bwd(da, f, CB_ACT_QUICK_GELU)
            dl2 = ops.linear_dgrad(df, L["w1"])
            ops.layernorm_bwd(dl2, h1, L["ln2g"], s2, dx=dh_, accumulate=True, dx_lp=dh16)
            dO = ops.linear_dgrad(dh16, L["wo"])
            dqkv = torch.empty_like(qkv)
            _Attn.bwd(dO, qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], P, images=batch, heads=H, dh=dh, nq=T, nk=T,
                      scale=scale, dq=dqkv[:, :c], dk=dqkv[:, c:2 * c], dv=dqkv[:, 2 * c:])
            dl1 = ops.linear_dgrad(dqkv, L["wqkv"])
            ops.layernorm_bwd(dl1, h, L["ln1g"], s1, dx=dh_, accumulate=True, dx_lp=dh16)
        return ops.axpby(dh_, 1.0 / S)
