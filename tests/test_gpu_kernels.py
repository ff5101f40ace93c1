"""GPU: every kernel family of libcelebbasis_b200.so against a plain PyTorch fp32 reference of the same op
(through the C-ABI).  Tolerances: fp16 operands / fp32 accumulate => relative Frobenius error < 2e-3 for GEMM-class
ops (the operands are rounded to fp16 in BOTH implementations so only accumulation order differs -> ~2e-4),
< 2e-3 for norm/pointwise ops whose outputs are stored in fp16; integer/index paths are bit-exact."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from celebbasis_b200 import lib
    assert lib.load().cb_device_ok() == 1, "tests must run on an sm_90 device"
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def rnd(*shape, dtype=torch.float16, scale=1.0, seed=[0]):
    seed[0] += 1
    g = torch.Generator().manual_seed(seed[0])
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


# ---------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K", [(128, 160, 64), (4096, 320, 320), (77, 768, 768), (300, 64, 40), (64, 16, 320),
                                   (1, 1280, 320), (1000, 1280, 2560)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_linear(dev, M, N, K, dtype):
    from celebbasis_b200 import ops
    x, w, b = rnd(M, K, dtype=dtype), rnd(N, K, dtype=dtype, scale=K ** -0.5), rnd(N, dtype=torch.float32)
    y = ops.linear(x, w, b, out_dtype=torch.float32)
    assert rel(y, x.float() @ w.float().t() + b) < 1e-3
    dy = rnd(M, N, dtype=dtype)
    dx = ops.linear_dgrad(dy, w, out_dtype=torch.float32)
    assert rel(dx, dy.float() @ w.float()) < 1e-3


def test_linear_epilogues(dev):
    from celebbasis_b200 import ops
    from celebbasis_b200.lib import CB_ACT_GELU, CB_ACT_QUICK_GELU, CB_ACT_SILU
    x, w, b = rnd(512, 640), rnd(640, 640, scale=640 ** -0.5), rnd(640, dtype=torch.float32)
    r32 = rnd(512, 640, dtype=torch.float32)
    base = x.float() @ w.float().t() + b
    assert rel(ops.linear(x, w, b, out_dtype=torch.float32, act=CB_ACT_SILU, residual=r32), F.silu(base) + r32) < 1e-3
    assert rel(ops.linear(x, w, b, out_dtype=torch.float32, act=CB_ACT_GELU), F.gelu(base)) < 1e-3
    assert rel(ops.linear(x, w, b, act=CB_ACT_QUICK_GELU), base * torch.sigmoid(1.702 * base)) < 2e-3
    assert rel(ops.linear(x, w, None, out_dtype=torch.float32, alpha=0.25), 0.25 * (x.float() @ w.float().t())) < 1e-3


@pytest.mark.parametrize("n,h,w,cin,cout,stride,pad", [
    (1, 64, 64, 320, 320, 1, (1, 1, 1, 1)), (1, 8, 8, 1280, 1280, 1, (1, 1, 1, 1)), (2, 8, 8, 2560, 1280, 1, (1, 1, 1, 1)),
    (1, 64, 64, 8, 320, 1, (1, 1, 1, 1)), (1, 64, 64, 320, 16, 1, (1, 1, 1, 1)),
    (2, 56, 56, 64, 64, 1, (1, 1, 1, 1)), (3, 7, 7, 512, 512, 1, (1, 1, 1, 1)), (2, 14, 14, 256, 256, 1, (1, 1, 1, 1)),
    (1, 256, 256, 128, 128, 1, (1, 1, 1, 1)), (1, 64, 64, 320, 320, 2, (1, 1, 1, 1)),
    (1, 128, 128, 128, 128, 2, (0, 1, 0, 1)), (2, 112, 112, 64, 64, 2, (1, 1, 1, 1)), (1, 1, 1, 256, 256, 1, (1, 1, 1, 1)),
    (2, 2, 2, 256, 128, 1, (1, 1, 1, 1))])
def test_conv3x3(dev, n, h, w, cin, cout, stride, pad):
    """Implicit-GEMM conv incl. zero padding via TMA OOB fill, stride 2 via traversal stride, ragged pixel boxes."""
    from celebbasis_b200 import ops
    x = rnd(n * h * w, cin)
    wt = rnd(cout, cin, 3, 3, scale=(9 * cin) ** -0.5)
    b = rnd(cout, dtype=torch.float32)
    y, og = ops.conv2d(x, ops.Geo(n, h, w), ops.pack_conv_weight(wt, torch.float16), cout, bias=b, stride=stride,
                       pad=pad, out_dtype=torch.float32)
    xr = F.pad(x.float().view(n, h, w, cin).permute(0, 3, 1, 2), (pad[2], pad[3], pad[0], pad[1]))
    ref = F.conv2d(xr, wt.float(), b, stride=stride).permute(0, 2, 3, 1).reshape(-1, cout)
    assert y.shape == ref.shape and rel(y, ref) < 1e-3


@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 32, 32, 640, 640), (1, 64, 64, 320, 320), (1, 16, 16, 1920, 1280),
                                            (2, 8, 8, 1280, 1280)])
def test_conv_dgrad(dev, n, h, w, cin, cout):
    from celebbasis_b200 import ops
    wt = rnd(cout, cin, 3, 3, scale=(9 * cin) ** -0.5)
    dy = rnd(n * h * w, cout)
    dx, _ = ops.conv2d_dgrad(dy, ops.Geo(n, h, w), ops.pack_conv_weight(wt, torch.float16), cin, out_dtype=torch.float32)
    ref = F.conv_transpose2d(dy.float().view(n, h, w, cout).permute(0, 3, 1, 2), wt.float(), padding=1)
    assert rel(dx, ref.permute(0, 2, 3, 1).reshape(-1, cin)) < 1e-3


def test_conv_stride2_dgrad_via_zero_insertion(dev):
    from celebbasis_b200 import ops
    n, h, c = 1, 32, 320
    wt = rnd(c, c, 3, 3, scale=(9 * c) ** -0.5)
    dy = rnd(n * (h // 2) ** 2, c)
    z, zg = ops.zero_insert2x(dy, ops.Geo(n, h // 2, h // 2))
    dx, _ = ops.conv2d_dgrad(z, zg, ops.pack_conv_weight(wt, torch.float16), c, out_dtype=torch.float32)
    ref = F.conv_transpose2d(dy.float().view(n, h // 2, h // 2, c).permute(0, 3, 1, 2), wt.float(), stride=2, padding=1,
                             output_padding=1)
    assert rel(dx, ref.permute(0, 2, 3, 1).reshape(-1, c)) < 1e-3


@pytest.mark.parametrize("nq,nk,dh,heads,images", [(1024, 1024, 40, 8, 1), (256, 77, 160, 8, 2), (77, 77, 64, 12, 2),
                                                   (64, 64, 160, 8, 1)])
def test_attention_fwd_bwd(dev, nq, nk, dh, heads, images):
    """q.k^T softmax p.v as batched wgmma GEMMs (K-major and MN-major operands), forward and backward."""
    from celebbasis_b200.unet_engine import _Attn
    C = heads * dh
    q, k, v = rnd(images * nq, C), rnd(images * nk, C), rnd(images * nk, C)
    do = rnd(images * nq, C)
    o = torch.empty_like(q)
    P = _Attn.fwd(q, k, v, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=dh ** -0.5, out=o)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    _Attn.bwd(do, q, k, v, P, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=dh ** -0.5, dq=dq, dk=dk, dv=dv)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    sp = lambda t, n: t.view(images, n, heads, dh).permute(0, 2, 1, 3)
    att = torch.softmax(sp(qf, nq) @ sp(kf, nk).transpose(-1, -2) * dh ** -0.5, -1)
    ref = (att @ sp(vf, nk)).permute(0, 2, 1, 3).reshape(images * nq, C)
    ref.backward(do.float())
    assert rel(o, ref) < 3e-3
    assert rel(dq, qf.grad) < 6e-3 and rel(dk, kf.grad) < 6e-3 and rel(dv, vf.grad) < 6e-3


# ---------------------------------------------------------------------------------------------------- norms
@pytest.mark.parametrize("n,hw,c,silu,eps,xdt", [
    # forward and backward on the cluster kernels (slabs of groups, statistics through DSMEM)
    (1, 4096, 320, True, 1e-5, torch.float32), (2, 64, 1280, True, 1e-5, torch.float32),
    (1, 1024, 960, False, 1e-6, torch.float32), (1, 4096, 128, True, 1e-6, torch.float16),
    (1, 1, 256, True, 1e-5, torch.float32),
    # also both on the cluster kernels: the UNet's 16^2 / 8^2 concat widths, 30- and 10-channel groups (quads straddle two
    # groups), several images, fewer rows than cluster CTAs
    (1, 256, 2560, True, 1e-5, torch.float32), (1, 64, 1280, True, 1e-5, torch.float16),
    (1, 1024, 1920, True, 1e-5, torch.float32), (4, 64, 320, False, 1e-5, torch.float32),
    (1, 4096, 640, True, 1e-5, torch.float16), (3, 9, 960, True, 1e-6, torch.float32),
    # a VAE 256^2 map: forward on the TMA-streamed statistics + apply pair, backward on the statistics + apply pair
    (1, 65536, 128, True, 1e-6, torch.float32),
    # forward on the cluster kernel (16-bit x fits), backward (x and dy staged) on the statistics + apply pair
    (2, 20001, 256, False, 1e-6, torch.float16)])
def test_groupnorm_fwd_bwd(dev, n, hw, c, silu, eps, xdt):
    from celebbasis_b200 import ops
    x = rnd(n * hw, c, dtype=xdt, scale=2.0) + 0.5
    g, b = rnd(c, dtype=torch.float32) * 0.1 + 1, rnd(c, dtype=torch.float32) * 0.1
    dy = rnd(n * hw, c)
    geo = ops.Geo(n, 1, hw)
    y, st = ops.groupnorm(x, geo, g, b, eps=eps, silu=silu)
    dx = ops.groupnorm_bwd(dy, x, geo, g, b, st, silu=silu)
    xr = x.float().view(n, hw, c).permute(0, 2, 1).requires_grad_(True)
    yr = F.group_norm(xr, 32, g, b, eps)
    yr = F.silu(yr) if silu else yr
    yr.backward(dy.float().view(n, hw, c).permute(0, 2, 1))
    assert rel(y, yr.permute(0, 2, 1).reshape(n * hw, c)) < 1e-3
    assert rel(dx, xr.grad.permute(0, 2, 1).reshape(n * hw, c)) < 2e-3
    acc = torch.ones_like(dx)
    ops.groupnorm_bwd(dy, x, geo, g, b, st, silu=silu, dx=acc, accumulate=True)
    assert rel(acc, dx + 1) < 1e-5


@pytest.mark.parametrize("m,c", [(4096, 320), (77, 768), (64, 1280), (3, 640), (1024, 640), (256, 1280), (130, 2048),
                                 (5, 66), (1025, 64), (9, 4100)])
def test_layernorm_fwd_bwd(dev, m, c):
    from celebbasis_b200 import ops
    x = rnd(m, c, dtype=torch.float32, scale=3.0)
    g, b = rnd(c, dtype=torch.float32) * 0.1 + 1, rnd(c, dtype=torch.float32) * 0.1
    dy = rnd(m, c)
    y, st = ops.layernorm(x, g, b)
    dx = ops.layernorm_bwd(dy, x, g, st)
    xr = x.clone().requires_grad_(True)
    yr = F.layer_norm(xr, (c,), g, b, 1e-5)
    yr.backward(dy.float())
    assert rel(y, yr) < 1e-3 and rel(dx, xr.grad) < 1e-3
    # accumulate into a running fp32 gradient and emit its 16-bit copy in the same launch
    acc = torch.ones_like(dx)
    lp = torch.full((m, c), float("nan"), dtype=torch.float16, device="cuda")
    ops.layernorm_bwd(dy, x, g, st, dx=acc, accumulate=True, dx_lp=lp)
    assert rel(acc, dx + 1) < 1e-5 and rel(lp, acc) < 1e-3


# ---------------------------------------------------------------------------------------------------- pointwise
def test_softmax_geglu_act_upsample(dev):
    from celebbasis_b200 import ops
    from celebbasis_b200.lib import CB_ACT_QUICK_GELU, CB_ACT_SILU
    s = rnd(300, 80, scale=3.0)
    p = ops.softmax_(s.clone(), 300, 77, 80)
    ref = torch.softmax(s[:, :77].float(), -1)
    assert rel(p[:, :77], ref) < 2e-3 and float(p[:, 77:].abs().max()) == 0
    pc = ops.softmax_(s[:231].clone(), 231, 77, 80, causal_period=77)
    mask = torch.full((77, 77), float("-inf"), device=s.device).triu_(1)
    refc = torch.softmax(s[:231, :77].float().view(3, 77, 77) + mask, -1).view(231, 77)
    assert rel(pc[:, :77], refc) < 2e-3
    dp = rnd(300, 80)
    ds = ops.softmax_bwd_(dp.clone(), p, 300, 77, 80)
    pf = p[:, :77].float()
    assert rel(ds[:, :77], pf * (dp[:, :77].float() - (dp[:, :77].float() * pf).sum(-1, keepdim=True))) < 3e-3
    x = rnd(256, 2560)
    xr = x.float().requires_grad_(True)
    a, gate = xr.chunk(2, -1)
    yr = a * F.gelu(gate)
    dy = rnd(256, 1280)
    yr.backward(dy.float())
    assert rel(ops.geglu(x), yr) < 1e-3 and rel(ops.geglu_bwd(dy, x), xr.grad) < 2e-3
    for act, fn in ((CB_ACT_SILU, F.silu), (CB_ACT_QUICK_GELU, lambda t: t * torch.sigmoid(1.702 * t))):
        v = rnd(77, 3072)
        vr = v.float().requires_grad_(True)
        o = fn(vr)
        dv = rnd(77, 3072)
        o.backward(dv.float())
        assert rel(ops.act_fwd(v, act), o) < 1e-3 and rel(ops.act_bwd(dv, v, act), vr.grad) < 2e-3
    u = rnd(2 * 8 * 8, 64)
    up, g2 = ops.upsample2x(u, ops.Geo(2, 8, 8))
    refu = F.interpolate(u.float().view(2, 8, 8, 64).permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    assert torch.equal(up.float(), refu.permute(0, 2, 3, 1).reshape(-1, 64))
    du = rnd(2 * 16 * 16, 64)
    dref = F.avg_pool2d(du.float().view(2, 16, 16, 64).permute(0, 3, 1, 2), 2) * 4
    assert rel(ops.upsample2x_bwd(du, ops.Geo(2, 8, 8), dx_dtype=torch.float32), dref.permute(0, 2, 3, 1).reshape(-1, 64)) < 1e-3


def test_layout_loss_schedule_kernels(dev):
    from celebbasis_b200 import ops
    from oracle import torch_ref
    x = rnd(2, 4, 8, 8, dtype=torch.float32)
    y, geo = ops.nchw_to_nhwc(x, 8, torch.float32)
    assert torch.equal(y.view(2, 64, 8)[:, :, :4], x.permute(0, 2, 3, 1).reshape(2, 64, 4)) and float(y[:, 4:].abs().max()) == 0
    assert torch.equal(ops.nhwc_to_nchw(y, geo, 4), x)
    pred, tgt = rnd(3, 4, 16, 16, dtype=torch.float32), rnd(3, 4, 16, 16, dtype=torch.float32)
    loss, grad = ops.mse_fwd_bwd(pred, tgt)
    pr = pred.clone().requires_grad_(True)
    lr = ((pr - tgt) ** 2).mean(dim=[1, 2, 3])
    lr.mean().backward()
    assert rel(loss, lr) < 1e-5 and rel(grad, pr.grad) < 1e-5
    t = torch.tensor([0, 1, 500, 999], device=x.device)
    assert rel(ops.timestep_embedding(t, 320, dtype=torch.float32), torch_ref.timestep_embedding(t, 320)) < 1e-5
    sched = torch_ref.make_schedule()
    z, nz = rnd(4, 4, 8, 8, dtype=torch.float32), rnd(4, 4, 8, 8, dtype=torch.float32)
    qs = ops.q_sample(z, nz, t, sched["sqrt_alphas_cumprod"].cuda(), sched["sqrt_one_minus_alphas_cumprod"].cuda())
    assert rel(qs, torch_ref.q_sample(sched, z, t, nz)) < 1e-6
    mom = rnd(2, 8, 4, 4, dtype=torch.float32, scale=3.0)
    eps = rnd(2, 4, 4, 4, dtype=torch.float32)
    assert rel(ops.posterior_sample(mom, eps, 0.18215), torch_ref.posterior_sample(mom, eps, 0.18215)) < 1e-6


def test_celeb_embedding_path_and_adamw(dev):
    """fp32 side kernels: MLP + L2 norm + basis contraction + inject, forward and gradient, vs the oracle functions."""
    from celebbasis_b200 import ops, synth
    from celebbasis_b200.train_step import build_inject_map
    from oracle import torch_ref
    Fn, es, K, D = 2, 2, 512, 768
    v = F.normalize(rnd(Fn, 512, dtype=torch.float32), dim=-1)
    W = rnd(es * K, 512, dtype=torch.float32).requires_grad_(True)
    b = (rnd(es * K, dtype=torch.float32) * 0.1).requires_grad_(True)
    basis = synth.synth_celeb_basis(seed=3).cuda()
    pre, coef, nrm = ops.celeb_mlp_fwd(v, W.detach(), b.detach(), es)
    z = ops.celeb_basis_fwd(coef, basis)
    coef_r = torch_ref.celeb_mlp(v, W, b, es)
    z_r = torch_ref.celeb_basis(coef_r, basis)
    assert rel(coef, coef_r.view(Fn, es, K)) < 1e-5 and rel(z, z_r) < 1e-5
    ids = torch.full((1, 77), 49407, dtype=torch.long)
    ids[0, :6] = torch.tensor([49406, 320, 48136, 539, 48136, 7])
    tok = rnd(1 * 77, D, dtype=torch.float32)
    pos = rnd(77, D, dtype=torch.float32)
    m, positions = build_inject_map(ids.numpy(), 48136, es, lambda i: i)
    mdev = torch.from_numpy(m).cuda()
    out = ops.embed_inject_fwd(tok, z.view(-1, D), mdev.view(-1), pos, 1, 77)
    ref_rows, ref_pos = torch_ref.inject_embeddings(ids, tok.view(1, 77, D), z_r[:1], 48136, es)
    assert [p.tolist() for p in positions[0]] == [p.tolist() for p in ref_pos[0]]
    assert rel(out, (ref_rows[0] + pos)) < 1e-6
    dout = rnd(77, D, dtype=torch.float32)
    (ref_rows[0] * dout).sum().backward()
    dz = ops.embed_inject_bwd(dout, mdev.view(-1), Fn * es, 1, 77)
    dcoef = ops.celeb_basis_bwd(dz.view(Fn, es, D), basis)
    dW, db = torch.empty_like(W), torch.empty_like(b)
    ops.celeb_mlp_bwd(dcoef, coef, nrm, pre, v, dW, db)
    assert rel(dW, W.grad) < 1e-4 and rel(db, b.grad) < 1e-4
    # AdamW == torch.optim.AdamW for 3 steps
    p0 = rnd(1000, dtype=torch.float32)
    pt = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pt], lr=5e-3)
    pm, mm, vv = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    step_dev = torch.zeros(1, dtype=torch.int32, device="cuda")
    for i in range(3):
        g = rnd(1000, dtype=torch.float32)
        pt.grad = g.clone()
        opt.step()
        ops.adamw_step(pm, g, mm, vv, lr=5e-3, step_dev=step_dev)
    assert rel(pm, pt.detach()) < 1e-6 and int(step_dev.item()) == 3


def test_face_warp_resize(dev):
    from celebbasis_b200 import ops
    from celebbasis_b200.train_step import TRANS_MATRIX
    from oracle import torch_ref
    faces = torch.rand(2, 96, 96, 6, generator=torch.Generator().manual_seed(5)).cuda() * 2 - 1
    out, geo = ops.face_warp_resize(faces, 2, TRANS_MATRIX, out_hw=112, cpad=8, dtype=torch.float32)
    ref = torch_ref.face_preprocess(torch.cat(faces.chunk(2, -1), 0))
    got = out.view(4, 112, 112, 8)
    assert rel(got[..., :3], ref.permute(0, 2, 3, 1)) < 1e-4 and float(got[..., 3:].abs().max()) == 0


@pytest.mark.parametrize("nq,nk,dh,heads,images,causal", [(4096, 4096, 40, 8, 1, False), (1024, 1024, 80, 8, 1, False),
                                                          (1024, 77, 80, 8, 2, False), (77, 77, 64, 12, 2, True),
                                                          (300, 200, 128, 2, 1, False), (64, 64, 40, 8, 1, False),
                                                          (200, 330, 40, 2, 2, True)])
def test_flash_attention_bwd(dev, nq, nk, dh, heads, images, causal):
    """cb_attention_bwd (P, dP, dS rebuilt tile by tile in registers from the forward's log-sum-exp; dQ then dK/dV, no
    atomics) vs torch.autograd of softmax(QK^T*scale)V in fp32 on the same fp16 inputs."""
    from celebbasis_b200 import ops
    C = heads * dh
    scale = dh ** -0.5
    # q/k/v and the gradients live in wider fused buffers (as the engines keep them): exercises the row pitches
    qkv = rnd(images * max(nq, nk), 3 * C + 8)
    q, k, v = qkv[:images * nq, :C], qkv[:images * nk, C:2 * C], qkv[:images * nk, 2 * C:3 * C]
    dO = rnd(images * nq, C)
    o = torch.empty(images * nq, C, dtype=torch.float16, device="cuda")
    _, lse = ops.attention_fwd(q, k, v, o, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale, causal=causal,
                               want_lse=True)
    dqkv = torch.full((images * max(nq, nk), 3 * C), float("nan"), dtype=torch.float16, device="cuda")
    dq, dk, dv = dqkv[:images * nq, :C], dqkv[:images * nk, C:2 * C], dqkv[:images * nk, 2 * C:]
    ops.attention_bwd(q, k, v, o, dO, lse, dq, dk, dv, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale,
                      causal=causal)
    sp = lambda t, n: t.float().reshape(images, n, heads, dh).permute(0, 2, 1, 3)
    qf, kf, vf = (sp(q, nq).requires_grad_(), sp(k, nk).requires_grad_(), sp(v, nk).requires_grad_())
    sc = qf @ kf.transpose(-1, -2) * scale
    if causal:
        sc = sc + torch.full((nq, nk), float("-inf"), device="cuda").triu_(1)
    ref_o = torch.softmax(sc, -1) @ vf
    ref_o.backward(sp(dO, nq))
    back = lambda t, n: t.permute(0, 2, 1, 3).reshape(images * n, C)
    for name, got, ref in (("dq", dq, back(qf.grad, nq)), ("dk", dk, back(kf.grad, nk)), ("dv", dv, back(vf.grad, nk))):
        assert torch.isfinite(got.float()).all(), name
        assert rel(got, ref) < 6e-3, (name, rel(got, ref))
    # query-stationary half alone, exporting dS = P o (dP - delta) * scale (the cross-attention backward's GEMM operand)
    ldds = (nk + 7) // 8 * 8
    dS = torch.full((images * heads * nq, ldds), float("nan"), dtype=torch.float16, device="cuda")
    dq2 = torch.empty(images * nq, C, dtype=torch.float16, device="cuda")
    ops.attention_bwd_dq(q, k, v, o, dO, lse, dq2, dS, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=scale,
                         causal=causal)
    att = torch.softmax(sc.detach(), -1)
    dP = sp(dO, nq) @ sp(v, nk).transpose(-1, -2)
    dS_ref = att * (dP - (dP * att).sum(-1, keepdim=True)) * scale
    assert rel(dq2, back(qf.grad, nq)) < 6e-3
    assert rel(dS.view(images, heads, nq, ldds)[..., :nk], dS_ref) < 8e-3
    assert float(dS.view(images, heads, nq, ldds)[..., nk:].abs().max() if ldds > nk else 0) == 0


@pytest.mark.parametrize("nq,nk,dh,heads,images,causal", [(4096, 4096, 40, 8, 1, False), (1024, 1024, 80, 8, 1, False),
                                                          (1024, 77, 80, 8, 2, False), (4096, 77, 40, 8, 1, False),
                                                          (77, 77, 64, 12, 2, True), (300, 200, 128, 2, 1, False),
                                                          (64, 64, 40, 8, 1, False)])
@pytest.mark.parametrize("want_p", [False, True])
def test_flash_attention_fwd(dev, nq, nk, dh, heads, images, causal, want_p):
    """cb_attention_fwd (scores in registers, online softmax, P.V in registers) vs softmax(QK^T*scale)V in fp32; one-pass
    (inference) and two-pass (probabilities exported for the backward) modes."""
    from celebbasis_b200 import ops
    C = heads * dh
    q, k, v = rnd(images * nq, C), rnd(images * nk, C), rnd(images * nk, C)
    o = torch.full((images * nq, C), float("nan"), dtype=torch.float16, device="cuda")
    P, lse = ops.attention_fwd(q, k, v, o, images=images, heads=heads, dh=dh, nq=nq, nk=nk, scale=dh ** -0.5,
                               causal=causal, want_p=want_p, want_lse=True)
    sp = lambda t, n: t.float().view(images, n, heads, dh).permute(0, 2, 1, 3)
    s = sp(q, nq) @ sp(k, nk).transpose(-1, -2) * dh ** -0.5
    if causal:
        s = s + torch.full((nq, nk), float("-inf"), device="cuda").triu_(1)
    att = torch.softmax(s, -1)
    ref = (att @ sp(v, nk)).permute(0, 2, 1, 3).reshape(images * nq, C)
    assert torch.isfinite(o.float()).all()
    assert rel(o, ref) < 3e-3
    assert rel(lse, torch.logsumexp(s, -1).reshape(-1)) < 1e-4
    if want_p:
        ldp = (nk + 7) // 8 * 8
        pr = P.view(images, heads, nq, ldp)
        assert rel(pr[..., :nk], att) < 3e-3 and float(pr[..., nk:].abs().max() if ldp > nk else 0) == 0


# ---------------------------------------------------------------------------------------------------- round-2 additions
@pytest.mark.parametrize("splits", [0, 4])
def test_gemm_second_destination_and_strided_out(dev, splits):
    """cb_gemm D2: the epilogue value is also stored at a second address with its own dtype / row pitch (the UNet's
    skip-connection concat without copies) -- fast path, ragged-N slow path and the split-K last-CTA path."""
    from celebbasis_b200 import ops
    from celebbasis_b200.lib import GemmDesc
    for (M, N, K) in ((256, 320, 640), (200, 72, 128)):
        x, w = rnd(M, K), rnd(N, K)
        bias = rnd(N, dtype=torch.float32)
        res = rnd(M, N, dtype=torch.float32)
        cat = torch.full((M, N + 96), -7.0, dtype=torch.float32, device="cuda")
        cat16 = torch.full((M, 2 * N), -7.0, dtype=torch.float16, device="cuda")
        ref = x.float() @ w.float().t() + bias + res
        if splits:
            # force split-K through the descriptor override
            orig = ops._gemm

            def forced(d, what):
                d.splits = splits
                return orig(d, what)
            ops._gemm = forced
        try:
            y = ops.linear(x, w, bias, out=cat[:, 96:], residual=res, out2=cat16[:, N:])
        finally:
            if splits:
                ops._gemm = orig
        assert rel(cat[:, 96:], ref) < 2e-3 and rel(cat16[:, N:], ref) < 2e-3
        assert float((cat[:, :96] + 7).abs().max()) == 0 and float((cat16[:, :N] + 7).abs().max()) == 0
    # conv with a second destination
    g = ops.Geo(2, 16, 16)
    xi = rnd(g.rows, 64)
    wc = torch.randn(128, 64, 3, 3, device="cuda") * 0.05
    pack = ops.pack_conv_weight(wc, torch.float16)
    d2 = torch.zeros(g.rows, 128 + 32, dtype=torch.float32, device="cuda")
    y, _ = ops.conv2d(xi, g, pack, 128, out_dtype=torch.float16, out2=d2[:, 32:])
    refc = F.conv2d(xi.float().view(2, 16, 16, 64).permute(0, 3, 1, 2), wc.half().float(), padding=1)
    refc = refc.permute(0, 2, 3, 1).reshape(g.rows, 128)
    assert rel(y, refc) < 2e-3 and rel(d2[:, 32:], refc) < 2e-3 and float(d2[:, :32].abs().max()) == 0


def test_gemm_tile256(dev):
    """128x256 output tiles (tile_n = 256, 4-stage ring): K-major and MN-major B, conv and ragged N."""
    from celebbasis_b200 import ops
    orig = ops._gemm

    def forced(d, what):
        d.tile_n = 256
        return orig(d, what)
    ops._gemm = forced
    try:
        x, w = rnd(1024, 640), rnd(1280, 640)
        y = ops.linear(x, w, out_dtype=torch.float32)
        assert rel(y, x.float() @ w.float().t()) < 2e-3
        dy = rnd(1024, 1280)
        dx = ops.linear_dgrad(dy, w, out_dtype=torch.float32)          # B read MN-major
        assert rel(dx, dy.float() @ w.float()) < 2e-3
        x2, w2 = rnd(512, 320), rnd(600, 320)                          # N = 600: 256 + 256 + 88
        y2 = ops.linear(x2, w2, out_dtype=torch.float32)
        assert rel(y2, x2.float() @ w2.float().t()) < 2e-3
        g = ops.Geo(1, 32, 32)
        xi = rnd(g.rows, 320)
        wc = torch.randn(512, 320, 3, 3, device="cuda") * 0.02
        yc, _ = ops.conv2d(xi, g, ops.pack_conv_weight(wc, torch.float16), 512, out_dtype=torch.float32)
        refc = F.conv2d(xi.float().view(1, 32, 32, 320).permute(0, 3, 1, 2), wc.half().float(), padding=1)
        assert rel(yc, refc.permute(0, 2, 3, 1).reshape(g.rows, 512)) < 2e-3
    finally:
        ops._gemm = orig


def test_groupnorm_bwd_emits_16bit_copy(dev):
    from celebbasis_b200 import ops
    # fp32 x, fp16 dy: the backward runs on the cluster kernel / on the statistics + apply pair
    for (hw, c) in ((32, 640), (256, 128)):
        geo = ops.Geo(1, hw, hw)
        x = rnd(geo.rows, c, dtype=torch.float32, scale=2.0)
        gm, bt = rnd(c, dtype=torch.float32) * 0.1 + 1, rnd(c, dtype=torch.float32) * 0.1
        dy = rnd(geo.rows, c)
        _, st = ops.groupnorm(x, geo, gm, bt, silu=True)
        dx = ops.groupnorm_bwd(dy, x, geo, gm, bt, st, silu=True)
        lp = torch.full((geo.rows, c), float("nan"), dtype=torch.float16, device="cuda")
        dx2 = ops.groupnorm_bwd(dy, x, geo, gm, bt, st, silu=True, dx_lp=lp)
        assert rel(dx2, dx) < 1e-5 and rel(lp, dx) < 1e-3


def test_ema_rows_and_prep_kernels(dev):
    from celebbasis_b200 import ops
    table = rnd(10, 2 * 768, dtype=torch.float32)
    t0 = table.clone()
    src = rnd(3, 2 * 768, dtype=torch.float32)
    idx = torch.tensor([[4, 4], [7, 7], [4, 4]], device="cuda")        # identity 4 appears twice: batch order matters
    ops.ema_rows(table, idx, src, 0.99)
    exp = t0.clone()
    for b, i in enumerate([4, 7, 4]):
        exp[i] = 0.99 * exp[i] + 0.01 * src[b]
    assert torch.allclose(table, exp, atol=1e-6)
    idx_bad = torch.tensor([[11, 0]], device="cuda")                    # out of range: skipped, like the reference's `if`
    ops.ema_rows(table, idx_bad, src[:1].contiguous(), 0.5)
    assert torch.allclose(table, exp, atol=1e-6)
    w = torch.randn(24, 10, 3, 3)
    sc = torch.rand(24) + 0.5
    pk = ops.pack_conv_weight(w, torch.float16, cin_pad=16, cout_pad=32, out_scale=sc, device="cuda")
    ref = torch.zeros(9, 32, 16)
    ref[:, :24, :10] = (w * sc.view(-1, 1, 1, 1)).permute(2, 3, 0, 1).reshape(9, 24, 10)
    assert rel(pk.float().cpu(), ref.view(9 * 32, 16)) < 1e-3
    assert rel(ops.to_device(torch.arange(7.0), "cuda", torch.float16).cpu(), torch.arange(7.0)) == 0


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_cta_pair(dev, bn):
    """desc.cta_pair = 1 requests (single-CTA 128 x bn tiles on sm_90).  Linear K-major / MN-major B,
    3x3 convolution (padding, ragged rows), odd tile counts, bias + residual + second destination."""
    from celebbasis_b200 import ops
    orig = ops._gemm

    def forced(d, what):
        d.cta_pair, d.tile_n = 1, bn
        return orig(d, what)
    ops._gemm = forced
    try:
        x, w = rnd(4096, 320), rnd(640, 320)
        bias, res = rnd(640, dtype=torch.float32), rnd(4096, 640, dtype=torch.float32)
        y = ops.linear(x, w, bias, out_dtype=torch.float32, residual=res)
        assert rel(y, x.float() @ w.float().t() + bias + res) < 2e-3
        dy = rnd(4096, 640)
        dx = ops.linear_dgrad(dy, w, out_dtype=torch.float32)                  # MN-major B
        assert rel(dx, dy.float() @ w.float()) < 2e-3
        x3, w3 = rnd(128 * 5 + 40, 192), rnd(300, 192)                          # odd number of m tiles, ragged M and N
        y3 = ops.linear(x3, w3, out_dtype=torch.float16)
        assert rel(y3, x3.float() @ w3.float().t()) < 2e-3
        g = ops.Geo(2, 48, 48)                                                  # 4608 rows: 36 tiles; 48-wide rows: ragged boxes
        xi = rnd(g.rows, 128)
        wc = torch.randn(256, 128, 3, 3, device="cuda") * 0.03
        d2 = torch.zeros(g.rows, 256 + 64, dtype=torch.float32, device="cuda")
        yc, _ = ops.conv2d(xi, g, ops.pack_conv_weight(wc, torch.float16), 256, out_dtype=torch.float32, out2=d2[:, 64:])
        refc = F.conv2d(xi.float().view(2, 48, 48, 128).permute(0, 3, 1, 2), wc.half().float(), padding=1)
        refc = refc.permute(0, 2, 3, 1).reshape(g.rows, 256)
        assert rel(yc, refc) < 2e-3 and rel(d2[:, 64:], refc) < 2e-3
        dyc = rnd(g.rows, 256)
        dxc, _ = ops.conv2d_dgrad(dyc, g, ops.pack_conv_weight(wc, torch.float16), 128, out_dtype=torch.float32)
        xr = xi.float().view(2, 48, 48, 128).permute(0, 3, 1, 2).requires_grad_(True)
        F.conv2d(xr, wc.half().float(), padding=1).backward(dyc.float().view(2, 48, 48, 256).permute(0, 3, 1, 2))
        assert rel(dxc, xr.grad.permute(0, 2, 3, 1).reshape(g.rows, 128)) < 2e-3
    finally:
        ops._gemm = orig


@pytest.mark.parametrize("splits,cap", [(2, 1), (5, 1), (12, 1), (3, 16)])
def test_gemm_cta_pair_splitk(dev, splits, cap):
    """Split-K with pair tile requests (desc.cta_pair >= 1, desc.splits > 1): the k-slices of a 128 x 256 tile meet in the
    L2 workspace.  Small-M / deep-K shapes of the 16^2 / 32^2 UNet levels, ragged M / N, odd tile counts,
    bias + residual, MN-major B, repeated launches (the workspace must come back zeroed)."""
    from celebbasis_b200 import ops
    orig = ops._gemm

    def forced(d, what):
        d.cta_pair, d.tile_n, d.splits = cap, 256, splits
        return orig(d, what)
    ops._gemm = forced
    try:
        x, w = rnd(256, 5120), rnd(1280, 5120) * 0.05
        bias, res = rnd(1280, dtype=torch.float32), rnd(256, 1280, dtype=torch.float32)
        ref = x.float() @ w.float().t() + bias + res
        for _ in range(3):
            y = ops.linear(x, w, bias, out_dtype=torch.float32, residual=res)
            assert rel(y, ref) < 2e-3
        dy = rnd(256, 1280)
        dx = ops.linear_dgrad(dy, w, out_dtype=torch.float16)                   # MN-major B, K = 1280 -> 20 k-iterations
        assert rel(dx, dy.float() @ w.float()) < 2e-3
        x3, w3 = rnd(128 * 2 + 44, 1024), rnd(1000, 1024) * 0.05                # 3 m tiles (odd), ragged M and N
        y3 = ops.linear(x3, w3, out_dtype=torch.float16)
        assert rel(y3, x3.float() @ w3.float().t()) < 2e-3
        g = ops.Geo(1, 16, 16)                                                  # the 16^2 level: M = 256, K = 9 * 640
        xi = rnd(g.rows, 640)
        wc = torch.randn(1280, 640, 3, 3, device="cuda") * 0.02
        pk = ops.pack_conv_weight(wc, torch.float16)
        bi = rnd(1280, dtype=torch.float32)
        refc = F.conv2d(xi.float().view(1, 16, 16, 640).permute(0, 3, 1, 2), wc.half().float(), bias=bi, padding=1)
        refc = refc.permute(0, 2, 3, 1).reshape(g.rows, 1280)
        for _ in range(2):
            yc, _ = ops.conv2d(xi, g, pk, 1280, bias=bi, out_dtype=torch.float32)
            assert rel(yc, refc) < 2e-3
        dyc = rnd(g.rows, 1280)
        dxc, _ = ops.conv2d_dgrad(dyc, g, pk, 640, out_dtype=torch.float32)
        xr = xi.float().view(1, 16, 16, 640).permute(0, 3, 1, 2).requires_grad_(True)
        F.conv2d(xr, wc.half().float(), padding=1).backward(dyc.float().view(1, 16, 16, 1280).permute(0, 3, 1, 2))
        assert rel(dxc, xr.grad.permute(0, 2, 3, 1).reshape(g.rows, 640)) < 2e-3
    finally:
        ops._gemm = orig
    # the single-CTA split-K kernel shares the workspace: it must still see zeros
    x, w = rnd(256, 2560), rnd(640, 2560) * 0.05
    assert rel(ops.linear(x, w, out_dtype=torch.float32), x.float() @ w.float().t()) < 2e-3


@pytest.mark.parametrize("bn,splits", [(64, 2), (64, 6), (64, 16), (128, 5), (128, 8), (128, 12), (160, 8)])
def test_gemm_cluster_splitk(dev, bn, splits):
    """desc.splitk_cluster = 1: the k-slices of a tile are a thread-block cluster (1,1,splits) that exchanges 8-column
    groups of the partial accumulators through distributed shared memory (no global workspace, no atomics).  Plain /
    bias + residual / activation epilogues, fp16 and fp32 outputs, ragged M and N, MN-major operands, batched launches,
    3x3 convolution and its dgrad; non-power-of-two and non-portable (16) cluster sizes."""
    from celebbasis_b200 import ops
    from celebbasis_b200.lib import CB_ACT_SILU
    orig = ops._gemm
    seen = []

    def forced(d, what):
        d.tile_n, d.splits, d.splitk_cluster = bn, splits, 1
        seen.append(d.N)
        return orig(d, what)
    ops._gemm = forced
    try:
        x, w = rnd(77, 3072), rnd(768, 3072) * 0.05
        bias, res = rnd(768, dtype=torch.float32), rnd(77, 768, dtype=torch.float32)
        ref = x.float() @ w.float().t()
        for _ in range(2):
            assert rel(ops.linear(x, w, bias, out_dtype=torch.float32, residual=res), ref + bias + res) < 2e-3
        assert rel(ops.linear(x, w, bias, act=CB_ACT_SILU), F.silu(ref + bias)) < 2e-3
        dy = rnd(300, 1000)                                                     # ragged M (3 m tiles) and N
        w2 = rnd(1000, 1536) * 0.05
        assert rel(ops.linear_dgrad(dy, w2, out_dtype=torch.float32), dy.float() @ w2.float()) < 2e-3     # MN-major B
        x3 = rnd(300, 1536)
        assert rel(ops.linear(x3, w2, out_dtype=torch.float16), x3.float() @ w2.float().t()) < 2e-3
        g = ops.Geo(1, 16, 16)
        xi = rnd(g.rows, 640)
        wc = torch.randn(1280, 640, 3, 3, device="cuda") * 0.02
        pk = ops.pack_conv_weight(wc, torch.float16)
        bi = rnd(1280, dtype=torch.float32)
        refc = F.conv2d(xi.float().view(1, 16, 16, 640).permute(0, 3, 1, 2), wc.half().float(), bias=bi, padding=1)
        refc = refc.permute(0, 2, 3, 1).reshape(g.rows, 1280)
        yc, _ = ops.conv2d(xi, g, pk, 1280, bias=bi, out_dtype=torch.float32)
        assert rel(yc, refc) < 2e-3
        dyc = rnd(g.rows, 1280)
        dxc, _ = ops.conv2d_dgrad(dyc, g, pk, 640, out_dtype=torch.float16)
        xr = xi.float().view(1, 16, 16, 640).permute(0, 3, 1, 2).requires_grad_(True)
        F.conv2d(xr, wc.half().float(), padding=1).backward(dyc.float().view(1, 16, 16, 1280).permute(0, 3, 1, 2))
        assert rel(dxc, xr.grad.permute(0, 2, 3, 1).reshape(g.rows, 640)) < 2e-3
        # batched, both operands MN-major (cross-attention dV = P^T dO over 1024 queries, 8 heads)
        heads, nq, nk, dh = 8, 1024, 77, 80
        P, dO = rnd(heads * nq, 80) * 0.1, rnd(nq, heads * dh)
        dv = torch.zeros(nk, heads * dh, dtype=torch.float16, device="cuda")
        ops.bmm(P, dO, dv, M=nk, N=dh, K=nq, heads=heads, images=1, lda=80, ldb=dO.stride(0), ldd=dv.stride(0),
                a_hs=nq * 80, b_hs=dh, d_hs=dh, a_is=heads * nq * 80, b_is=nq * dO.stride(0), d_is=nk * dv.stride(0),
                a_major=ops.CB_MAJOR_MN, b_major=ops.CB_MAJOR_MN)
        refv = torch.einsum("hqk,qhd->khd", P.float().view(heads, nq, 80)[:, :, :nk], dO.float().view(nq, heads, dh))
        assert rel(dv.view(nk, heads, dh), refv) < 2e-3
    finally:
        ops._gemm = orig
    assert len(seen) >= 8


def test_front_end_sm_budget(dev):
    """ops.FE_CTAS (env CB_FE_CTAS): inside the front-end lane the large GEMMs run as pair tile requests (stride-2 / asymmetric padding of the VAE downsample included) and the streaming GroupNorm pair on at
    most n CTAs; results are unchanged."""
    from celebbasis_b200 import ops
    old = ops.FE_CTAS
    ops.FE_CTAS = 24
    try:
        with ops.lane(2):
            for (n, h, cin, cout, stride, pad) in [(1, 128, 128, 128, 2, (0, 1, 0, 1)), (1, 96, 128, 256, 1, (1, 1, 1, 1)),
                                                   (1, 64, 8, 128, 1, (1, 1, 1, 1))]:
                x = rnd(n * h * h, cin)
                wt = rnd(cout, cin, 3, 3, scale=(9 * cin) ** -0.5)
                b = rnd(cout, dtype=torch.float32)
                y, _ = ops.conv2d(x, ops.Geo(n, h, h), ops.pack_conv_weight(wt, torch.float16), cout, bias=b, stride=stride,
                                  pad=pad, out_dtype=torch.float32)
                xr = F.pad(x.float().view(n, h, h, cin).permute(0, 3, 1, 2), (pad[2], pad[3], pad[0], pad[1]))
                ref = F.conv2d(xr, wt.float(), b, stride=stride).permute(0, 2, 3, 1).reshape(-1, cout)
                assert y.shape == ref.shape and rel(y, ref) < 1e-3
            xl, wl = rnd(4096, 512), rnd(512, 512) * 0.05
            res = rnd(4096, 512, dtype=torch.float32)
            assert rel(ops.linear(xl, wl, out_dtype=torch.float32, residual=res), xl.float() @ wl.float().t() + res) < 1e-3
            hw, c = 65536, 128
            xg = rnd(hw, c, dtype=torch.float32, scale=2.0) + 0.5
            g, b = rnd(c, dtype=torch.float32) * 0.1 + 1, rnd(c, dtype=torch.float32) * 0.1
            y, _ = ops.groupnorm(xg, ops.Geo(1, 256, 256), g, b, eps=1e-6, silu=True)
            yr = F.silu(F.group_norm(xg.view(1, hw, c).permute(0, 2, 1), 32, g, b, 1e-6)).permute(0, 2, 1).reshape(hw, c)
            assert rel(y, yr) < 1e-3
    finally:
        ops.FE_CTAS = old


def test_gemm_prelu_epilogue_and_d2_affine(dev):
    """CB_ACT_PRELU (per-column slopes) and the per-column affine of the second destination: an IBasicBlock's PReLU and
    the next block's bn1 inside the conv epilogues (iresnet.py:41-58)."""
    from celebbasis_b200 import ops
    from celebbasis_b200.lib import CB_ACT_PRELU
    g = ops.Geo(2, 14, 14)
    xi = rnd(g.rows, 64)
    wc = torch.randn(72, 64, 3, 3, device="cuda") * 0.05                       # N = 72: fast path + ragged tail
    bias = rnd(72, dtype=torch.float32)
    slope = torch.rand(72, device="cuda") * 0.5
    sc, sh = torch.rand(72, device="cuda") + 0.5, rnd(72, dtype=torch.float32)
    res = rnd(g.rows, 72, dtype=torch.float32)
    d2 = torch.empty(g.rows, 72, dtype=torch.float16, device="cuda")
    y, _ = ops.conv2d(xi, g, ops.pack_conv_weight(wc, torch.float16), 72, bias=bias, out_dtype=torch.float32, act=CB_ACT_PRELU,
                      act_param=slope, residual=res, out2=d2, out2_affine=(sc, sh))
    ref = F.conv2d(xi.float().view(2, 14, 14, 64).permute(0, 3, 1, 2), wc.half().float(), padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(g.rows, 72) + bias
    ref = torch.where(ref > 0, ref, ref * slope) + res
    assert rel(y, ref) < 2e-3 and rel(d2, ref * sc + sh) < 2e-3


def test_iresnet_fused_epilogues_equal_unfused(dev):
    from celebbasis_b200 import synth
    from celebbasis_b200.iresnet_engine import IResNetEngine
    from oracle import torch_ref
    net = torch_ref.IResNet().eval()
    pre = "embedding_manager.meta_id_net.id_model."
    sd = synth.synth_state_dict(net, seed=0, prefix=pre)
    net.load_state_dict(sd)
    eng = IResNetEngine({pre + k: v for k, v in sd.items()}, "cuda", prefix=pre)
    x = rnd(2 * 112 * 112, 8)
    x[:, 3:] = 0
    from celebbasis_b200 import ops
    geo = ops.Geo(2, 112, 112)
    a = eng.forward(x, geo)
    eng.FUSE_EPILOGUES = False
    b = eng.forward(x, geo)
    assert rel(a, b) < 5e-3, rel(a, b)
    with torch.no_grad():
        ref = net.cuda()(x[:, :3].float().view(2, 112, 112, 3).permute(0, 3, 1, 2).contiguous())
    assert rel(a, ref) < 5e-3, rel(a, ref)


@pytest.mark.parametrize("M,C", [(4096, 320), (256, 1280), (70, 64)])
def test_linear_geglu_epilogue(dev, M, C):
    """GEGLU (attention.py:37-45: x, gate = proj(x).chunk(2); x * gelu(gate)) inside the FF-in GEMM's epilogue on the
    interleaved weight layout; the kept pre-activations feed cb_geglu_bwd(interleave=1)."""
    from celebbasis_b200 import ops
    x = rnd(M, C)
    w = rnd(8 * C, C, scale=C ** -0.5)
    b = rnd(8 * C, dtype=torch.float32) * 0.1
    w_il = ops.glu_interleave_rows(w).contiguous()
    b_il = ops.glu_interleave_rows(b).contiguous()
    u, g = ops.linear_geglu(x, w_il, b_il, keep_preact=True)
    pre = x.float() @ w.float().t() + b
    a_ref, g_ref = pre.chunk(2, -1)
    u_ref = a_ref * F.gelu(g_ref)
    assert rel(u, u_ref) < 3e-3, rel(u, u_ref)
    assert rel(g, ops.glu_interleave_rows(pre.t()).t()) < 2e-3
    u2, g2 = ops.linear_geglu(x, w_il, b_il, keep_preact=False)        # inference: no pre-activation store
    assert g2 is None and rel(u2, u_ref) < 3e-3
    assert rel(ops.geglu(g, interleaved=True), u_ref) < 3e-3
    du = rnd(M, 4 * C)
    dg = ops.geglu_bwd(du, g, interleaved=True)
    pr = pre.clone().requires_grad_(True)
    a2, g2r = pr.chunk(2, -1)
    (a2 * F.gelu(g2r)).backward(du.float())
    assert rel(dg, ops.glu_interleave_rows(pr.grad.t()).t()) < 5e-3
