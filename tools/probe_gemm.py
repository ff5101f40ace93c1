"""GPU probe for cb_gemm: correctness of every operand-major / conv mode + a few timings.

Run on the GPU box:  python tools/probe_gemm.py [group ...]
Each group runs in its own subprocess so a device trap in one group does not mask the others.
Results: tools_out/gemm_probe.jsonl
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tools_out")
os.makedirs(OUT, exist_ok=True)

GROUPS = ["basic", "mn", "conv", "conv_s2", "dgrad", "timing"]


def emit(rec):
    with open(os.path.join(OUT, "gemm_probe.jsonl"), "a") as f:
        f.write(json.dumps(rec) + "\n")
    print(json.dumps(rec), flush=True)


def run_group(group):
    import torch
    import torch.nn.functional as F
    from celebbasis_b200 import raw
    from celebbasis_b200.lib import (CB_ACT_GELU, CB_ACT_NONE, CB_ACT_QUICK_GELU, CB_ACT_SILU, CB_MAJOR_K,
                                     CB_MAJOR_MN)

    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(1234)

    def rnd(*shape, dtype=torch.float16, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(dtype).to(dev)

    def report(name, got, ref, **extra):
        torch.cuda.synchronize()
        got = got.float()
        ref = ref.float()
        err = (got - ref).abs().max().item()
        den = ref.abs().max().item() + 1e-12
        rel_fro = ((got - ref).norm() / (ref.norm() + 1e-12)).item()
        emit(dict(group=group, case=name, max_abs_err=err, ref_max=den, rel_fro=rel_fro,
                  ok=bool(rel_fro < 2e-3 and err / den < 1e-2), **extra))

    def guarded(name, fn):
        try:
            fn()
        except Exception as e:  # noqa
            emit(dict(group=group, case=name, ok=False, error=repr(e)[:400]))

    if group == "basic":
        def plain(M, N, K, dtype=torch.float16, out_dtype=torch.float16, bias=False, act=CB_ACT_NONE, res=None,
                  alpha=1.0, transposed=False, name=None):
            A = rnd(M, K, dtype=dtype)
            B = rnd(N, K, dtype=dtype, scale=K ** -0.5)
            bvec = rnd(N, dtype=torch.float32) if bias else None
            R = rnd(M, N, dtype=res) if res is not None else None
            D = torch.full((N, M) if transposed else (M, N), float("nan"), dtype=out_dtype, device=dev)
            raw.gemm(A, B, D, M=M, N=N, K=K, lda=K, ldb=K, ldd=(M if transposed else N), bias=bvec, ldbias=N,
                     R=R, ldr=N, alpha=alpha, act=act, d_transposed=transposed)
            ref = alpha * (A.float() @ B.float().t())
            if bias:
                ref = ref + bvec
            if act == CB_ACT_SILU:
                ref = F.silu(ref)
            elif act == CB_ACT_GELU:
                ref = F.gelu(ref)
            elif act == CB_ACT_QUICK_GELU:
                ref = ref * torch.sigmoid(1.702 * ref)
            if R is not None:
                ref = ref + R.float()
            if transposed:
                ref = ref.t()
            report(name or f"plain_{M}x{N}x{K}", D, ref, dtype=str(dtype), out=str(out_dtype))

        guarded("p1", lambda: plain(128, 160, 64, name="p1_128x160x64"))
        guarded("p2", lambda: plain(256, 320, 320))
        guarded("p3", lambda: plain(4096, 320, 320))
        guarded("p4", lambda: plain(4096, 2560, 320, out_dtype=torch.float32, bias=True))
        guarded("p5", lambda: plain(77, 768, 768, bias=True, act=CB_ACT_QUICK_GELU, name="clip_77x768x768"))
        guarded("p6", lambda: plain(300, 64, 40, name="ktail_300x64x40"))
        guarded("p7", lambda: plain(1000, 1280, 2560, dtype=torch.bfloat16, out_dtype=torch.bfloat16,
                                     name="bf16_1000x1280x2560"))
        guarded("p8", lambda: plain(512, 640, 640, bias=True, act=CB_ACT_SILU, res=torch.float32,
                                     out_dtype=torch.float32, name="epi_silu_res32"))
        guarded("p9", lambda: plain(512, 128, 640, res=torch.float16, act=CB_ACT_GELU, bias=True, alpha=0.5,
                                     name="epi_gelu_res16_alpha"))
        guarded("p10", lambda: plain(200, 96, 128, transposed=True, name="transposed_out"))
        guarded("p11", lambda: plain(64, 4, 320, out_dtype=torch.float32, bias=False, name="n4_scalar_tail"))

        def batched():
            # attention-like: Q [Nq][8*d], K [Nk][8*d]; S[h] = Q_h K_h^T * scale
            Nq, Nk, H, dh = 1024, 1024, 8, 40
            Q = rnd(Nq, H * dh)
            Kt = rnd(Nk, H * dh)
            S = torch.full((H, Nq, Nk), float("nan"), dtype=torch.float16, device=dev)
            raw.gemm(Q, Kt, S, M=Nq, N=Nk, K=dh, batch=H, lda=H * dh, ldb=H * dh, ldd=Nk, a_bs=dh, b_bs=dh,
                     d_bs=Nq * Nk, alpha=dh ** -0.5)
            qh = Q.float().view(Nq, H, dh).permute(1, 0, 2)
            kh = Kt.float().view(Nk, H, dh).permute(1, 0, 2)
            report("batched_qk_d40", S, torch.einsum("hqd,hkd->hqk", qh, kh) * dh ** -0.5)
        guarded("batched", batched)

    if group == "mn":
        def b_mn(M, N, K):
            A = rnd(M, K)
            Bm = rnd(K, N, scale=K ** -0.5)  # stored [K][N]
            D = torch.full((M, N), float("nan"), dtype=torch.float16, device=dev)
            raw.gemm(A, Bm, D, M=M, N=N, K=K, lda=K, ldb=N, ldd=N, b_major=CB_MAJOR_MN)
            report(f"b_mn_{M}x{N}x{K}", D, A.float() @ Bm.float())
        guarded("bmn1", lambda: b_mn(256, 128, 128))
        guarded("bmn2", lambda: b_mn(1024, 320, 640))
        guarded("bmn3", lambda: b_mn(300, 40, 72))

        def ab_mn(M, N, K):
            Am = rnd(K, M)
            Bm = rnd(K, N, scale=K ** -0.5)
            D = torch.full((M, N), float("nan"), dtype=torch.float32, device=dev)
            raw.gemm(Am, Bm, D, M=M, N=N, K=K, lda=M, ldb=N, ldd=N, a_major=CB_MAJOR_MN, b_major=CB_MAJOR_MN)
            report(f"ab_mn_{M}x{N}x{K}", D, Am.float().t() @ Bm.float())
        guarded("abmn1", lambda: ab_mn(256, 128, 128))
        guarded("abmn2", lambda: ab_mn(1024, 80, 1024))
        guarded("abmn3", lambda: ab_mn(72, 40, 300))

        def pv():
            # P [H][Nq][Nk] x V [Nk][H*d] -> O [Nq][H*d]  (B MN-major, batched over heads)
            Nq, Nk, H, dh = 512, 77, 8, 80
            P = torch.zeros(H, Nq, 80, dtype=torch.float16, device=dev)
            P[:, :, :Nk] = torch.softmax(rnd(H, Nq, Nk, dtype=torch.float32), -1).half()
            V = rnd(Nk, H * dh)
            O = torch.full((Nq, H * dh), float("nan"), dtype=torch.float16, device=dev)
            raw.gemm(P, V, O, M=Nq, N=dh, K=Nk, batch=H, lda=80, ldb=H * dh, ldd=H * dh, a_bs=Nq * 80, b_bs=dh,
                     d_bs=dh, b_major=CB_MAJOR_MN)
            vh = V.float().view(Nk, H, dh).permute(1, 0, 2)
            ref = torch.einsum("hqk,hkd->qhd", P[:, :, :Nk].float(), vh).reshape(Nq, H * dh)
            report("pv_cross_d80", O, ref)
        guarded("pv", pv)

    def conv_case(name, n, h, w, cin, cout, stride=1, pads=(1, 1, 1, 1), dtype=torch.float16):
        # pads = (top, bottom, left, right)
        x = rnd(n, h, w, cin, dtype=dtype)  # NHWC
        wt = rnd(cout, cin, 3, 3, dtype=dtype, scale=(9 * cin) ** -0.5)
        bias = rnd(cout, dtype=torch.float32)
        wp = wt.permute(2, 3, 0, 1).contiguous().view(9 * cout, cin)  # [tap][cout][cin]
        oh = (h + pads[0] + pads[1] - 3) // stride + 1
        ow = (w + pads[2] + pads[3] - 3) // stride + 1
        D = torch.full((n * oh * ow, cout), float("nan"), dtype=torch.float32, device=dev)
        raw.gemm(x, wp, D, M=n * oh * ow, N=cout, K=cin, lda=cin, ldb=cin, ldd=cout, bias=bias, ldbias=cout,
                 conv=dict(img_n=n, img_h=h, img_w=w, out_h=oh, out_w=ow, kh=3, kw=3, stride=stride,
                           pad_top=pads[0], pad_left=pads[2], b_tap_rows=cout, flip_taps=0))
        xr = F.pad(x.float().permute(0, 3, 1, 2), (pads[2], pads[3], pads[0], pads[1]))
        ref = F.conv2d(xr, wt.float(), bias, stride=stride)
        ref = ref.permute(0, 2, 3, 1).reshape(n * oh * ow, cout)
        report(name, D, ref)

    if group == "conv":
        guarded("c1", lambda: conv_case("conv_64x64_320_320", 1, 64, 64, 320, 320))
        guarded("c2", lambda: conv_case("conv_32x32_640_640", 1, 32, 32, 640, 640))
        guarded("c3", lambda: conv_case("conv_16x16_1280_1280", 1, 16, 16, 1280, 1280))
        guarded("c4", lambda: conv_case("conv_8x8_1280_1280", 1, 8, 8, 1280, 1280))
        guarded("c5", lambda: conv_case("conv_8x8_b2_2560_1280", 2, 8, 8, 2560, 1280))
        guarded("c6", lambda: conv_case("conv_64x64_8_320_stem", 1, 64, 64, 8, 320))
        guarded("c7", lambda: conv_case("conv_64x64_320_16_head", 1, 64, 64, 320, 16))
        guarded("c8", lambda: conv_case("conv_56x56_64_64_ragged", 2, 56, 56, 64, 64))
        guarded("c9", lambda: conv_case("conv_14x14_256_256_ragged", 2, 14, 14, 256, 256))
        guarded("c10", lambda: conv_case("conv_7x7_512_512_ragged", 3, 7, 7, 512, 512))
        guarded("c11", lambda: conv_case("conv_256x256_128_128_wide", 1, 256, 256, 128, 128))
        guarded("c12", lambda: conv_case("conv_bf16_32x32_320_640", 1, 32, 32, 320, 640, dtype=torch.bfloat16))

    if group == "conv_s2":
        guarded("s1", lambda: conv_case("conv_s2_64_320", 1, 64, 64, 320, 320, stride=2))
        guarded("s2", lambda: conv_case("conv_s2_16_1280", 1, 16, 16, 1280, 1280, stride=2))
        guarded("s3", lambda: conv_case("conv_s2_asym_vae_128", 1, 128, 128, 128, 128, stride=2, pads=(0, 1, 0, 1)))
        guarded("s4", lambda: conv_case("conv_s2_112_ragged", 2, 112, 112, 64, 64, stride=2))

    if group == "dgrad":
        def dgrad(n, h, w, cin, cout):
            # dX = conv_transpose(dY, W): use forward weight pack [tap][cout][cin] as MN-major B with flipped taps
            wt = rnd(cout, cin, 3, 3, scale=(9 * cin) ** -0.5)
            wp = wt.permute(2, 3, 0, 1).contiguous().view(9 * cout, cin)
            dy = rnd(n, h, w, cout)
            D = torch.full((n * h * w, cin), float("nan"), dtype=torch.float32, device=dev)
            raw.gemm(dy, wp, D, M=n * h * w, N=cin, K=cout, lda=cout, ldb=cin, ldd=cin, b_major=CB_MAJOR_MN,
                     conv=dict(img_n=n, img_h=h, img_w=w, out_h=h, out_w=w, kh=3, kw=3, stride=1, pad_top=1,
                               pad_left=1, b_tap_rows=cout, flip_taps=1))
            ref = F.conv_transpose2d(dy.float().permute(0, 3, 1, 2), wt.float(), padding=1)
            report(f"dgrad_{h}x{w}_{cin}_{cout}", D, ref.permute(0, 2, 3, 1).reshape(n * h * w, cin))
        guarded("d1", lambda: dgrad(1, 32, 32, 640, 640))
        guarded("d2", lambda: dgrad(1, 64, 64, 320, 320))
        guarded("d3", lambda: dgrad(1, 16, 16, 1920, 1280))

        def lin_dgrad(M, cin, cout):
            W = rnd(cout, cin, scale=cin ** -0.5)
            dy = rnd(M, cout)
            D = torch.full((M, cin), float("nan"), dtype=torch.float32, device=dev)
            raw.gemm(dy, W, D, M=M, N=cin, K=cout, lda=cout, ldb=cin, ldd=cin, b_major=CB_MAJOR_MN)
            report(f"lin_dgrad_{M}_{cin}_{cout}", D, dy.float() @ W.float())
        guarded("l1", lambda: lin_dgrad(4096, 320, 2560))
        guarded("l2", lambda: lin_dgrad(77, 768, 3072))

    if group == "timing":
        def timeit(name, fn, flops):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            iters = 20
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / iters
            emit(dict(group=group, case=name, ms=ms, tflops=flops / ms / 1e9, ok=True))

        def conv_t(h, cin, cout):
            x = rnd(1, h, h, cin)
            wp = rnd(9 * cout, cin)
            D = torch.empty(h * h, cout, dtype=torch.float16, device=dev)
            cv = dict(img_n=1, img_h=h, img_w=h, out_h=h, out_w=h, kh=3, kw=3, stride=1, pad_top=1, pad_left=1,
                      b_tap_rows=cout, flip_taps=0)
            timeit(f"conv3x3_{h}_{cin}_{cout}",
                   lambda: raw.gemm(x, wp, D, M=h * h, N=cout, K=cin, lda=cin, ldb=cin, ldd=cout, conv=cv),
                   18.0 * cin * cout * h * h)
        guarded("t1", lambda: conv_t(64, 320, 320))
        guarded("t2", lambda: conv_t(64, 640, 640))
        guarded("t3", lambda: conv_t(32, 640, 640))
        guarded("t4", lambda: conv_t(32, 1280, 1280))
        guarded("t5", lambda: conv_t(16, 1280, 1280))
        guarded("t6", lambda: conv_t(8, 1280, 1280))
        guarded("t7", lambda: conv_t(256, 128, 128))
        guarded("t8", lambda: conv_t(512, 128, 128))

        def lin_t(M, N, K):
            A = rnd(M, K)
            B = rnd(N, K)
            D = torch.empty(M, N, dtype=torch.float16, device=dev)
            timeit(f"linear_{M}x{N}x{K}", lambda: raw.gemm(A, B, D, M=M, N=N, K=K, lda=K, ldb=K, ldd=N),
                   2.0 * M * N * K)
            Dt = torch.empty(M, N, dtype=torch.float16, device=dev)
            timeit(f"torch_linear_{M}x{N}x{K}", lambda: torch.matmul(A, B.t(), out=Dt), 2.0 * M * N * K)
        guarded("t9", lambda: lin_t(4096, 2560, 320))
        guarded("t10", lambda: lin_t(4096, 320, 1280))
        guarded("t11", lambda: lin_t(8192, 8192, 8192))
        guarded("t12", lambda: lin_t(16384, 1280, 1280))


if __name__ == "__main__":
    if len(sys.argv) >= 3 and sys.argv[1] == "--group":
        run_group(sys.argv[2])
        sys.exit(0)
    groups = sys.argv[1:] or GROUPS
    for grp in groups:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--group", grp], timeout=240)
            rc = r.returncode
        except subprocess.TimeoutExpired:
            rc = "timeout"
        emit(dict(group=grp, case="__group_exit__", rc=rc, secs=round(time.time() - t0, 1)))
