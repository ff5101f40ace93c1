"""CPU: host-side integer logic, tokenizer, workload, mirror construction, and the world_size-2 data-parallel path."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_placeholder_row_map_matches_reference_kats(golden_dir):
    """Product-side mirror of helpers.py (celebbasis_b200.train_step) against fixtures from the reference itself."""
    from celebbasis_b200.train_step import get_rep_pos, placeholder_row_map
    cases = torch.load(os.path.join(golden_dir, "helpers_kat.pt"))
    for i, c in enumerate(cases):
        tok = c["tokens"].numpy()
        pos = get_rep_pos(tok, c["rep_tokens"])
        assert [p.tolist() for p in pos] == c["rep_pos"]
        src, fin = placeholder_row_map(tok.shape[0], pos, c["reps"])
        assert [f.tolist() for f in fin] == c["final_pos"]
        got = tok[src] if i == 0 else src
        assert got.tolist() == c["result"].tolist()


def test_edge_cases_row_map():
    from celebbasis_b200.train_step import build_inject_map, get_rep_pos, placeholder_row_map
    # no placeholder: identity map, no z rows
    src, fin = placeholder_row_map(77, [np.zeros(0, dtype=np.int64)], 2)
    assert src.tolist() == list(range(77)) and fin[0].shape == (0, 2)
    # reps == 1: rows stay, placeholder row replaced in place
    ids = np.full((1, 77), 49407)
    ids[0, :4] = [49406, 5, 48136, 6]
    m, pos = build_inject_map(ids, 48136, 1, lambda b: b)
    assert m[0, 2] == -1 and (m[0, :2] == [0, 1]).all() and m[0, 3] == 3
    # placeholder in the last usable slot with reps == 2: the tail token is dropped
    ids = np.full((1, 77), 49407)
    ids[0, 0], ids[0, 75] = 49406, 48136
    m, pos = build_inject_map(ids, 48136, 2, lambda b: b)
    assert m[0, 75] == -1 and m[0, 76] == -2 and pos[0][0].tolist() == [[75, 76]]
    # two occurrences
    ids = np.full((1, 77), 49407)
    ids[0, :6] = [49406, 48136, 7, 48136, 8, 9]
    m, pos = build_inject_map(ids, 48136, 2, lambda b: b)
    assert m[0, :8].tolist() == [0, -1, -2, 2, -1, -2, 4, 5] and pos[0][0].tolist() == [[1, 2], [4, 5]]


def test_tokenizer_contract():
    from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
    tok = SyntheticCLIPTokenizer()
    ids = tok(["a photo of a face of sks person", ""])["input_ids"]
    assert ids.shape == (2, 77) and ids.dtype == torch.int64
    assert ids[0, :5].tolist() == [49406, 320, 1125, 539, 320] and int(ids[0, 7]) == 48136 and int(ids[0, 9]) == 49407
    assert ids[1].tolist() == [49406] + [49407] * 76
    assert tok("a photo of Elon Musk")["input_ids"][0, :7].tolist() == [49406, 320, 1125, 539, 20406, 19063, 49407]


def test_mirror_constructs_with_reference_keys():
    """The host mirror exposes the reference's import paths, constructor keywords and state-dict keys."""
    from celebbasis_b200 import synth, workload
    from ldm.models.diffusion.ddpm import LatentDiffusion
    from ldm.util import instantiate_from_config
    params = workload.model_params("tiny")
    params["cond_stage_config"]["params"]["num_hidden_layers"] = 2
    model = instantiate_from_config({"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": params})
    assert isinstance(model, LatentDiffusion)
    keys = set(model.state_dict().keys())
    for k in ["model.diffusion_model.input_blocks.1.1.transformer_blocks.0.attn2.to_k.weight",
              "model.diffusion_model.output_blocks.1.1.conv.weight", "model.diffusion_model.out.2.bias",
              "first_stage_model.encoder.down.0.downsample.conv.weight", "first_stage_model.quant_conv.weight",
              "first_stage_model.decoder.up.1.upsample.conv.bias",
              "cond_stage_model.transformer.text_model.encoder.layers.1.self_attn.q_proj.weight",
              "cond_stage_model.transformer.text_model.embeddings.position_embedding.weight",
              "embedding_manager.meta_id_net.stylegan_mlp.net.0.weight",
              "embedding_manager.meta_id_net.id_model.layer3.29.bn3.running_var", "betas", "alphas_cumprod"]:
        assert k in keys, k
    trainable = [n for n, p in model.named_parameters() if p.requires_grad]
    assert "embedding_manager.meta_id_net.stylegan_mlp.net.0.weight" in trainable
    assert not any(n.startswith(("model.", "first_stage_model.", "cond_stage_model.")) for n in trainable)
    # full-size UNet: 686 tensors / 859.52 M parameters like the reference (SURVEY.md §8 a19)
    from ldm.modules.diffusionmodules.openaimodel import UNetModel
    with torch.device("meta"):
        u = UNetModel(**workload.model_params("full")["unet_config"]["params"])
    assert len(u.state_dict()) == 686 and sum(p.numel() for p in u.parameters()) == 859520964


def test_schedule_buffers_match_oracle():
    from celebbasis_b200 import workload
    from ldm.models.diffusion.ddpm import DDPM
    from oracle import torch_ref
    params = workload.model_params("tiny")
    sched = torch_ref.make_schedule(1000, params["linear_start"], params["linear_end"])
    m = DDPM(params["unet_config"], timesteps=1000, linear_start=params["linear_start"], linear_end=params["linear_end"],
             use_ema=False, conditioning_key="crossattn")
    assert torch.equal(m.sqrt_alphas_cumprod, sched["sqrt_alphas_cumprod"])
    assert torch.equal(m.sqrt_one_minus_alphas_cumprod, sched["sqrt_one_minus_alphas_cumprod"])


def _dp_worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from celebbasis_b200 import dist as cbd
    w, r, _ = cbd.init(backend="gloo")
    assert (w, r) == (world, rank)
    g = torch.full((1024 * 512 + 1024,), float(rank + 1))
    cbd.allreduce_mean_(g)
    owned = cbd.identity_shard(10)
    coeff = torch.zeros(10, 2, 1, 4)
    for i in owned:
        coeff[i] = i + 1
    full = cbd.gather_identity_state(coeff, owned, 10)
    # identities that NO rank trained keep their initial value (identical on all ranks)
    init = torch.full((10, 2, 1, 4), 7.0)
    part = init.clone()
    part[rank] = 100.0 + rank
    kept = cbd.gather_identity_state(part, [rank], 10)
    assert float(kept[0, 0, 0, 0]) == 100.0 and float(kept[1, 0, 0, 0]) == 101.0 and bool((kept[2:] == 7.0).all())
    torch.save({"g0": g[0].item(), "gl": g[-1].item(), "owned": owned, "full": full, "lr": cbd.scaled_lr(5e-3, 1)},
               os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


def test_data_parallel_gloo_world2(tmp_path):
    """N>1 path on CPU: one collective on the flat gradient (mean), identity sharding, EMA gather, LR scaling."""
    import torch.multiprocessing as mp
    port = 29000 + (os.getpid() % 2000)
    mp.spawn(_dp_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    assert r0["g0"] == r1["g0"] == 1.5 and r0["gl"] == 1.5
    assert r0["owned"] == [0, 2, 4, 6, 8] and r1["owned"] == [1, 3, 5, 7, 9]
    expect = torch.arange(1, 11).float().view(10, 1, 1, 1).expand(10, 2, 1, 4)
    assert torch.equal(r0["full"], expect) and torch.equal(r1["full"], expect)
    assert abs(r0["lr"] - 2 * 5e-3) < 1e-12


def test_gemm_autotune_key_and_lanes():
    """Host plumbing of the tile autotuner and of the per-branch workspace lanes (no GPU needed)."""
    from celebbasis_b200 import ops
    from celebbasis_b200.lib import GemmDesc
    a, b = GemmDesc(), GemmDesc()
    for d in (a, b):
        d.M, d.N, d.K, d.batch, d.lda, d.ldb, d.ldd = 4096, 320, 320, 1, 320, 320, 320
    assert ops._tune_key(a) == ops._tune_key(b)
    b.conv, b.kh, b.kw = 1, 3, 3
    assert ops._tune_key(a) != ops._tune_key(b)
    b = GemmDesc.from_buffer_copy(bytes(a))
    b.tile_n, b.splits, b.stages, b.cta_pair = 128, 3, 3, 1   # tuning overrides are not part of the shape key
    assert ops._tune_key(a) == ops._tune_key(b)
    assert ops._LANE == 0
    with ops.lane(1):
        assert ops._LANE == 1
        with ops.lane(0):
            assert ops._LANE == 0
        assert ops._LANE == 1
    assert ops._LANE == 0


def test_gemm_config_and_groupnorm_flags_per_lane(monkeypatch):
    """The autotuner's winner reaches cb_gemm through the descriptor; a winner that launches a cluster of k-slices
    (splitk_cluster) is only used on the lane-0 stream -- other lanes take the best non-cluster configuration -- and the
    front-end SM budget turns large lane-2 GEMMs into capped CTA-pair launches (no GPU: cb_gemm is a recording stub) and
    caps the lane-2 GroupNorm's CTAs through its flag word (SiLU in bit 0, CB_GN_CTA_CAP(n) in bits 8..23)."""
    import torch
    from celebbasis_b200 import ops
    from celebbasis_b200.lib import GemmDesc
    seen = []

    class FakeLib:
        def cb_gemm(self, dref, stream):
            d = dref._obj
            seen.append((d.tile_n, d.splits, d.stages, d.cta_pair, d.splitk_cluster))
            return 0

    class FakeWs:
        def data_ptr(self):
            return 0x1000

        def numel(self):
            return 1 << 20
    monkeypatch.setattr(ops, "_L", lambda: FakeLib())
    monkeypatch.setattr(ops, "_st", lambda: None)
    monkeypatch.setattr(ops, "_splitk_workspace", lambda dev: FakeWs())
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)    # never autotune here
    monkeypatch.setattr(ops, "AUTOTUNE", True)
    monkeypatch.setattr(ops, "CLUSTER_SK_ALL_LANES", False)
    monkeypatch.setattr(ops, "FE_CTAS", 0)

    def desc(M=77, N=768, K=768):
        d = GemmDesc()
        d.M, d.N, d.K, d.batch, d.lda, d.ldb, d.ldd = M, N, K, 1, K, K, N
        return d
    key = ops._tune_key(desc())
    monkeypatch.setitem(ops._TUNE, key, (64, 4, 0, 0, 1))
    monkeypatch.setitem(ops._TUNE_NC, key, (64, 6, 0, 0, 0))
    ops._gemm(desc(), "t")                                  # lane 0: the cluster winner
    with ops.lane(3):
        ops._gemm(desc(), "t")                              # text branch on its own stream: best non-cluster configuration
    monkeypatch.setattr(ops, "CLUSTER_SK_ALL_LANES", True)
    with ops.lane(3):
        ops._gemm(desc(), "t")
    assert seen == [(64, 4, 0, 0, 1), (64, 6, 0, 0, 0), (64, 4, 0, 0, 1)]
    # an explicit configuration from the caller is never overridden
    d = desc()
    d.tile_n, d.splits = 128, 2
    ops._gemm(d, "t")
    assert seen[-1] == (128, 2, 0, 0, 0)
    # untuned shape while capturing: the library's own cost model (all zeros)
    ops._gemm(desc(M=4096, N=320, K=320), "t")
    assert seen[-1] == (0, 0, 0, 0, 0)
    # front-end SM budget: lane 2, M >= 2048, K-major A -> persistent CTA-pair kernel on at most FE_CTAS CTAs
    monkeypatch.setattr(ops, "FE_CTAS", 64)
    with ops.lane(2):
        ops._gemm(desc(M=65536, N=256, K=256), "t")
        ops._gemm(desc(M=65536, N=128, K=128), "t")
        ops._gemm(desc(M=512, N=256, K=256), "t")           # small: untouched
    assert seen[-3:] == [(256, 1, 0, 64, 0), (128, 1, 0, 64, 0), (0, 0, 0, 0, 0)]
    ops._gemm(desc(M=65536, N=256, K=256), "t")              # lane 0: no budget
    assert seen[-1] == (0, 0, 0, 0, 0)
    assert ops._gn_flags(True) == 1
    with ops.lane(2):
        assert ops._gn_flags(True) == (1 | (64 << 8))        # SiLU | CB_GN_CTA_CAP(64)


def test_groupnorm_cluster_plan_covers_the_step():
    """cb_groupnorm_cluster_plan (host-only entry point of the library): every GroupNorm of the bs=1 SD-v1 UNet step --
    forward (fp32 or 16-bit input) and backward (input + 16-bit gradient staged) -- runs on the cluster variant: 128 CTAs as
    8 slabs x 16, staged rows within 200 KiB; each CTA's thread map (4-channel accesses, row lanes) touches every element of
    its rows x slab exactly once; tensors that do not fit (VAE 512^2 maps, a 16-image UNet batch) report 0.  The route of
    every forward of the VAE encoder (bs=1), the txt2img UNet (16 images: classifier-free guidance at batch 8) and the VAE
    decoder (1 and 8 images) is pinned, and every shape without a plan has the 16-byte rows the streaming pair needs;
    cb_groupnorm_fwd refuses other rows before any launch."""
    import ctypes
    import numpy as np
    from celebbasis_b200 import lib
    L = lib.load()
    plan = (ctypes.c_int32 * 4)()

    def ask(N, HW, C, bpe):
        rc = L.cb_groupnorm_cluster_plan(N, HW, C, 32, bpe, ctypes.cast(plan, ctypes.c_void_p))
        assert rc in (0, 1), (rc, N, HW, C)
        return tuple(plan) if rc == 1 else None
    unet = [(4096, 320), (4096, 640), (4096, 960), (1024, 320), (1024, 640), (1024, 960), (1024, 1280), (1024, 1920),
            (256, 640), (256, 1280), (256, 1920), (256, 2560), (64, 1280), (64, 2560)]
    for hw, c in unet:
        for bpe in (4, 2, 6, 4 + 4):                      # fwd fp32 / fwd 16-bit / bwd fp32 x + 16-bit dy / bwd fp32 + fp32
            p = ask(1, hw, c, bpe)
            if p is None:
                assert bpe == 8 and hw * c * bpe > 128 * 200 * 1024      # only the all-fp32 backward of the widest 64^2 map
                continue
            S, gpc, rows, smem = p
            cpg, cw = c // 32, gpc * (c // 32)
            assert S * (32 // gpc) <= 132 and S * rows >= hw and S <= 16 and 32 % gpc == 0
            assert rows * cw * bpe <= smem <= 200 * 1024 and cw % 4 == 0
            # the kernels' thread map on one CTA: quad cq = tid % nq, row lane ry = tid // nq, RY = 512 // nq row lanes
            nq = cw // 4
            RY = 512 // nq
            assert 1 <= RY and nq >= 2
            cover = np.zeros((min(rows, 40), cw), dtype=np.int32)
            for tid in range(512):
                cq, ry = tid % nq, tid // nq
                if ry >= RY:
                    continue
                assert (4 * cq) // cpg < gpc and (4 * cq + 2) // cpg < gpc
                cover[ry::RY, 4 * cq:4 * cq + 4] += 1
            assert (cover == 1).all()
    assert ask(1, 512 * 512, 128, 4) is None and ask(16, 4096, 320, 4) is None and ask(2, 4096, 960, 4) is None
    assert ask(2, 4096, 320, 4)[0] == 8 and ask(4, 64, 320, 4)[0] == 4 and ask(1, 1, 256, 4)[0] == 1
    assert L.cb_groupnorm_cluster_plan(1, 64, 48, 32, 4, ctypes.cast(plan, ctypes.c_void_p)) < 0      # odd channels per group
    enc = [(512 * 512, 128), (256 * 256, 128), (256 * 256, 256), (128 * 128, 256), (128 * 128, 512), (64 * 64, 512)]
    dec = [(64 * 64, 512), (128 * 128, 512), (256 * 256, 512), (256 * 256, 256), (512 * 512, 256), (512 * 512, 128)]
    # (images, (HW, C) shapes, the (HW, C, sizeof(x)) forwards that take the cluster kernel); x is fp32 or 16-bit
    routes = [
        (1, enc, {(256 * 256, 128, 2), (128 * 128, 256, 4), (128 * 128, 256, 2), (128 * 128, 512, 2), (64 * 64, 512, 4),
                  (64 * 64, 512, 2)}),
        (16, unet, {(4096, 320, 2), (1024, 320, 4), (1024, 320, 2), (1024, 640, 4), (1024, 640, 2), (1024, 960, 2),
                    (1024, 1280, 2)} | {(hw, c, bpe) for hw, c in unet if hw <= 256 for bpe in (4, 2)}),
        (1, dec, {(64 * 64, 512, 4), (64 * 64, 512, 2), (128 * 128, 512, 2)}),
        (8, dec, {(64 * 64, 512, 2)}),
    ]
    for N, shapes, cluster in routes:
        for hw, c in shapes:
            for bpe in (4, 2):
                assert (ask(N, hw, c, bpe) is not None) == ((hw, c, bpe) in cluster), (N, hw, c, bpe)
                assert (hw, c, bpe) in cluster or c * bpe % 16 == 0, (N, hw, c, bpe)    # the streaming pair's rows
    # rows that are not a multiple of 16 bytes (G = 3, C = 6, fp16: 12-byte rows): refused before anything is launched
    assert L.cb_groupnorm_fwd(None, lib.CB_F16, None, lib.CB_F16, None, None, 1, 16, 6, 3, 1e-5, 0, None, None, None,
                              None) < 0
    assert b"16 bytes" in L.cb_last_error()


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the arm the driver times beside ours): the oracle port of the reference step on the host
    cores, one JSON line with the contract's keys (no GPU involved)."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=900, cwd=root,
                       env=dict(os.environ, CB_BENCH_CPU_MIN_STEPS="2"))
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    out = json.loads(lines[0])
    assert out["impl"] == "reference" and out["unit"] == "steps/s" and out["value"] > 0 and out["higher_is_better"] is True
    assert out["metric"].startswith("celeb-basis training steps/sec") and out["n_gpus"] == 1
    assert out["cpu_baseline"]["kind"] == "port" and 1 <= out["cpu_baseline"]["cores"] <= len(os.sched_getaffinity(0))
    assert "first step dropped as cold" in out["cpu_baseline"]["sample"]
    assert set(out["config"]) == {"workload", "per_gpu_batch", "parallelism", "l2"}
    assert out["e2e"]["h2d_bytes_per_step"] == 0 and out["e2e"]["d2h_bytes_per_step"] == 0 and out["e2e"]["value"] == out["value"]


def test_embedding_checkpoint_format_matches_reference(golden_dir, tmp_path):
    """SURVEY a32: the file `EmbeddingManagerId.save` writes every checkpoint and `scripts/stable_txt2img.py:230` loads
    (embedding_manager.py:396-426).  The fixture was written by the UNMODIFIED reference's save(); the mirror must read it
    and write the same structure (keys, container types, dtypes, shapes) in both precisions."""
    import torch.nn.functional as F
    from celebbasis_b200 import workload
    from ldm.models.diffusion.ddpm import LatentDiffusion
    gold = torch.load(os.path.join(golden_dir, "embeddings_ref.pt"))
    params = workload.model_params("tiny")
    params["cond_stage_config"]["params"]["num_hidden_layers"] = 2
    em = LatentDiffusion(**params).embedding_manager
    g = torch.Generator().manual_seed(gold["coef_seed"])
    coefs = [F.normalize(torch.randn(2, 1, 512, generator=g), dim=-1) for _ in range(10)]
    for prec, save_fp16 in (("fp32", False), ("fp16", True)):
        ref_file = tmp_path / f"ref_{prec}.pt"
        torch.save(gold[prec], ref_file)
        em.load(str(ref_file))                                             # reference-written file -> mirror
        assert len(em.id_coefficients) == 10 and all(c.dtype == torch.float32 for c in em.id_coefficients)
        tol = 0.0 if prec == "fp32" else 1e-3
        for got, want in zip(em.id_coefficients, coefs):
            assert (got - want).abs().max().item() <= tol
        em.save_fp16 = save_fp16
        out_file = tmp_path / f"mirror_{prec}.pt"
        em.save(str(out_file))                                             # mirror-written file == reference structure
        mine = torch.load(out_file)
        assert set(mine.keys()) == set(gold[prec].keys())
        for k in mine:
            assert type(mine[k]) is type(gold[prec][k]) and len(mine[k]) == len(gold[prec][k])
            for a, b in zip(mine[k], gold[prec][k]):
                assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    em.save_fp16 = False


def test_celeb_basis_construction_vs_reference(golden_dir, tmp_path):
    """SURVEY f3: FrozenCLIPEmbedder._get_celeb_embeddings (modules.py:472-624).  The fixture was produced by the
    UNMODIFIED reference on infer_images/wiki_names_v2.txt with the real CLIP BPE ids of infer_images/token_len.txt
    (oracle/make_golden.py basis): per-column basis (aigc_id.yaml), the flattened basis (constructor default) and the
    sample-reduced variant.  Singular vectors are compared up to sign."""
    from celebbasis_b200 import synth
    from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
    from ldm.modules.encoders.modules import FrozenCLIPEmbedder
    gold = torch.load(os.path.join(golden_dir, "celeb_basis.pt"), weights_only=False)
    names_file = tmp_path / "names.txt"
    names_file.write_text("\n".join(gold["names"]) + "\n")
    for case in gold["cases"]:
        emb = FrozenCLIPEmbedder(device="cpu", celeb_txt=str(names_file), use_celeb=False, use_svd=True, n_components=512,
                                 rm_repeats=True, n_samples=513, num_embeds_per_token=2, num_hidden_layers=1, **case["cfg"])
        emb.tokenizer = SyntheticCLIPTokenizer(phrases=gold["phrases"])
        sd = synth.synth_state_dict(emb, seed=0, prefix="cond_stage_model.")
        emb.load_state_dict({k: v for k, v in sd.items() if "token_embedding" in k}, strict=False)
        emb._get_celeb_embeddings(512)
        ce = emb.celeb_embeddings.float().cpu()
        assert tuple(ce.shape) == tuple(case["shape"]) == (2, 513, 768)
        assert torch.allclose(ce[:, 0], case["mean_rows"], atol=1e-6), case["cfg"]
        assert torch.allclose(ce.norm(dim=-1), case["row_norms"], atol=1e-4)
        head = case["head"]
        cosv = (ce[:, 1:33] * head[:, 1:33]).sum(-1).abs()                  # right-singular vectors: up to sign
        assert float(cosv.min()) > 0.9999, (case["cfg"], float(cosv.min()))
        eye = torch.eye(512)
        assert float((ce[0, 1:] @ ce[0, 1:].t() - eye).abs().max()) < 1e-4    # orthonormal basis rows
        if case["cfg"]["use_flatten"]:
            assert torch.equal(ce[0], ce[1])                                   # the one flat basis, repeated (:617-618)


def test_textual_inversion_row_map_vs_reference(golden_dir):
    """SURVEY f4 (integer path, bit-exact): the host row map of the vanilla EmbeddingManager reproduces the UNMODIFIED
    reference's forward (embedding_manager.py:96-151) -- replacement for one vector per token, right-to-left expansion with
    truncation for three, the in-place token rewrite a later placeholder sees."""
    from ldm.modules.embedding_manager import build_ti_map
    gold = torch.load(os.path.join(golden_dir, "ti_manager.pt"), weights_only=False)
    for case in gold["cases"]:
        g = torch.Generator().manual_seed(case["text_seed"])
        text = torch.randn(len(gold["prompts"]), 77, 768, generator=g)
        assert abs(float(text.double().sum()) - case["text_sum"]) < 1e-6
        nv = case["nv"]
        placeholders, base, z = [], 0, []
        for key, tok in case["tokens"].items():
            placeholders.append((tok, base, nv))
            z.append(case["params"][key])
            base += nv
        m, new_tok = build_ti_map(case["ids"].numpy(), placeholders, nv, nv)
        zr = torch.cat(z, 0)
        out = torch.empty_like(text)
        for b in range(text.shape[0]):
            for i in range(77):
                out[b, i] = text[b, m[b, i]] if m[b, i] >= 0 else zr[-(m[b, i] + 1)]
        exp = torch.randn(len(gold["prompts"]), 77, 768, generator=torch.Generator().manual_seed(case["text_seed"]))
        exp[case["out_rows"][:, 0], case["out_rows"][:, 1]] = case["out_vals"]      # rows the manager rewrote
        assert torch.equal(out, exp), nv
        if nv > 1:
            assert torch.equal(torch.from_numpy(new_tok), case["ids_after"])
        assert case["ckpt_keys"] == ["string_to_param", "string_to_token"]


def _rng_digest():
    import hashlib
    import pickle
    import random
    return hashlib.sha1(pickle.dumps((random.getstate(), np.random.get_state()[1].tobytes(), np.random.get_state()[2],
                                      torch.get_rng_state().numpy().tobytes()))).hexdigest()


def test_data_path_draws_match_reference(golden_dir, tmp_path):
    """SURVEY f2 (host half): the dataset mirror makes exactly the reference's random draws -- after every __getitem__ the
    state of python's `random`, numpy's and torch's generators equals the state the UNMODIFIED reference dataset left
    behind (fixture: oracle/make_golden.py data), and captions / identity lists / dataset length are identical."""
    import random
    from celebbasis_b200 import workload
    from ldm.data.face_id import FaceIdDatasetOneShot
    gold = torch.load(os.path.join(golden_dir, "data_path.pt"), weights_only=False)
    pk, _ = workload.synth_face_files(str(tmp_path), n=4, hw=gold["hw"], seed=0)
    items = iter(gold["items"])
    for split, diff in (("train", 0), ("train", 1)):
        random.seed(gold["seed"])
        np.random.seed(gold["seed"])
        torch.manual_seed(gold["seed"])
        ds = FaceIdDatasetOneShot(pk, num_ids=3, specific_ids=[0, 1, 3], image_size=gold["hw"], repeats=5, split=split,
                                  diff_cnt=diff)
        for i in (0, 4, 7):
            g = next(items)
            ex = ds[i]
            assert len(ds) == g["len"] and ex["caption"] == g["caption"]
            assert ex["image_ori"]["ids"].tolist() == g["ids"].tolist() and ex["image_ori"]["num_ids"] == g["num_ids"]
            assert _rng_digest() == g["rng_digest"], (split, diff, i)
            k = 2 + 2 * diff
            assert ex["image_u8"].shape == (k, gold["hw"], gold["hw"], 3) and ex["image_u8"].dtype == torch.uint8
            rh, rw, ph, pw = ex["aug_geo"].tolist()
            # the pasted rectangle of the reference's `image` is where it differs from the -1 background
            ref_img = g["image"]
            inside = ref_img[ph:ph + rh, pw:pw + rw]
            outside = ref_img.clone()
            outside[ph:ph + rh, pw:pw + rw] = -1.0
            assert float((outside + 1.0).abs().max()) == 0.0 and inside.shape[:2] == (rh, rw)


def test_glu_interleave_and_host_limits():
    """Host helpers added in round 2: the FF-in weight interleave of the GEGLU epilogue is a permutation that maps value row
    32*g+i -> 64*g+i and gate row F+32*g+i -> 64*g+32+i; the CPU-arm thread limit never exceeds the scheduler affinity."""
    import importlib
    from celebbasis_b200 import ops
    F_ = 96
    w = torch.arange(2 * F_ * 3, dtype=torch.float32).view(2 * F_, 3)
    il = ops.glu_interleave_rows(w)
    assert il.shape == w.shape and sorted(il[:, 0].tolist()) == sorted(w[:, 0].tolist())
    for g in range(F_ // 32):
        assert torch.equal(il[64 * g: 64 * g + 32], w[32 * g: 32 * g + 32])
        assert torch.equal(il[64 * g + 32: 64 * g + 64], w[F_ + 32 * g: F_ + 32 * g + 32])
    bench = importlib.import_module("bench")
    lim = bench.host_cpu_limits()
    assert 1 <= lim["limit"] <= lim["affinity"] <= (os.cpu_count() or 1)
