"""The synthetic CelebBasis training workload (BASELINE.json configs; SURVEY.md §8d "Synthetic inputs").

`model_params(kind)` mirrors configs/stable-diffusion/aigc_id.yaml:model.params of the reference ("full"), or a
structurally identical miniature ("tiny") that CPU parity tests can run in seconds.  `synth_batch` produces the
batch dict FaceIdDatasetOneShot + default collate yield (ldm/data/face_id.py:598-644) and the per-step random draws
(t, noise, posterior eps) so that every implementation replays the same step.
"""
import torch

CAPTION = "a photo of a face of sks person"
PLACEHOLDERS = ['sks', 'ks', 'ata', 'tre', 'ry', 'bop', 'rn', '&', '*', '`']


def model_params(kind="full"):
    full = kind == "full"
    unet = dict(image_size=32, in_channels=4, out_channels=4, model_channels=320 if full else 64,
                attention_resolutions=[4, 2, 1], num_res_blocks=2 if full else 1, channel_mult=[1, 2, 4, 4],
                num_heads=8, use_spatial_transformer=True, transformer_depth=1, context_dim=768,
                use_checkpoint=True, legacy=False)
    dd = dict(double_z=True, z_channels=4, resolution=512 if full else 64, in_channels=3, out_ch=3,
              ch=128 if full else 64, ch_mult=[1, 2, 4, 4], num_res_blocks=2 if full else 1, attn_resolutions=[],
              dropout=0.0)
    return dict(
        linear_start=0.00085, linear_end=0.0120, num_timesteps_cond=1, log_every_t=200, timesteps=1000,
        first_stage_key="image", cond_stage_key="caption", image_size=64 if full else 8, channels=4,
        cond_stage_trainable=True, conditioning_key="crossattn", monitor="val/loss_simple_ema",
        scale_factor=0.18215, use_ema=False, embedding_reg_weight=0.0, unfreeze_model=False, model_lr=0.0,
        personalization_config=dict(
            target="ldm.modules.embedding_manager.EmbeddingManagerId",
            params=dict(placeholder_strings=list(PLACEHOLDERS), initializer_words=["face"] * 10, max_ids=10,
                        num_embeds_per_token=2, meta_mlp_depth=1, loss_type="none", meta_inner_dim=512, meta_heads=1,
                        use_rm_mlp=False, test_mode="coefficient", momentum=0.99, save_fp16=False)),
        unet_config=dict(target="ldm.modules.diffusionmodules.openaimodel.UNetModel", params=unet),
        first_stage_config=dict(target="ldm.models.autoencoder.AutoencoderKL",
                                params=dict(embed_dim=4, monitor="val/rec_loss", ddconfig=dd,
                                            lossconfig=dict(target="torch.nn.Identity"))),
        cond_stage_config=dict(target="ldm.modules.encoders.modules.FrozenCLIPEmbedder",
                               params=dict(use_celeb=False, use_svd=True, rm_repeats=True, n_components=512,
                                           use_sample_reduce=False, n_samples=513, use_flatten=False,
                                           num_embeds_per_token=2, device="cpu")),
    )


def clip_layers(kind="full"):
    return 12 if kind == "full" else 2


def image_hw(kind="full"):
    return 512 if kind == "full" else 64


def synth_batch(kind="full", B=1, seed=1234, step=0):
    """Returns (batch dict on CPU, draws dict with t (B,), noise (B,4,h,w), posterior_eps (B,4,h,w))."""
    hw = image_hw(kind)
    g = torch.Generator().manual_seed(seed + 7919 * step)
    image = torch.rand(B, hw, hw, 3, generator=g) * 2 - 1
    other = torch.rand(B, hw, hw, 3, generator=g) * 2 - 1
    faces = torch.cat([image, other], dim=-1)
    ids = (torch.arange(B) % 10)[:, None].repeat(1, 2).long()
    batch = {"image": image, "caption": [CAPTION] * B,
             "image_ori": {"faces": faces, "ids": ids, "num_ids": torch.ones(B, dtype=torch.long)}}
    lat = hw // 8
    gt = torch.Generator().manual_seed(23 + step)
    draws = {"t": torch.randint(0, 1000, (B,), generator=gt).long(),
             "noise": torch.randn(B, 4, lat, lat, generator=gt),
             "posterior_eps": torch.randn(B, 4, lat, lat, generator=gt)}
    return batch, draws


def ti_model_params(kind="full", num_vectors_per_token=2):
    """configs/stable-diffusion/v1-finetune.yaml:model.params (Textual Inversion: EmbeddingManager, placeholder '*',
    initializer word 'person') on the same UNet / VAE / CLIP sizes as model_params(kind)."""
    p = model_params(kind)
    p["personalization_config"] = dict(
        target="ldm.modules.embedding_manager.EmbeddingManager",
        params=dict(placeholder_strings=["*"], initializer_words=["person"], per_image_tokens=False,
                    num_vectors_per_token=num_vectors_per_token, progressive_words=False))
    return p


def synth_photo_files(out_dir, seed=0, sizes=((40, 56), (64, 48), (37, 37), (50, 33)), modes=("RGB", "RGBA", "L", "P")):
    """Seeded synthetic photos for PersonalizedBase: lossless PNGs, non-square, one per PIL mode (a smooth colour field
    plus noise, so every resampling filter gives different pixels).  Returns the written paths."""
    import os
    import numpy as np
    from PIL import Image
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.RandomState(seed)
    paths = []
    for i, ((h, w), mode) in enumerate(zip(sizes, modes)):
        low = rng.rand(6, 6, 3)
        img = np.asarray(Image.fromarray((low * 255).astype(np.uint8)).resize((w, h), Image.BICUBIC), dtype=np.float32)
        img = Image.fromarray(np.clip(img + rng.randn(h, w, 3) * 12.0, 0, 255).astype(np.uint8))
        if mode == "RGBA":
            img = img.convert("RGBA")
            img.putalpha(Image.fromarray(rng.randint(0, 256, (h, w)).astype(np.uint8)))
        elif mode != "RGB":
            img = img.convert(mode)
        p = os.path.join(out_dir, f"photo_{i}.png")
        img.save(p)
        paths.append(p)
    return paths


def synth_face_files(out_dir, n=4, hw=64, seed=0):
    """n deterministic smooth colour images (stand-ins for aligned face crops) written as lossless PNGs named like the
    reference's fixtures (`0000N_idN.png`: identity = file stem) + the pickle FaceIdDataset* reads (gen_pickle.py: a list
    of paths).  Returns (pickle path, list of image paths)."""
    import os
    import pickle
    import numpy as np
    from PIL import Image
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.RandomState(seed)
    paths = []
    for i in range(n):
        low = rng.rand(8, 8, 3)
        img = np.asarray(Image.fromarray((low * 255).astype(np.uint8)).resize((hw, hw), Image.BICUBIC), dtype=np.float32)
        img = np.clip(img + rng.randn(hw, hw, 3) * 6.0, 0, 255).astype(np.uint8)
        p = os.path.join(out_dir, f"{i:05d}_id{i}.png")
        Image.fromarray(img).save(p)
        paths.append(p)
    pk = os.path.join(out_dir, "ffhq.pickle")
    with open(pk, "wb") as f:
        pickle.dump(paths, f)
    return pk, paths


PERSON_CAPTIONS = {1: "a photo of a face of sks person", 2: "a photo of sks person and ks person",
                   3: "a photo of sks and ks and ata together"}
PERSON_MIX = ([1, 2], [3, 1], [2, 3], [1, 1], [3, 2], [2, 2], [1, 3], [2, 1])
TI_OPTION_CAPTIONS = ["a photo of *", "a photo of sks and *", "a sks photo", "* in a photo of sks"]


def synth_persons_batch(step, B=2, id_cnt=4, seed=11, hw=64):
    """A CelebBasis batch whose prompts name 1, 2 or 3 persons (PERSON_MIX[step]): `id_cnt` face crops and identities
    per sample, identity 3 shared by both samples as their second person, so the EMA order matters."""
    g = torch.Generator().manual_seed(seed + 7919 * step)
    image = torch.rand(B, hw, hw, 3, generator=g) * 2 - 1
    faces = torch.rand(B, hw, hw, 3 * id_cnt, generator=g) * 2 - 1
    ids = torch.stack([torch.randperm(10, generator=g)[:id_cnt] for _ in range(B)])
    ids[:, 1] = 3
    nid = torch.tensor(PERSON_MIX[step % len(PERSON_MIX)][:B], dtype=torch.long)
    return {"image": image, "caption": [PERSON_CAPTIONS[int(k)] for k in nid],
            "image_ori": {"faces": faces, "ids": ids, "num_ids": nid}}


def synth_ti_option_batch(step, B=2, seed=5, hw=64):
    """A Textual Inversion batch naming the placeholders '*' and 'sks' (two per prompt at most)."""
    g = torch.Generator().manual_seed(seed + 7919 * step)
    return {"image": torch.rand(B, hw, hw, 3, generator=g) * 2 - 1,
            "caption": [TI_OPTION_CAPTIONS[(step + b) % len(TI_OPTION_CAPTIONS)] for b in range(B)]}


def option_draws(step, B=2, lat=8, seed=41):
    g = torch.Generator().manual_seed(seed + step)
    return {"t": torch.tensor([0, 999]) if step == 0 else torch.randint(0, 1000, (B,), generator=g).long(),
            "noise": torch.randn(B, 4, lat, lat, generator=g), "posterior_eps": torch.randn(B, 4, lat, lat, generator=g)}
