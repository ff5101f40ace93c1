"""Host mirror of ldm/data/personalized.py: the Textual Inversion dataset of configs/stable-diffusion/v1-finetune.yaml.

`PersonalizedBase` keeps the reference's constructor keywords, length, file order (`os.listdir`, unsorted), caption
templates and -- call for call -- its random draws: `np.random.uniform()` only with `per_image_tokens`, then
`random.choice` of the template, then the `torch.rand(1)` of the horizontal flip.  Items are the same bits: PIL's RGB
conversion, the integer centre crop and PIL's resize with the selected filter, the flip after the resize, and
`image / 127.5 - 1.0` in float64 cast to float32.

The resized source image is a pure function of (file, size, filter), so it is computed once per source image and kept;
an item then costs only its caption draw, the flip and the normalisation.  Training reads each photo `repeats` times
per epoch, and decoding plus resampling a full-size phone photo dominates the per-item cost otherwise.
"""
import os
import random

import numpy as np
import torch
from PIL import Image
from torch.utils.data import Dataset

from ldm.data.face_id import imagenet_templates_small, imagenet_templates_smallest  # noqa: F401  (same 81 templates)

imagenet_dual_templates_small = [t.replace("{}", "{} with {}") for t in imagenet_templates_small[:27]]

per_img_token_list = [
    'א', 'ב', 'ג', 'ד', 'ה', 'ו', 'ז', 'ח', 'ט', 'י', 'כ', 'ל', 'מ', 'נ', 'ס', 'ע', 'פ', 'צ', 'ק', 'ר', 'ש', 'ת',
]

# "linear" was Pillow's alias of BILINEAR until Pillow 10 removed the name
_FILTERS = {"linear": Image.BILINEAR, "bilinear": Image.BILINEAR, "bicubic": Image.BICUBIC, "lanczos": Image.LANCZOS}


class PersonalizedBase(Dataset):
    def __init__(self, data_root, size=None, repeats=100, interpolation="bicubic", flip_p=0.5, set="train",
                 placeholder_token="*", per_image_tokens=False, center_crop=False, mixing_prob=0.25,
                 coarse_class_text=None):
        self.data_root = data_root
        self.image_paths = [os.path.join(self.data_root, name) for name in os.listdir(self.data_root)]
        self.num_images = len(self.image_paths)
        self._length = self.num_images
        self.placeholder_token = placeholder_token
        self.per_image_tokens = per_image_tokens
        self.center_crop = center_crop
        self.mixing_prob = mixing_prob
        self.coarse_class_text = coarse_class_text
        if per_image_tokens:
            assert self.num_images < len(per_img_token_list), (
                f"Can't use per-image tokens when the training set contains more than {len(per_img_token_list)} "
                f"tokens. To enable larger sets, add more tokens to 'per_img_token_list'.")
        if set == "train":
            self._length = self.num_images * repeats
        self.size = size
        self.interpolation = _FILTERS[interpolation]
        self.flip_p = flip_p
        self._pixels = {}           # source index -> cropped + resized uint8 HWC image

    def __len__(self):
        return self._length

    def _resized(self, k):
        img = self._pixels.get(k)
        if img is None:
            image = Image.open(self.image_paths[k])
            if image.mode != "RGB":
                image = image.convert("RGB")
            arr = np.array(image).astype(np.uint8)
            if self.center_crop:
                crop = min(arr.shape[0], arr.shape[1])
                h, w = arr.shape[0], arr.shape[1]
                arr = arr[(h - crop) // 2:(h + crop) // 2, (w - crop) // 2:(w + crop) // 2]
            image = Image.fromarray(arr)
            if self.size is not None:
                image = image.resize((self.size, self.size), resample=self.interpolation)
            img = np.array(image).astype(np.uint8)
            self._pixels[k] = img
        return img

    def __getitem__(self, i):
        k = i % self.num_images
        placeholder_string = self.placeholder_token
        if self.coarse_class_text:
            placeholder_string = f"{self.coarse_class_text} {placeholder_string}"
        if self.per_image_tokens and np.random.uniform() < self.mixing_prob:
            text = random.choice(imagenet_dual_templates_small).format(placeholder_string, per_img_token_list[k])
        else:
            text = random.choice(imagenet_templates_small).format(placeholder_string)
        img = self._resized(k)
        if torch.rand(1) < self.flip_p:         # torchvision's RandomHorizontalFlip draw, after the resize
            img = img[:, ::-1]
        return {"caption": text, "image": (img / 127.5 - 1.0).astype(np.float32)}
