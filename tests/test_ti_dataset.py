"""CPU tests of the Textual Inversion dataset mirror (ldm.data.personalized.PersonalizedBase, v1-finetune.yaml's data).

The fixture tests/golden/ti_train_tiny.pt was written by the UNMODIFIED reference dataset (oracle/make_golden_ti.py) over
seeded synthetic PNGs that workload.synth_photo_files regenerates here: captions, flip draws, image tensors and the
random / numpy / torch generator states after every item must be the same bits."""
import hashlib
import os
import pickle
import random
import subprocess
import sys
import textwrap

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _digest():
    return hashlib.sha1(pickle.dumps((random.getstate(), np.random.get_state()[1].tobytes(), np.random.get_state()[2],
                                      torch.get_rng_state().numpy().tobytes()))).hexdigest()


def _photos(tmp_path, gold):
    from celebbasis_b200 import workload
    root = str(tmp_path / "photos")
    workload.synth_photo_files(root, seed=gold["photo_seed"])
    assert sorted(os.listdir(root)) == sorted(gold["files"])
    return root


def _load():
    return torch.load(os.path.join(ROOT, "tests", "golden", "ti_train_tiny.pt"), weights_only=False)


def test_personalized_base_matches_reference_items_bit_for_bit(tmp_path):
    from ldm.data.personalized import PersonalizedBase
    gold = _load()
    root = _photos(tmp_path, gold)
    for case in gold["data"]:
        random.seed(gold["seed"])
        np.random.seed(gold["seed"])
        torch.manual_seed(gold["seed"])
        ds = PersonalizedBase(root, size=gold["size"], repeats=4, **case["kwargs"])
        # the file order is os.listdir's, unsorted, as in the reference; replay the order the fixture saw
        assert ds.image_paths == [os.path.join(root, f) for f in os.listdir(root)]
        ds.image_paths = [os.path.join(root, f) for f in gold["files"]]
        assert len(ds) == case["len"]
        for item in case["items"]:
            before = torch.get_rng_state()
            ex = ds[item["index"]]
            assert ex["caption"] == item["caption"], (case["kwargs"], item["index"])
            assert isinstance(ex["caption"], str)
            assert ex["image"].dtype == np.float32 and ex["image"].shape == (gold["size"], gold["size"], 3)
            assert torch.equal(torch.from_numpy(np.ascontiguousarray(ex["image"])), item["image"]), case["kwargs"]
            assert _digest() == item["rng_digest"], (case["kwargs"], item["index"])
            after = torch.get_rng_state()
            torch.set_rng_state(before)
            assert float(torch.rand(1)) == item["flip_draw"]
            torch.set_rng_state(after)


def test_personalized_base_resizes_each_source_once(tmp_path):
    from ldm.data.personalized import PersonalizedBase
    from PIL import Image
    gold = _load()
    root = _photos(tmp_path, gold)
    ds = PersonalizedBase(root, size=16, repeats=3)
    n = ds.num_images
    opened = []
    orig = Image.open

    def spy(path, *a, **k):
        opened.append(path)
        return orig(path, *a, **k)
    Image.open = spy
    try:
        first = [ds[i]["image"] for i in range(len(ds))]
    finally:
        Image.open = orig
    assert len(opened) == n and len(first) == 3 * n
    # a cached source gives the same pixels as a fresh dataset (up to the flip draw)
    fresh = PersonalizedBase(root, size=16, repeats=3, flip_p=0.0)
    cached = PersonalizedBase(root, size=16, repeats=3, flip_p=0.0)
    for i in range(n):
        cached[i]
    for i in range(n, 2 * n):
        assert np.array_equal(cached[i]["image"], fresh[i]["image"])


def test_v1_finetune_data_block_instantiates_the_mirror(tmp_path):
    from celebbasis_b200.compat.omegaconf import OmegaConf
    from ldm.util import instantiate_from_config
    gold = _load()
    root = _photos(tmp_path, gold)
    # configs/stable-diffusion/v1-finetune.yaml data.params.train, with main.py's --data_root / --init_word additions
    cfg = OmegaConf.create({"target": "ldm.data.personalized.PersonalizedBase",
                            "params": {"size": 512, "set": "train", "per_image_tokens": False, "repeats": 1000,
                                       "data_root": root, "placeholder_token": "*", "coarse_class_text": None}})
    ds = instantiate_from_config(cfg)
    assert "celebbasis_b200" in sys.modules[type(ds).__module__].__file__
    assert len(ds) == 1000 * len(gold["files"])
    ex = ds[0]
    assert ex["image"].shape == (512, 512, 3) and ex["image"].dtype == np.float32 and "*" in ex["caption"]


def test_compat_overlay_resolves_personalized_base(tmp_path):
    """A reference checkout's own ldm/data stays on the overlay path; the mirror's PersonalizedBase wins."""
    ref = tmp_path / "ref"
    (ref / "ldm" / "data").mkdir(parents=True)
    (ref / "ldm" / "data" / "only_in_reference.py").write_text("VALUE = 5\n")
    script = ref / "driver.py"
    marker = tmp_path / "ok.txt"
    script.write_text(textwrap.dedent(f"""
        import ldm.data.personalized as P
        from ldm.data.only_in_reference import VALUE
        from ldm.util import instantiate_from_config
        assert "celebbasis_b200" in P.__file__, P.__file__
        cls = instantiate_from_config({{"target": "ldm.data.personalized.PersonalizedBase", "params": {{"data_root": {str(tmp_path)!r}}}}}).__class__
        assert cls is P.PersonalizedBase
        open({str(marker)!r}, "w").write(str(VALUE))
    """))
    env = dict(os.environ, PYTHONPATH=ROOT, PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, "-m", "celebbasis_b200.compat.run", str(script)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert marker.read_text() == "5"
