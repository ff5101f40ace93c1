"""CPU tests of the driver-compatibility layer (SURVEY.md 8b / 8f-1): omegaconf + pytorch_lightning stand-ins and the
script runner.  The stand-ins are exercised under their own package names so a real installation is never shadowed."""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

YAML = """
model:
  base_learning_rate: 5.0e-03
  target: ldm.models.diffusion.ddpm.LatentDiffusion
  params:
    timesteps: 1000
    personalization_config:
      target: ldm.modules.embedding_manager.EmbeddingManagerId
      params:
        placeholder_strings: ["*"]
        initializer_words: ["sculpture"]
        num_embeds_per_token: 2
    unet_config:
      params:
        attention_resolutions: [4, 2, 1]
        channel_mult: [1, 2, 4, 4]
data:
  params:
    batch_size: 2
lightning:
  trainer:
    max_steps: 800
"""


def test_omegaconf_standin(tmp_path):
    from celebbasis_b200.compat.omegaconf import DictConfig, ListConfig, OmegaConf
    f = tmp_path / "cfg.yaml"
    f.write_text(YAML)
    cfg = OmegaConf.load(str(f))
    assert cfg.model.params.timesteps == 1000 and cfg["model"]["base_learning_rate"] == 5e-3
    assert type(cfg.model.params.unet_config.params.channel_mult) is ListConfig          # openaimodel.py:476 checks the type
    assert "target" in cfg.model and cfg.model.get("nope", 7) == 7
    # main_id_embed.py:590-595,611-617: merge with the CLI dotlist, pop the lightning section, item assignment through attrs
    cli = OmegaConf.from_dotlist(["model.params.timesteps=500", "data.params.batch_size=4", "model.base_learning_rate=1e-3"])
    merged = OmegaConf.merge(cfg, cli)
    assert merged.model.params.timesteps == 500 and merged.data.params.batch_size == 4
    assert merged.model.base_learning_rate == pytest.approx(1e-3)
    assert cfg.model.params.timesteps == 1000                                             # inputs untouched
    light = merged.pop("lightning", OmegaConf.create())
    assert light.trainer.max_steps == 800 and "lightning" not in merged
    merged.model.params.personalization_config.params.embedding_manager_ckpt = "x.pt"
    merged.model.params.personalization_config.params.initializer_words[0] = "face"
    assert merged.model.params.personalization_config.params["embedding_manager_ckpt"] == "x.pt"
    trainer_cfg = light.get("trainer", OmegaConf.create())
    trainer_cfg["accelerator"] = "ddp"
    del trainer_cfg["accelerator"]
    assert isinstance(OmegaConf.create({"a": {"b": 1}}).a, DictConfig)
    # yaml round trip (SetupCallback prints and saves the configs, main_id_embed.py:323-330)
    out = tmp_path / "saved.yaml"
    OmegaConf.save(merged, str(out))
    again = OmegaConf.load(str(out))
    assert OmegaConf.to_container(again) == OmegaConf.to_container(merged)
    assert "timesteps: 500" in OmegaConf.to_yaml(merged)


def test_instantiate_from_config_with_standin_config():
    from celebbasis_b200.compat.omegaconf import OmegaConf
    from ldm.util import instantiate_from_config
    cfg = OmegaConf.create({"target": "torch.nn.Linear", "params": {"in_features": 3, "out_features": 2}})
    lin = instantiate_from_config(cfg)
    assert isinstance(lin, torch.nn.Linear) and lin.weight.shape == (2, 3)


def test_trainer_standin_fit_loop(tmp_path):
    from celebbasis_b200.compat import pytorch_lightning as pl
    from celebbasis_b200.compat.pytorch_lightning.callbacks import LearningRateMonitor, ModelCheckpoint
    events = []

    class Toy(pl.LightningModule):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(4))
            self.frozen = torch.nn.Parameter(torch.ones(4), requires_grad=False)
            self.learning_rate = 0.1

        def training_step(self, batch, batch_idx):
            loss = ((self.w - batch["x"].mean(0)) ** 2).sum()
            self.log("train/loss", loss)
            return loss

        def on_train_batch_end(self, *args, **kwargs):
            events.append(("module_batch_end", self.global_step))

        def configure_optimizers(self):
            return torch.optim.SGD([self.w], lr=self.learning_rate)

        def on_save_checkpoint(self, checkpoint):
            checkpoint["extra"] = {"steps": self.global_step}

    class Spy(pl.Callback):
        def on_pretrain_routine_start(self, trainer, pl_module):
            events.append(("pretrain", trainer.global_step))

        def on_train_batch_end(self, trainer, pl_module, outputs, batch, batch_idx, dataloader_idx=0):
            events.append(("cb_batch_end", trainer.global_step, float(outputs["loss"])))

        def on_train_end(self, trainer, pl_module):
            events.append(("end", trainer.global_step))

    class Data(pl.LightningDataModule):
        def setup(self, stage=None):
            self.datasets = {"train": [{"x": torch.full((4,), float(i))} for i in range(3)]}

        def train_dataloader(self):
            return torch.utils.data.DataLoader(self.datasets["train"], batch_size=1)

    ck = ModelCheckpoint(dirpath=str(tmp_path / "ck"), filename="gs-{step}", every_n_train_steps=2, save_last=True)
    import argparse
    parser = pl.Trainer.add_argparse_args(argparse.ArgumentParser())
    ns = parser.parse_args(["--max_steps", "5"])
    trainer = pl.Trainer.from_argparse_args(ns, callbacks=[Spy(), ck, LearningRateMonitor("step")], logger=None)
    model = Toy()
    trainer.fit(model, Data())
    assert trainer.global_step == 5 and trainer.current_epoch >= 1            # 3 batches per epoch -> second epoch entered
    assert events[0] == ("pretrain", 0) and events[-1] == ("end", 5)
    losses = [e[2] for e in events if e[0] == "cb_batch_end"]
    assert len(losses) == 5 and model.w.abs().sum() > 0
    assert float(model.frozen.sum()) == 4.0
    assert sorted(os.listdir(tmp_path / "ck")) == ["gs-2.ckpt", "gs-4.ckpt", "last.ckpt"]
    ckpt = torch.load(tmp_path / "ck" / "last.ckpt", map_location="cpu")
    assert ckpt["global_step"] == 5 and ckpt["extra"] == {"steps": 5} and "w" in ckpt["state_dict"]
    assert trainer.logged_metrics["lr-SGD"] == pytest.approx(0.1) and "train/loss" in trainer.logged_metrics
    assert pl.seed_everything(7) == 7 and trainer.profiler.summary() == "" and trainer.training_type_plugin.reduce(3.0) == 3.0


def test_compat_run_executes_script_with_standins(tmp_path):
    script = tmp_path / "driver.py"
    marker = tmp_path / "ok.txt"
    script.write_text(textwrap.dedent(f"""
        import sys
        from omegaconf import OmegaConf
        from omegaconf.listconfig import ListConfig
        from pytorch_lightning import seed_everything
        from pytorch_lightning.trainer import Trainer
        from pytorch_lightning.callbacks import ModelCheckpoint, Callback, LearningRateMonitor
        from pytorch_lightning.utilities.distributed import rank_zero_only
        from pytorch_lightning.utilities import rank_zero_info
        from taming.modules.vqvae.quantize import VectorQuantizer2
        import kornia, clip
        from ldm.util import instantiate_from_config
        from ldm.models.diffusion.ddim import DDIMSampler
        from ldm.models.diffusion.plms import PLMSSampler
        import ldm
        assert "celebbasis_b200" in ldm.__path__[0], ldm.__path__
        seed_everything(int(sys.argv[1]))
        open({str(marker)!r}, "w").write(OmegaConf.to_yaml(OmegaConf.create({{"seed": int(sys.argv[1])}})))
    """))
    env = dict(os.environ, PYTHONPATH=ROOT, PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, "-m", "celebbasis_b200.compat.run", str(script), "23"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert marker.read_text().strip() == "seed: 23"


def _ddp_sampler_worker(rank, world, port, out_dir):
    import sys
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    sys.path.insert(0, ROOT)
    from celebbasis_b200.compat import pytorch_lightning as pl
    pl.seed_everything(23)                    # main_id_embed.py seeds every rank identically
    seen = []

    class Toy(pl.LightningModule):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(1))

        def training_step(self, batch, batch_idx):
            seen.extend(int(i) for i in batch["idx"])
            return (self.w * batch["x"].float().mean()).sum()

        def configure_optimizers(self):
            return torch.optim.SGD([self.w], lr=0.1)

    ds = [{"idx": i, "x": torch.tensor(float(i))} for i in range(8)]
    loader = torch.utils.data.DataLoader(ds, batch_size=2, shuffle=True)
    tr = pl.Trainer(max_epochs=2)
    model = Toy()
    tr.fit(model, train_dataloaders=loader)
    torch.save({"seen": seen, "w": model.w.detach().clone()}, os.path.join(out_dir, f"r{rank}.pt"))
    import torch.distributed as dist
    dist.destroy_process_group()


def test_trainer_installs_distributed_sampler_world2(tmp_path):
    """ADVICE r1 (medium): with WORLD_SIZE > 1 Lightning replaces the sampler by a DistributedSampler; without it every
    rank (all seeded alike by main_id_embed.py) would train on the same samples while the LR is scaled by ngpu.  Two
    gloo ranks: disjoint shards per epoch, a different order per epoch (set_epoch), identical averaged weights."""
    import torch.multiprocessing as mp
    port = 31000 + (os.getpid() % 2000)
    mp.spawn(_ddp_sampler_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    e0 = (set(r0["seen"][:4]), set(r1["seen"][:4]))
    e1 = (set(r0["seen"][4:]), set(r1["seen"][4:]))
    assert e0[0].isdisjoint(e0[1]) and e0[0] | e0[1] == set(range(8))
    assert e1[0].isdisjoint(e1[1]) and e1[0] | e1[1] == set(range(8))
    assert r0["seen"][:4] != r0["seen"][4:]                     # set_epoch reshuffles
    assert torch.equal(r0["w"], r1["w"])                        # gradients were averaged over the two ranks
