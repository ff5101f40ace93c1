"""Host mirror of ldm/models/autoencoder.py:285-333 (AutoencoderKL): encode -> DiagonalGaussianDistribution,
decode -> image; parameters keep the reference names (first_stage_model.* keys of SD-v1 checkpoints)."""
import torch
from torch import nn

from celebbasis_b200.vae_engine import VAEDecoderEngine, VAEEncoderEngine
from ldm.modules.diffusionmodules.model import Decoder, Encoder
from ldm.modules.distributions.distributions import DiagonalGaussianDistribution


def _plain(cfg):
    return {k: (list(v) if not isinstance(v, (int, float, bool, str, type(None))) else v) for k, v in dict(cfg).items()}


def _reset_engines(module, incompatible_keys):
    """load_state_dict post-hook: packed device weights are rebuilt lazily after a checkpoint load."""
    for name in ("_engine", "_face_engine", "_enc", "_dec"):
        if hasattr(module, name):
            setattr(module, name, None)


class AutoencoderKL(nn.Module):
    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=[], image_key="image",
                 colorize_nlabels=None, monitor=None):
        super().__init__()
        dd = _plain(ddconfig)
        self.ddconfig = dd
        self.image_key = image_key
        self.encoder = Encoder(**dd)
        self.decoder = Decoder(**dd)
        self.loss = nn.Identity()
        assert dd["double_z"]
        self.quant_conv = nn.Conv2d(2 * dd["z_channels"], 2 * embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, dd["z_channels"], 1)
        self.embed_dim = embed_dim
        if monitor is not None:
            self.monitor = monitor
        self._enc = self._dec = None
        self.register_load_state_dict_post_hook(_reset_engines)
        if ckpt_path is not None:
            sd = torch.load(ckpt_path, map_location="cpu")["state_dict"]
            self.load_state_dict({k: v for k, v in sd.items() if not any(k.startswith(i) for i in ignore_keys)},
                                 strict=False)

    def _dev(self):
        dev = self.quant_conv.weight.device
        if dev.type != "cuda":
            raise RuntimeError("celebbasis_b200 AutoencoderKL runs on sm_90a only (no CPU fallback)")
        return dev

    def encode(self, x):
        dev = self._dev()
        if self._enc is None or self._enc.dev != dev:
            self._enc = VAEEncoderEngine(self.ddconfig, self.embed_dim, self.state_dict(), dev)
        return DiagonalGaussianDistribution(self._enc.encode_moments(x.to(dev)))

    def decode(self, z):
        dev = self._dev()
        if self._dec is None or self._dec.dev != dev:
            self._dec = VAEDecoderEngine(self.ddconfig, self.embed_dim, self.state_dict(), dev)
        return self._dec.decode(z.to(dev))

    def forward(self, input, sample_posterior=True):
        posterior = self.encode(input)
        z = posterior.sample() if sample_posterior else posterior.mode()
        return self.decode(z), posterior
