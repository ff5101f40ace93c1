"""Deterministic synthetic checkpoints (there is no network for SD-v1 / CLIP / CosFace weights).

Every tensor is drawn from a CPU generator seeded by (seed, sha1(key)), so a checkpoint is a pure function
of its key names and shapes: the reference modules, the oracle restatement and the H100 engines all see
bit-identical fp32 weights without shipping gigabytes.  Rules (SURVEY.md §8c "synthetic-weight rules"):
variance-preserving fan-in init for every matrix/conv (including the reference's zero-initialised
modules, which would otherwise make every output and gradient exactly 0, and iresnet convs, whose own
N(0,0.1) init overflows), norm scales ~ 1, small biases, benign BatchNorm running statistics.
"""
import hashlib

import torch


def _gen(seed, key):
    h = int.from_bytes(hashlib.sha1(key.encode()).digest()[:6], "little")
    g = torch.Generator(device="cpu")
    g.manual_seed((int(seed) * 1000003 + h) % (2 ** 62))
    return g


def synth_tensor(key, shape, seed=0, dtype=torch.float32):
    shape = tuple(shape)
    g = _gen(seed, key)
    leaf = key.rsplit(".", 1)[-1]
    if leaf == "num_batches_tracked":
        return torch.zeros(shape, dtype=torch.int64)
    if leaf == "running_mean":
        return (0.05 * torch.randn(shape, generator=g)).to(dtype)
    if leaf == "running_var":
        return (1.0 + 0.1 * torch.randn(shape, generator=g).abs()).to(dtype)
    if leaf == "weight" and len(shape) >= 2:
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        if "stylegan_mlp" in key:            # EqualLinear: reference init is N(0,1) (meta_net.py:30)
            std = 1.0
        else:
            std = fan_in ** -0.5
        return (std * torch.randn(shape, generator=g)).to(dtype)
    if leaf == "weight":                      # norm scales, PReLU slopes
        if "prelu" in key:
            return (0.25 + 0.02 * torch.randn(shape, generator=g)).to(dtype)
        return (1.0 + 0.1 * torch.randn(shape, generator=g)).to(dtype)
    if leaf == "bias":
        return (0.05 * torch.randn(shape, generator=g)).to(dtype)
    return None


def synth_state_dict(module, seed=0, prefix=""):
    """A synthetic state dict for every floating parameter / BN buffer of `module` (keys as in module.state_dict())."""
    out = {}
    for k, v in module.state_dict().items():
        t = synth_tensor(prefix + k, v.shape, seed, v.dtype if v.dtype.is_floating_point else torch.float32)
        if t is not None and (v.dtype.is_floating_point or k.endswith("num_batches_tracked")):
            out[k] = t
    return out


def synth_celeb_basis(es=2, k=512, d=768, seed=0):
    """(es, 1+k, d): row 0 = mean embedding, rows 1.. = orthonormal PCA directions (as modules.py:594-600 builds)."""
    g = _gen(seed, "celeb_basis")
    mean = 0.03 * torch.randn(es, 1, d, generator=g)
    raw = torch.randn(es, d, k, generator=g)
    q, _ = torch.linalg.qr(raw)               # (es, d, k) orthonormal columns
    return torch.cat([mean, q.transpose(1, 2).contiguous()], dim=1)
