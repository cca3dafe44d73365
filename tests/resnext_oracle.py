"""Grouped-convolution (ResNeXt) extension of the CPU oracle (oracle/byol_oracle.py), for the tests of the grouped
kernels.

The oracle restates torchvision ResNets with dense convolutions.  ResNeXt differs in one place: conv2 of every
bottleneck is a grouped 3x3 (torchvision resnet.py Bottleneck with groups > 1, width = planes * width_per_group / 64
* groups).  This module adds the ResNeXt names, the "resnext:<groups>x<width per group>:d1,d2,d3,d4" spec of shallow
test nets, and a block forward with grouped convolutions.  :func:`install` routes the oracle's module-level
dispatch through them for one test (pytest's monkeypatch restores it afterwards); every dense arch takes exactly
the oracle's own code path.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import byol_oracle as O

# name -> (stage depths, groups, width per group)
RESNEXT = {
    "resnext50_32x4d": ([3, 4, 6, 3], 32, 4),
    "resnext101_32x8d": ([3, 4, 23, 3], 32, 8),
    "resnext101_64x4d": ([3, 4, 23, 3], 64, 4),
}

_dense_arch_spec = O.arch_spec
_dense_build_reference_modules = O.build_reference_modules


def resnext_spec(arch):
    """(stage depths, groups, width per group) of a ResNeXt name or "resnext:GxW:d1,d2,d3,d4" spec, else None."""
    if arch in RESNEXT:
        return RESNEXT[arch]
    if arch.startswith("resnext:"):
        _, gw, depths = arch.split(":")
        g, w = gw.split("x")
        return [int(d) for d in depths.split(",")], int(g), int(w)
    return None


def arch_spec(arch):
    spec = resnext_spec(arch)
    return ("bottleneck", spec[0]) if spec is not None else _dense_arch_spec(arch)


def build_reference_modules(arch, representation, projection=256, head_latent=4096, num_classes=1000):
    """The oracle's module construction (same order as main.py:190-208) with a ResNeXt backbone."""
    spec = resnext_spec(arch)
    if spec is None:
        return _dense_build_reference_modules(arch, representation, projection, head_latent, num_classes)
    import torchvision
    from torchvision.models.resnet import ResNet, Bottleneck
    if arch in torchvision.models.__dict__:
        net = torchvision.models.__dict__[arch](weights=None)
    else:
        net = ResNet(Bottleneck, spec[0], groups=spec[1], width_per_group=spec[2])

    class _Container(nn.Module):
        pass

    m = _Container()
    m.base_network = nn.Sequential(*list(net.children())[:-1])
    m.head = nn.Sequential(nn.Linear(representation, head_latent), nn.BatchNorm1d(head_latent), nn.ReLU(),
                           nn.Linear(head_latent, projection))
    m.predictor = nn.Sequential(nn.Linear(projection, head_latent), nn.BatchNorm1d(head_latent), nn.ReLU(),
                                nn.Linear(head_latent, projection))
    m.linear_classifier = nn.Linear(representation, num_classes)
    return m


def block_forward(kind, P, bn, x, p, stride, train, q=O._identity):
    """oracle.block_forward where a weight with fewer input channels than its input is a grouped convolution
    (groups = Cin / weight.shape[1]); for dense weights it computes exactly what the oracle computes."""
    conv = lambda inp, name, st=1, pad=0: q(F.conv2d(inp, q(P[name]), None, st, pad, 1,
                                                     inp.shape[1] // P[name].shape[1]))
    identity = x
    if kind == "bottleneck":
        out = q(torch.relu(bn(conv(x, p + ".conv1.weight"), p + ".bn1", P, train)))
        out = q(torch.relu(bn(conv(out, p + ".conv2.weight", stride, 1), p + ".bn2", P, train)))
        out = bn(conv(out, p + ".conv3.weight"), p + ".bn3", P, train)
    else:
        out = q(torch.relu(bn(conv(x, p + ".conv1.weight", stride, 1), p + ".bn1", P, train)))
        out = bn(conv(out, p + ".conv2.weight", 1, 1), p + ".bn2", P, train)
    if (p + ".downsample.0.weight") in P:
        identity = bn(conv(x, p + ".downsample.0.weight", stride), p + ".downsample.1", P, train)
    return q(torch.relu(out + identity))


def install(monkeypatch):
    """Make oracle.byol_oracle handle ResNeXt for the duration of one test."""
    monkeypatch.setattr(O, "arch_spec", arch_spec)
    monkeypatch.setattr(O, "build_reference_modules", build_reference_modules)
    monkeypatch.setattr(O, "block_forward", block_forward)
