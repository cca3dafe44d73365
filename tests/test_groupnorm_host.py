"""CPU: BYOL(norm="group_ws") construction.  Same parameters, initial values and weight-decay groups as the BatchNorm
model, GroupNorm(32) layers, every encoder conv a WSConv2d, the heads unchanged, the option errors, and WSConv2d's
weight standardisation against a float64 numpy restatement."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from byol_b200.model import BYOL, WSConv2d


def _pair(arch, draws=None, **kw):
    models = []
    for norm in ("batch", "group_ws"):
        torch.manual_seed(3)
        models.append(BYOL(512 if arch == "resnet18" else 2048, 64, 10, 10, arch=arch, head_latent_size=128,
                           norm=norm, **kw))
        if draws is not None:
            draws.append(torch.rand(8))
    return models


ARCHS = ["resnet18", "resnet50", "resnext:32x4:1,1,1,1"]


@pytest.mark.parametrize("arch", ARCHS)
def test_theta0_and_parameters_equal_the_batchnorm_model(arch):
    draws = []
    bn, gn = _pair(arch, draws)
    assert torch.equal(draws[0], draws[1])           # construction consumed the same random numbers
    assert [(k, tuple(p.shape)) for k, p in bn.named_parameters()] == \
        [(k, tuple(p.shape)) for k, p in gn.named_parameters()]
    t_bn = torch.nn.utils.parameters_to_vector(bn.parameters())
    t_gn = torch.nn.utils.parameters_to_vector(gn.parameters())
    assert torch.equal(t_bn, t_gn)
    assert torch.equal(bn.target_network.mean, gn.target_network.mean)
    assert gn.norm == "group_ws" and bn.norm == "batch"


@pytest.mark.parametrize("arch", ARCHS)
def test_modules(arch):
    _, gn = _pair(arch)
    enc = list(gn.base_network.modules())
    convs = [m for m in enc if isinstance(m, nn.Conv2d)]
    assert convs and all(type(m) is WSConv2d for m in convs)
    norms = [m for m in enc if isinstance(m, (nn.GroupNorm, nn.modules.batchnorm._BatchNorm))]
    assert norms and all(type(m) is nn.GroupNorm and m.num_groups == 32 and m.affine for m in norms)
    for seq in (gn.head, gn.predictor):
        assert type(seq[1]) is nn.BatchNorm1d


def test_state_dict_keys():
    bn, gn = _pair("resnet50")
    buffers = ("running_mean", "running_var", "num_batches_tracked")
    k_bn, k_gn = list(bn.state_dict().keys()), list(gn.state_dict().keys())
    enc = [k for k in k_bn if not (k.startswith("base_network.") and k.rsplit(".", 1)[1] in buffers)]
    assert k_gn == enc
    assert len(k_bn) - len(k_gn) == 3 * 53


def test_weight_decay_groups():
    from byol_b200.wiring import add_weight_decay
    bn, gn = _pair("resnet18")
    g_bn, g_gn = add_weight_decay(bn, 1e-6), add_weight_decay(gn, 1e-6)
    assert len(g_bn) == len(g_gn)
    names = {id(p): k for k, p in gn.named_parameters()}
    names_bn = {id(p): k for k, p in bn.named_parameters()}
    for a, b in zip(g_bn, g_gn):
        assert {k: v for k, v in a.items() if k != "params"} == {k: v for k, v in b.items() if k != "params"}
        assert [names_bn[id(p)] for p in a["params"]] == [names[id(p)] for p in b["params"]]
    # GroupNorm's affine parameters sit where BatchNorm's do: in the group without weight decay
    no_decay = [g for g in g_gn if g.get("weight_decay", 1) == 0]
    assert no_decay
    gn_params = {id(p) for m in gn.base_network.modules() if isinstance(m, nn.GroupNorm) for p in m.parameters()}
    assert gn_params <= {id(p) for g in no_decay for p in g["params"]}


def test_option_errors():
    with pytest.raises(ValueError, match="norm"):
        BYOL(512, 64, 10, 10, arch="resnet18", norm="layer")
    for precision in ("fp32", "bf16x2"):
        with pytest.raises(ValueError, match="group_ws"):
            BYOL(512, 64, 10, 10, arch="resnet18", norm="group_ws", precision=precision)
    with pytest.raises(ValueError, match="group_ws"):
        BYOL(512, 64, 10, 10, arch="resnet18", norm="group_ws", precision="fp32", backward_precision="fp32")
    # 2 groups x 8 channels: the ResNeXt width 16 is not divisible by 32
    with pytest.raises(ValueError, match=r"layer base_network\.4\.0\.bn1 has 16 channels"):
        BYOL(2048, 64, 10, 10, arch="resnext:2x8:1,1,1,1", norm="group_ws")


def test_wsconv2d_against_float64():
    rng = np.random.default_rng(0)
    for cin, cout, k, groups in [(3, 64, 7, 1), (64, 256, 1, 1), (64, 64, 3, 1), (128, 128, 3, 32)]:
        torch.manual_seed(1)
        m = WSConv2d(cin, cout, k, padding=k // 2, groups=groups, bias=False)
        w = m.weight.detach().double().numpy().reshape(cout, -1)
        mean = w.mean(1, keepdims=True)
        var = ((w - mean) ** 2).mean(1, keepdims=True)
        wh = (w - mean) / np.sqrt(var + 1e-5)
        got = m.standardized_weight().detach().double().numpy().reshape(cout, -1)
        assert np.abs(got - wh).max() <= 1e-5 * np.abs(wh).max()
        x = torch.from_numpy(rng.standard_normal((2, cin, 9, 9)))
        ref = F.conv2d(x, torch.from_numpy(wh).view(m.weight.shape), None, 1, k // 2, 1, groups)
        out = m.double()(x).detach()
        assert float((out - ref).abs().max()) <= 1e-10 * float(ref.abs().max())
