"""CPU: grouped 3x3 convolutions (ResNeXt) — the oracle against the reference's ResNeXt-50 golden run, the algebra
of the block-diagonal tile layouts the CUDA kernels use, and which networks BYOL accepts."""
import pytest
import torch
import torch.nn.functional as F

from tests import resnext_oracle
from tests.test_oracle_golden import test_oracle_matches_reference_golden as oracle_matches_golden


def test_oracle_matches_resnext50_golden(monkeypatch):
    """The oracle with grouped convolutions (tests/resnext_oracle.py) against the reference's ResNeXt-50 run: losses,
    outputs, gradients, EMA and bookkeeping of two steps, at test_oracle_golden's tolerances."""
    resnext_oracle.install(monkeypatch)
    oracle_matches_golden("rnx50_b8_r64")


# ---- tile layouts (mirrors byol_prep_weights_grouped and the kernels' K loops, in float64) ------------------------
def _same_group(c, cg):
    """[C, 64] mask: row r and its tile partner (r & ~63) + j lie in one group."""
    r = torch.arange(c).view(-1, 1)
    partner = (r // 64) * 64 + torch.arange(64).view(1, -1)
    return partner, (r // cg) == (partner // cg)


def _fprop_tiles(w):
    """w [C, Cg, 3, 3] -> [C, 9, 64]: row co, column (tap, ci - n0) = w[co, ci % Cg, tap] within the group, else 0."""
    c, cg = w.shape[:2]
    partner, same = _same_group(c, cg)
    vals = w.reshape(c, cg, 9)[torch.arange(c).view(-1, 1), partner % cg]        # [C, 64, 9]
    return (vals * same.unsqueeze(-1)).permute(0, 2, 1)


def _dgrad_tiles(w):
    """w [C, Cg, 3, 3] -> [C, 9, 64]: row ci, column (tap, co - n0) = w[co, ci % Cg, tap] within the group, else 0."""
    c, cg = w.shape[:2]
    partner, same = _same_group(c, cg)
    vals = w.reshape(c, cg, 9)[partner, (torch.arange(c) % cg).view(-1, 1)]      # [C, 64, 9]: co = partner
    return (vals * same.unsqueeze(-1)).permute(0, 2, 1)


@pytest.mark.parametrize("cg", [4, 8, 16, 32, 64])
@pytest.mark.parametrize("stride", [1, 2])
def test_tile_layouts_equal_grouped_conv(cg, stride):
    c, n, h = 128, 2, 10
    g = torch.Generator().manual_seed(cg * 10 + stride)
    x = torch.randn(n, c, h, h, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(c, cg, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(x, w, None, stride, 1, 1, c // cg)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    wf, wd = _fprop_tiles(w.detach()), _dgrad_tiles(w.detach())
    cols = F.unfold(x.detach(), 3, padding=1, stride=stride)                    # [N, C*9, L], row = ci*9 + tap
    ho = y.shape[-1]
    y_t, dx_t, dw_t = torch.zeros_like(y), torch.zeros_like(x), torch.zeros(c, 64, 3, 3, dtype=torch.float64)
    for n0 in range(0, c, 64):
        t = slice(n0, n0 + 64)
        # fprop: the tile is a dense GEMM over its own 64 channels x 9 taps
        a = cols.view(n, c, 9, -1)[:, t].permute(0, 3, 2, 1).reshape(n, -1, 9 * 64)   # [N, L, tap*64 + ci]
        y_t[:, t] = (a @ wf[t].reshape(64, 9 * 64).t()).permute(0, 2, 1).reshape(n, 64, ho, ho)
        # dgrad: the transposed conv of the tile's dense weight wt[co, ci, tap] = wd[ci, tap, co]
        wt = wd[t].permute(2, 0, 1).reshape(64, 64, 3, 3)
        dx_t[:, t] = F.conv_transpose2d(dy[:, t], wt, None, stride, 1, output_padding=h - (ho - 1) * stride - 1)
        # wgrad: the tile's dense weight gradient, of which only the in-group entries are kept
        dw_t[t] = torch.nn.grad.conv2d_weight(x.detach()[:, t], (64, 64, 3, 3), dy[:, t], stride, 1)
    partner, same = _same_group(c, cg)
    dw_keep = torch.zeros_like(w)
    rows = torch.arange(c).view(-1, 1).expand(c, 64)
    dw_keep[rows[same], (partner % cg)[same]] = dw_t.view(c, 64, 3, 3)[same]
    torch.testing.assert_close(y_t, y.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dx_t, x.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dw_keep, w.grad, rtol=1e-12, atol=1e-12)


# ---- construction ---------------------------------------------------------------------------------------------------
FAMILY = ["resnet18", "resnet34", "resnet50", "resnet101", "resnet152", "wide_resnet50_2", "wide_resnet101_2",
          "resnext50_32x4d", "resnext101_32x8d", "resnext101_64x4d"]


@pytest.mark.parametrize("arch", FAMILY)
def test_every_torchvision_resnet_builds(arch):
    from byol_b200.model import BYOL
    rep = 512 if arch in ("resnet18", "resnet34") else 2048
    model = BYOL(rep, 256, 1000, 10, arch=arch)
    groups = {m.groups for m in model.base_network.modules() if isinstance(m, torch.nn.Conv2d)}
    assert (max(groups) > 1) == arch.startswith("resnext")


def test_resnext_spec(monkeypatch):
    from byol_b200.model import BYOL
    from oracle import byol_oracle as O
    resnext_oracle.install(monkeypatch)
    model = BYOL(2048, 256, 1000, 10, arch="resnext:32x8:1,1,1,1")
    conv2 = [m for n, m in model.base_network.named_modules() if n.endswith("conv2")]
    assert [(m.in_channels, m.groups) for m in conv2] == [(256, 32), (512, 32), (1024, 32), (2048, 32)]
    assert O.arch_spec("resnext:32x8:1,1,1,1") == ("bottleneck", [1, 1, 1, 1])
    params, _ = O.init_reference_state("resnext:32x8:1,1,1,1", 0)
    assert [tuple(p.shape) for k, p in model.named_parameters()] == [tuple(p.shape) for p in params.values()]


@pytest.mark.parametrize("arch,precision,match", [
    ("resnext:2x64:1,1,1,1", "bf16", "base_network.5.0.conv2"),      # stage 2: 128 channels per group
    ("resnext50_32x4d", "fp32", "precision"),
    ("resnext50_32x4d", "bf16x2", "precision"),
])
def test_unsupported_grouped_nets_are_rejected(arch, precision, match):
    from byol_b200.model import BYOL
    with pytest.raises(ValueError, match=match):
        BYOL(2048, 256, 1000, 10, arch=arch, precision=precision)


def test_grouped_conv_shapes_are_checked():
    import torch.nn as nn
    from byol_b200.model import check_grouped_convs
    ok = nn.Sequential(nn.Conv2d(128, 128, 3, 2, 1, groups=32, bias=False))
    check_grouped_convs(ok, "bf16")
    for bad in (nn.Conv2d(128, 256, 3, 1, 1, groups=32, bias=False),     # Cin != Cout
                nn.Conv2d(96, 96, 3, 1, 1, groups=32, bias=False),       # C % 64
                nn.Conv2d(128, 128, 5, 1, 2, groups=32, bias=False),     # 5x5
                nn.Conv2d(128, 128, 3, 1, 0, groups=32, bias=False),     # pad 0
                nn.Conv2d(128, 128, 3, 3, 1, groups=32, bias=False),     # stride 3
                nn.Conv2d(384, 384, 3, 1, 1, groups=4, bias=False)):     # 96 channels per group
        with pytest.raises(ValueError, match="grouped conv 0"):
            check_grouped_convs(nn.Sequential(bad), "bf16")
