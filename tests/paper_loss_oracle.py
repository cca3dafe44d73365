"""torch restatement of the BYOL paper's loss, and the CPU oracle's training step with it (the GPU tests compare
against both).

r(x) = max(sum x^2, eps)^(-1/2) with eps = 1e-12 under the square root (the BYOL authors' l2_normalize), x^ = r(x) x,
L = mean_i |q1^_i - z2^_i|^2 + |q2^_i - z1^_i|^2, the targets constant.  F.normalize clamps the norm at 1e-12 instead;
the two agree on rows with |x| >= 1e-6.
"""
import torch

from oracle import byol_oracle as O


def l2_normalize(x, eps=1e-12):
    """x * max(sum x^2, eps)^(-1/2) per row."""
    return x * torch.rsqrt(torch.clamp(torch.sum(x * x, dim=-1, keepdim=True), min=eps))


def normalized_regression_loss(x, y):
    """Per-row |x^ - y^|^2 (= 2 - 2 cos(x, y) when neither row is clamped)."""
    return torch.sum((l2_normalize(x) - l2_normalize(y)) ** 2, dim=-1)


def paper_loss_function(online_prediction1, online_prediction2, target_projection1, target_projection2):
    """The paper's symmetric loss, mean over rows; the targets are constants."""
    loss_ab = normalized_regression_loss(online_prediction1, target_projection2.detach())
    loss_ba = normalized_regression_loss(online_prediction2, target_projection1.detach())
    return torch.mean(loss_ab + loss_ba)


LOSSES = {"reference": O.loss_function, "byol": paper_loss_function}


class OracleBYOL(O.OracleBYOL):
    """oracle.byol_oracle.OracleBYOL whose train_step takes loss="reference" | "byol".  The step itself is the pinned
    one: for the duration of the call the module's loss_function, which the step calls once per emulated rank, is the
    selected loss."""

    def train_step(self, aug1, aug2, labels, lr, world=1, sync_bn=False, loss="reference"):
        fn = LOSSES[loss]
        saved = O.loss_function
        O.loss_function = fn
        try:
            return super(OracleBYOL, self).train_step(aug1, aug2, labels, lr, world=world, sync_bn=sync_bn)
        finally:
            O.loss_function = saved
