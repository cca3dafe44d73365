"""BYOL objective — drop-in for /root/reference/objective.py (same function names and call signature).

``loss_function`` keeps the reference's semantics exactly (SURVEY.md Q1/Q2): the "normalisation" is by the
Frobenius norm of the WHOLE [batch, dim] matrices (``x.norm()`` without ``dim``), it is rank-local under data
parallelism (no collective), targets are constants, and the result is ``mean_i(loss_ab_i + loss_ba_i)`` — one
reduction kernel forward and one elementwise kernel backward instead of ~34 ATen launches.  That is the default.

``loss_function(..., variant="byol")`` is the BYOL paper's loss instead: each row of the predictions q and targets z
is L2-normalised on its own, x^ = x / sqrt(max(sum x^2, 1e-12)), and the loss is the mean over rows of
|q1^ - z2^|^2 + |q2^ - z1^|^2 (in [0, 8]; 4 - 2 cos - 2 cos when no row is clamped).  It is per sample, so under data
parallelism each rank's mean followed by the engine's gradient average is the gradient of the global batch's loss,
whatever the world size.  Two launches forward (one warp per sample, then an ordered fp64 sum) and one backward.
"""
import torch

from . import ops


class _ByolLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q1, q2, z1, z2):
        q1, q2 = q1.contiguous().float(), q2.contiguous().float()
        z1, z2 = z1.detach().contiguous().float(), z2.detach().contiguous().float()
        dev = q1.device
        ws = torch.empty(6, dtype=torch.float64, device=dev)
        out = torch.empty(7, dtype=torch.float32, device=dev)   # [loss, 6 saved scalars]
        ops.loss_fwd(q1, q2, z1, z2, ws, out[0:1], out[1:7])
        ctx.save_for_backward(q1, q2, z1, z2, out)
        return out[0].clone().view(())

    @staticmethod
    def backward(ctx, grad_out):
        q1, q2, z1, z2, out = ctx.saved_tensors
        dq1, dq2 = torch.empty_like(q1), torch.empty_like(q2)
        go = grad_out.contiguous().float().view(1)
        ops.loss_bwd(q1, q2, z1, z2, out[1:7], go, dq1, dq2)
        return dq1, dq2, None, None


def _rows(t):
    """fp32, contiguous and 16-byte aligned (the kernels load float4s)."""
    t = t.contiguous().float()
    return t if t.data_ptr() % 16 == 0 else t.clone()


class _PaperLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q1, q2, z1, z2):
        q1, q2, z1, z2 = _rows(q1), _rows(q2), _rows(z1.detach()), _rows(z2.detach())
        loss = torch.empty((), dtype=torch.float32, device=q1.device)
        saved = torch.empty(q1.shape[0], 8, dtype=torch.float32, device=q1.device)
        ops.loss_rows_fwd(q1, q2, z1, z2, loss.view(1), saved)
        ctx.save_for_backward(q1, q2, z1, z2, saved)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        q1, q2, z1, z2, saved = ctx.saved_tensors
        dq1, dq2 = torch.empty_like(q1), torch.empty_like(q2)
        ops.loss_rows_bwd(q1, q2, z1, z2, saved, grad_out.contiguous().float().view(1), dq1, dq2)
        return dq1, dq2, None, None


LOSS_VARIANTS = ("reference", "byol")


def check_variant(variant):
    if variant not in LOSS_VARIANTS:
        raise ValueError("loss_function: variant must be one of %s, got %r" % (LOSS_VARIANTS, variant))


def regression_loss(x, y):
    """Per-row loss of objective.py:6-9 (kept for API completeness; `loss_function` is the fused hot path)."""
    norm_x, norm_y = x.norm(), y.norm()
    return -2 * torch.sum(x * y, dim=-1) / (norm_x * norm_y)


def loss_function(online_prediction1, online_prediction2, target_projection1, target_projection2,
                  variant="reference"):
    """BYOL loss.  variant="reference" (default, objective.py:12-25): regression_loss(q1, sg(z2)) +
    regression_loss(q2, sg(z1)), mean over rows, with whole-matrix norms.  variant="byol": the paper's per-row
    normalised loss (module docstring); the targets are constants in both."""
    check_variant(variant)
    if not online_prediction1.is_cuda:
        raise RuntimeError("byol_b200.objective.loss_function needs CUDA tensors (no CPU path)")
    fn = _PaperLossFn if variant == "byol" else _ByolLossFn
    return fn.apply(online_prediction1, online_prediction2, target_projection1, target_projection2)


class _CrossEntropyTopkFn(torch.autograd.Function):
    """Softmax cross-entropy + top-1 / top-5 accuracy of the linear probe in ONE launch
    (/root/reference/main.py:596-598: F.cross_entropy(linear_preds, labels) and helpers.metrics.topk)."""

    @staticmethod
    def forward(ctx, logits, labels):
        lg = logits if (logits.dtype == torch.float32 and logits.stride(-1) == 1) else logits.contiguous().float()
        lab = labels.contiguous()
        out, row_lse = ops.ce_topk_fwd(lg, lab)
        ctx.save_for_backward(lg, lab, row_lse)
        ctx.mark_non_differentiable(out[1:2], out[2:3])
        return out[0].clone().view(()), out[1:2], out[2:3]

    @staticmethod
    def backward(ctx, grad_loss, _g1, _g5):
        lg, lab, row_lse = ctx.saved_tensors
        go = grad_loss.contiguous().float().view(1)
        return ops.ce_bwd(lg, lab, row_lse, go), None


def cross_entropy_topk(logits, labels):
    """(mean cross-entropy loss [differentiable w.r.t. logits], top-1 %, top-5 %) — the reference computes these with
    F.cross_entropy + metrics.topk(output, target, topk=(1, 5)) (main.py:596-598); accuracies are 1-element
    tensors like the reference's."""
    if not logits.is_cuda:
        raise RuntimeError("byol_b200.objective.cross_entropy_topk needs CUDA tensors (no CPU path)")
    return _CrossEntropyTopkFn.apply(logits, labels)
