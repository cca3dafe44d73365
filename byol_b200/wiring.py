"""Model / optimizer wiring and the per-step hot loop, mirroring /root/reference/main.py so the CUDA path drops
into the reference's training script (see INTEGRATION.md).

* add_weight_decay                 main.py:321  (helpers.layers.add_weight_decay — source missing; behaviour
                                   inferred from optimizers/lars.py:88,99-100: bias / 1-d params -> no decay, 'ignore')
* build_optimizer                  main.py:303-344 (lr = 0.2 * global_batch / 256, SGD momentum 0.9, LARS eps=0)
* DistributedDataParallelPassthrough  main.py:440-443 — the engine averages the flat gradient itself, so the
                                   wrapper only forwards attribute access (no c10d Reducer, no graph walk)
* topk                             main.py:598  (helpers.metrics.topk)
* train_step                       main.py:579-624, the body of execute_graph for one minibatch
"""
import torch
import torch.nn as nn

from .lars import LARS  # noqa: F401 (re-exported)
from .objective import check_variant, cross_entropy_topk, loss_function


def add_weight_decay(model, weight_decay=1e-5, skip_list=()):
    decay, no_decay = [], []
    for name, param in model.named_parameters():
        if not param.requires_grad:
            continue
        if len(param.shape) == 1 or name.endswith(".bias") or name in skip_list:
            no_decay.append(param)
        else:
            decay.append(param)
    return [{'params': no_decay, 'weight_decay': 0.0, 'ignore': True},
            {'params': decay, 'weight_decay': weight_decay, 'ignore': False}]


def build_optimizer(model, base_lr=0.2, global_batch_size=4096, weight_decay=1e-6, optimizer="lars_momentum"):
    """main.py:303-344 for the 'sgd' / 'momentum' / 'lars_*' choices (schedules are per-epoch wiring, kept in main.py)."""
    name = optimizer.lower().strip()
    is_lars = 'lars' in name
    opt_name = name.split('_')[-1] if is_lars else name
    if opt_name not in ("momentum", "sgd"):
        raise NotImplementedError("optimizer %r: only sgd / momentum (optionally lars_) are wired" % optimizer)
    lr = base_lr * (global_batch_size / 256)   # Following BYOL/SimCLR (main.py:334)
    groups = add_weight_decay(model, weight_decay)
    opt = torch.optim.SGD(groups, lr=lr, momentum=0.9 if opt_name == "momentum" else 0.0)
    if is_lars:
        opt = LARS(opt, eps=0.0)
    return opt


class DistributedDataParallelPassthrough(nn.Module):
    """Stand-in for helpers.layers.DistributedDataParallelPassthrough: byol_b200.BYOL all-reduces its flat
    gradient buffer once per backward (engine.Engine._finish_backward), so no DDP machinery is needed."""

    def __init__(self, module, *args, **kwargs):
        super(DistributedDataParallelPassthrough, self).__init__()
        self.module = module

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def __getattr__(self, name):
        try:
            return super(DistributedDataParallelPassthrough, self).__getattr__(name)
        except AttributeError:
            return getattr(self.module, name)


def topk(output, target, topk=(1,)):
    """helpers.metrics.topk (main.py:598) for k in {1, 5}: percentage of rows whose label is among the k largest
    logits, from the fused kernel (rank of the label's logit = number of other logits not <= it; a NaN label logit or
    a label outside [0, classes) is a miss)."""
    from . import ops
    if any(k not in (1, 5) for k in topk):
        raise NotImplementedError("byol_b200.wiring.topk: k must be 1 or 5")
    with torch.no_grad():
        lg = output.detach()
        lg = lg if (lg.dtype == torch.float32 and lg.stride(-1) == 1) else lg.contiguous().float()
        out, _ = ops.ce_topk_fwd(lg, target.contiguous())
        return [out[1:2] if k == 1 else out[2:3] for k in topk]


def train_step(model, optimizer, augmentation1, augmentation2, labels, loss_variant="reference"):
    """One optimisation step exactly as the reference's loop body (main.py:589-624) orders it.  loss_variant selects
    the BYOL objective (objective.loss_function's variant: "reference" or the paper's "byol")."""
    check_variant(loss_variant)
    output_dict = model(augmentation1, augmentation2)
    byol_loss = loss_function(online_prediction1=output_dict['online_prediction1'],
                              online_prediction2=output_dict['online_prediction2'],
                              target_projection1=output_dict['target_projection1'],
                              target_projection2=output_dict['target_projection2'],
                              variant=loss_variant)
    # F.cross_entropy + metrics.topk on cat([labels, labels]) (main.py:591,596-598) in one kernel: row r of the
    # [2b, classes] logits uses labels[r % b], so the concatenated label vector is never materialised
    classifier_loss, acc1, acc5 = cross_entropy_topk(output_dict['linear_preds'], labels)
    loss = byol_loss + classifier_loss
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return {'loss_mean': loss.detach(), 'byol_loss_mean': byol_loss.detach(),
            'linear_loss_mean': classifier_loss.detach(), 'top1_mean': acc1, 'top5_mean': acc5}
