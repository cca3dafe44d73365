"""Host-side mirror of the reference's model API (``/root/reference/main.py:133-276``): ``CosEMA`` and ``BYOL``
with the same constructor arguments, attributes, ``state_dict`` keys and 13-key forward dict — but the compute
runs in the sm_90a kernels of ``byol_b200`` through :class:`byol_b200.engine.Engine`.

The nn.Module tree (torchvision ResNet children[:-1], head, predictor, linear_classifier) is kept only as the
*container* of parameters and buffers, so ``named_parameters()``, ``state_dict()``, ``nn.SyncBatchNorm
.convert_sync_batchnorm``, ``.cuda()`` and ``helpers.layers.add_weight_decay`` behave exactly as with the
reference; none of the torch modules' ``forward`` methods is ever called.
"""
import numpy as np
import torch
import torch.nn as nn
import torchvision.models as models

from . import ops
from .engine import Engine

BF16 = torch.bfloat16


class CosEMA(nn.Module):
    """Flat-vector EMA with cosine-annealed decay — mirrors /root/reference/main.py:133-164.

    ``mean`` is a registered buffer (checkpointed); ``step`` is a plain attribute (not checkpointed, SURVEY.md Q13).
    The update runs in place on ``mean`` with ``byol_ema_update`` (bit-exact with the reference's three fp32 ops).
    """

    def __init__(self, total_steps, base_decay=0.996):
        super(CosEMA, self).__init__()
        self.step = 0
        self.total_steps = total_steps
        self.base_decay = base_decay
        self.register_buffer('mean', None)

    def decay_at(self, step):
        # numpy float64, exactly as main.py:159
        return 1 - (1 - self.base_decay) * (np.cos(np.pi * step / self.total_steps) + 1) / 2.0

    def forward(self, x):
        if self.mean is None:
            self.mean = torch.zeros_like(x)
        if self.training:
            if not x.is_cuda:
                raise RuntimeError("byol_b200.CosEMA updates run on CUDA only (no CPU path)")
            decay = self.decay_at(self.step)
            ops.ema_update(x.detach(), self.mean, np.float32(1 - decay), np.float32(decay))
            self.step += 1
        return x


def _resnet(arch):
    if arch in models.__dict__:
        return models.__dict__[arch](weights=None)
    from torchvision.models.resnet import ResNet, Bottleneck, BasicBlock
    if arch == "resnet200":   # BASELINE.json config 5: bottleneck [3, 24, 36, 3]; not a torchvision constructor
        return ResNet(Bottleneck, [3, 24, 36, 3])
    if arch.startswith("resnet:"):   # custom depth: "resnet:<basic|bottleneck>:d1,d2,d3,d4"
        _, kind, depths = arch.split(":")
        return ResNet(Bottleneck if kind == "bottleneck" else BasicBlock, [int(d) for d in depths.split(",")])
    raise ValueError("unknown arch %r" % arch)


class _OnlineTargetFn(torch.autograd.Function):
    """All four encoder passes of one step (main.py:244-247) as ONE autograd node.

    Outputs 0-5: online (representation, projection, prediction) for view 1 and 2 — differentiable;
    outputs 6-11: the same for the target network — non-differentiable (the loss detaches them anyway,
    objective.py:23-24)."""

    @staticmethod
    def forward(ctx, model, aug1, aug2, anchor):
        eng = model._engine
        saved = [{}, {}]
        lanes = [(eng.theta, eng.w_online, saved[0]), (eng.theta, eng.w_online, saved[1]),
                 (model.target_network.mean, eng.w_target, None), (model.target_network.mean, eng.w_target, None)]
        outs, reps_b = eng.forward_lanes([aug1, aug2, aug1, aug2], lanes, True,
                                         rep_bf16_out=[model._rep_cat[:aug1.shape[0]], model._rep_cat[aug1.shape[0]:],
                                                       None, None])
        ctx.model = model
        ctx.saved = saved
        ctx.set_materialize_grads(False)
        flat = [t for o in outs for t in o]
        ctx.mark_non_differentiable(*flat[6:])
        return tuple(flat)

    @staticmethod
    def backward(ctx, *grads):
        eng = ctx.model._engine
        saved, ctx.saved = ctx.saved, None
        eng.backward_online(saved, [grads[0], grads[3]], [grads[1], grads[4]], [grads[2], grads[5]])
        return None, None, None, None


class _GraphedOnlineTargetFn(torch.autograd.Function):
    """Same node as _OnlineTargetFn, but both passes are CUDA-graph replays over fixed buffers
    (engine.Engine.graphed_step).  The returned tensors alias step-persistent buffers: they are valid until the next
    training forward (the reference's loop consumes them immediately, main.py:589-617)."""

    @staticmethod
    def forward(ctx, model, gs, anchor):
        from ._lib import launch_count
        gs.fwd.replay()
        gs.pending = True
        launch_count[0] += gs.fwd_launches
        ctx.model, ctx.gs = model, gs
        ctx.set_materialize_grads(False)
        flat = [t.detach() for t in gs.outs]
        ctx.mark_non_differentiable(*flat[6:])
        return tuple(flat)

    @staticmethod
    def backward(ctx, *grads):
        from ._lib import launch_count
        eng, gs = ctx.model._engine, ctx.gs
        gs.pending = False
        d_reps, d_projs, d_preds = [grads[0], grads[3]], [grads[1], grads[4]], [grads[2], grads[5]]
        if all(g is None for g in d_reps + d_projs) and all(g is not None for g in d_preds):
            eng.notify_backward()
            gs.d_pred[0].copy_(d_preds[0])
            gs.d_pred[1].copy_(d_preds[1])
            gs.bwd.replay()
            launch_count[0] += gs.bwd_launches
        else:
            # unusual gradient pattern (e.g. a loss on the projections): eager kernels over the same saved buffers
            eng.backward_online(gs.saved, d_reps, d_projs, d_preds)
        return None, None, None


class _ClassifierFn(torch.autograd.Function):
    """Stop-gradient linear classifier (main.py:250-252): logits are differentiable w.r.t. its own weights only."""

    @staticmethod
    def forward(ctx, model, rep_cat_b, anchor, logits=None, reps_f32=None):
        ctx.model = model
        ctx.rep = rep_cat_b
        return model._engine.classifier_forward(rep_cat_b, reps_f32) if logits is None else logits.detach()

    @staticmethod
    def backward(ctx, d_logits):
        ctx.model._engine.classifier_backward(ctx.rep, d_logits)
        return None, None, None, None, None


class BYOL(nn.Module):
    """Drop-in for ``main.BYOL`` (/root/reference/main.py:167-276).

    The reference reads ``args.arch`` / ``args.head_latent_size`` from a module global (main.py:190,195); here they
    are keyword arguments with the reference's defaults (main.py:57,63)."""

    def __init__(self, base_network_output_size, projection_output_size, classifier_output_size,
                 total_training_steps, base_decay=0.996, arch="resnet50", head_latent_size=4096, precision="bf16"):
        super(BYOL, self).__init__()
        self.base_network_output_size = base_network_output_size
        self.arch = arch
        # identical construction order to main.py:190-208 => identical parameter order and default initialisation
        self.base_network = nn.Sequential(*list(_resnet(arch).children())[:-1])
        self.head = nn.Sequential(
            nn.Linear(base_network_output_size, head_latent_size),
            nn.BatchNorm1d(head_latent_size),
            nn.ReLU(),
            nn.Linear(head_latent_size, projection_output_size),
        )
        self.predictor = nn.Sequential(
            nn.Linear(projection_output_size, head_latent_size),
            nn.BatchNorm1d(head_latent_size),
            nn.ReLU(),
            nn.Linear(head_latent_size, projection_output_size),
        )
        self.linear_classifier = nn.Linear(base_network_output_size, classifier_output_size)
        self.target_network = CosEMA(total_training_steps, base_decay)
        # main.py:211-212 runs the EMA once at construction, on the host: mean = (1 - d0) * theta0 + d0 * 0 with
        # d0 = decay(step 0) = base_decay, and step -> 1 (SURVEY.md Q4).  Same here (host tensors, fp32), so that
        # checkpoint restores and params-only loads see exactly the reference's state.
        with torch.no_grad():
            theta0 = torch.cat([p.detach().reshape(-1) for p in self.parameters()])
            d0 = self.target_network.decay_at(0)
            self.target_network.mean = (1 - d0) * theta0 + d0 * torch.zeros_like(theta0)
        self.target_network.step = 1
        self._engine = Engine(self)
        # forward arithmetic: "bf16" = bf16 tensor-core operands (fast path); "fp32" = the reference's fp32 results
        # from exact 3-way bf16 splits of every operand (6 product terms, fp64 statistics; BASELINE configs[1]);
        # "bf16x2" = 2-way splits (3 terms, ~16 mantissa bits).  The backward pass always uses bf16 operands.
        if precision not in ("bf16", "bf16x2", "fp32"):
            raise ValueError("precision must be 'bf16', 'bf16x2' or 'fp32', got %r" % (precision,))
        self.precision = precision
        self._engine.T = {"bf16": 0, "bf16x2": 3, "fp32": 6}[precision]
        self._anchor = None
        self._rep_cat = None

    # ---- keep the engine in sync with module surgery (.cuda(), convert_sync_batchnorm, ...) ----
    def _apply(self, fn, *args, **kwargs):
        out = super(BYOL, self)._apply(fn, *args, **kwargs)
        self._engine.ready = False
        return out

    def _ensure_ready(self, batch):
        eng = self._engine
        if not eng.plan_is_current():
            eng.flatten()
            eng.build_plan()
        if self._anchor is None or self._anchor.device != eng.device:
            self._anchor = torch.zeros(1, device=eng.device, requires_grad=True)
        if self._rep_cat is None or self._rep_cat.shape[0] != 2 * batch or self._rep_cat.device != eng.device:
            self._rep_cat = torch.empty((2 * batch, eng.rep_dim), dtype=BF16, device=eng.device)
        return eng

    def parameters_vector(self):
        """The flat fp32 vector of all parameters in registration order (what the reference builds with
        nn.utils.parameters_to_vector at main.py:212,223,255) — here a persistent buffer, not a copy."""
        return self._ensure_ready(1).theta if self._rep_cat is None else self._engine.theta

    def forward(self, augmentation1, augmentation2):
        """Returns the online and target network representations, projections and predictions (main.py:242-276)."""
        if not augmentation1.is_cuda:
            raise RuntimeError("byol_b200.BYOL.forward needs CUDA tensors (no CPU path)")
        b = augmentation1.shape[0]
        eng = self._ensure_ready(b)
        a1 = augmentation1.contiguous().float()
        a2 = augmentation2.contiguous().float()
        gs = eng.graphed_step(self, a1, a2) if (self.training and torch.is_grad_enabled()) else None
        if gs is not None and gs.mean_ptr != self.target_network.mean.data_ptr():
            eng.graphs = {}          # the EMA buffer was replaced (e.g. load_state_dict with assign): re-capture later
            gs = None
        if gs is not None and gs.pending:
            gs = None                # a graphed forward still awaits its backward: its fixed buffers must survive
        if gs is not None:
            # the whole forward (weight layouts, 4 lanes, classifier) is one graph launch over fixed buffers
            eng.convert_inputs([a1], outs=gs.inputs[0:1])
            eng.convert_inputs([a2], outs=gs.inputs[1:2])
            o = _GraphedOnlineTargetFn.apply(self, gs, self._anchor)
            linear_preds = _ClassifierFn.apply(self, self._rep_cat, self._anchor, gs.logits)
        else:
            eng.prep_step(self.target_network.mean, self.training)
        if gs is not None:
            pass
        elif self.training and torch.is_grad_enabled():
            o = _OnlineTargetFn.apply(self, a1, a2, self._anchor)
            rep_cat = self._rep_cat
            linear_preds = _ClassifierFn.apply(self, rep_cat, self._anchor, None, (o[0].detach(), o[3].detach()))
        else:
            lanes = [(eng.theta, eng.w_online, None), (eng.theta, eng.w_online, None),
                     (self.target_network.mean, eng.w_target, None), (self.target_network.mean, eng.w_target, None)]
            outs, reps_b = eng.forward_lanes([a1, a2, a1, a2], lanes, self.training,
                                             rep_bf16_out=[self._rep_cat[:b], self._rep_cat[b:], None, None])
            o = [t for oo in outs for t in oo]
            rep_cat = self._rep_cat if self.training else self._rep_cat[:b]   # eval: view 1 only (main.py:250-251)
            linear_preds = eng.classifier_forward(rep_cat, [o[0], o[3]] if self.training else [o[0]])

        # Update the EMA parameters with the pre-update online weights (main.py:254-255)
        self.target_network(eng.theta)

        return {
            'linear_preds': linear_preds,
            'online_representation1': o[0], 'online_projection1': o[1], 'online_prediction1': o[2],
            'online_representation2': o[3], 'online_projection2': o[4], 'online_prediction2': o[5],
            'target_representation1': o[6], 'target_projection1': o[7], 'target_prediction1': o[8],
            'target_representation2': o[9], 'target_projection2': o[10], 'target_prediction2': o[11],
        }
