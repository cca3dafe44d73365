"""Step engine: walks the (torchvision-shaped) module tree of :class:`byol_b200.model.BYOL`, keeps every
parameter / gradient in flat fp32 buffers, and runs the BYOL forward and backward as explicit sequences of the
sm_90a kernels in ``ops`` — no autograd graph, no ATen compute on the hot path.

Reference semantics reproduced (file:line are /root/reference):

* main.py:229-240  prediction(): encoder -> view(-1, C) -> head -> predictor
* main.py:242-247  four passes per step in the order online(v1), online(v2), target(v1), target(v2); here they
                   run layer by layer in lock-step ("lanes") so BN running statistics see the same update order
                   per layer (SURVEY.md Q7) while weights stay hot in L2 and, under SyncBatchNorm, ONE
                   all-reduce per layer carries the statistics of all lanes
* main.py:214-227  target passes evaluate the same graph at the EMA weights (flat `target_network.mean`); no
                   activations are kept for them
* main.py:433      SyncBatchNorm: cross-rank sum of (sum, sum of squares) [fwd] and (sum dz, sum dz*xhat) [bwd]
* main.py:440,617  DDP: gradients are averaged over ranks once per backward (one flat all-reduce)

Data layout: activations NHWC bf16; conv outputs are stored raw ("y") and normalised copies ("a") are
materialised by a fused BN-apply(+residual)+ReLU kernel; BN statistics come from the conv epilogue.
"""
import collections
import gc
import os

import torch
import torch.nn as nn

from . import comm, ops

BF16 = torch.bfloat16
F32 = torch.float32

# GroupNorm "coefficients" of one lane: the layer's gamma / beta (views of the lane's parameter vector) and the conv
# output's per-(image, group) fp32 (mean, rstd) [N, 32, 2].  BatchNorm layers carry a [4, C] tensor instead.
_GN = collections.namedtuple("_GN", "gamma beta stats")


class _Unit(object):
    """One conv/linear (+ optional BN) layer: static geometry plus offsets into the flat parameter vector."""
    __slots__ = ("idx", "kind", "cin", "cout", "cpad", "k", "stride", "pad", "w_off", "w_numel", "b_off", "bn",
                 "g_off", "beta_off", "name", "want_dgrad", "fold", "kcols", "groups", "gn", "ws", "ws_off")


class _Block(object):
    __slots__ = ("kind", "c1", "c2", "c3", "down", "idx")


class _Weights(object):
    """bf16 tensor-core layouts of one weight set (online or target)."""

    def __init__(self, units, device, want_dgrad, ws=None):
        # ws = (numel, rows) of the standardised conv weights (weight-standardised nets): this set's standardised fp32
        # weights, their per-row (mean, rstd) and, with want_dgrad, the gradient the wgrad kernels write for them
        self.ws_w = self.ws_stats = self.ws_grad = None
        if ws is not None:
            self.ws_w = torch.empty(ws[0], dtype=F32, device=device)
            self.ws_stats = torch.empty((ws[1], 2), dtype=F32, device=device)
            self.ws_grad = torch.zeros(ws[0], dtype=F32, device=device) if want_dgrad else None
        # grouped units (ResNeXt conv2) keep block-diagonal tiles [C/64, 64, 9*64] in both layouts
        nf = sum(u.cout * u.kcols for u in units)
        self.pool_f = torch.empty(nf, dtype=BF16, device=device)
        self.pool_d = None
        self.wf, self.wd = [], []
        self.off_f, self.off_d = [], []
        off = 0
        for u in units:
            n = u.cout * u.kcols
            shape = (u.cout // 64, 64, u.kcols) if u.groups > 1 else (u.cout, u.kcols)
            self.wf.append(self.pool_f[off:off + n].view(shape))
            self.off_f.append(off)
            off += n
        if want_dgrad:
            nd = sum(u.cin * (u.kcols if u.groups > 1 else u.k * u.k * u.cout) for u in units if u.want_dgrad)
            self.pool_d = torch.empty(nd, dtype=BF16, device=device)
            off = 0
            for u in units:
                if u.want_dgrad:
                    if u.groups > 1:
                        n, shape = u.cin * u.kcols, (u.cin // 64, 64, u.kcols)
                    else:
                        n, shape = u.cin * u.k * u.k * u.cout, (u.cin, u.k * u.k * u.cout)
                    self.wd.append(self.pool_d[off:off + n].view(shape))
                    self.off_d.append(off)
                    off += n
                else:
                    self.wd.append(None)
                    self.off_d.append(-1)
        else:
            self.wd = [None] * len(units)
            self.off_d = [-1] * len(units)
        # descriptor tables of the grouped units' one-launch conversion (with and without the dgrad layouts)
        grouped = [u for u in units if u.groups > 1]
        self.grouped_max_c = max([u.cout for u in grouped] or [0])
        self.gdesc_with_dgrad = self.gdesc_fprop_only = None
        if grouped:
            assert ws is None or all(u.ws for u in grouped)
            rows = [[u.ws_off if u.ws else u.w_off, self.off_f[u.idx], -1, u.cout, u.cin // u.groups]
                    for u in grouped]
            self.gdesc_fprop_only = torch.tensor(rows, dtype=torch.int64, device=device)
            for r, u in zip(rows, grouped):
                r[2] = self.off_d[u.idx]
            self.gdesc_with_dgrad = torch.tensor(rows, dtype=torch.int64, device=device)
        # descriptor tables for the one-launch weight conversion (with and without the dgrad layouts); the
        # standardised weights have tables of their own (source: ws_w instead of the parameter vector)
        tables = {False: ([], []), True: ([], [])}
        for u in units:
            if u.groups > 1:
                continue
            rows_d, rows_n = tables[bool(u.ws)]
            fold = (u.k * 16 + u.k) if u.fold else 0
            base = [u.ws_off if u.ws else u.w_off, self.off_f[u.idx], -1, u.cout, u.cin, u.cpad, u.k * u.k, fold]
            rows_n.append(list(base))
            base[2] = self.off_d[u.idx] if (u.want_dgrad and not u.fold) else -1
            rows_d.append(base)
        self.desc_with_dgrad = self.desc_fprop_only = self.ws_desc_with_dgrad = self.ws_desc_fprop_only = None
        rows_d, rows_n = tables[False]
        if rows_n:
            self.desc_with_dgrad = torch.tensor(rows_d, dtype=torch.int64, device=device)
            self.desc_fprop_only = torch.tensor(rows_n, dtype=torch.int64, device=device)
        self.prep_blocks = ops.prep_blocks(rows_n)      # same shapes in both tables
        rows_d, rows_n = tables[True]
        if rows_n:
            self.ws_desc_with_dgrad = torch.tensor(rows_d, dtype=torch.int64, device=device)
            self.ws_desc_fprop_only = torch.tensor(rows_n, dtype=torch.int64, device=device)
        self.ws_prep_blocks = ops.prep_blocks(rows_n)
        # dedicated stem kernel layout ([7][4][64][8]) when the first conv is the torchvision 7x7/2 stem
        st = units[0]
        self.stem4_ok = (st.kind == "conv" and st.k == 7 and st.stride == 2 and st.pad == 3 and st.cin <= 4 and
                         st.cout == 64)
        self.w_stem4 = torch.empty(7 * 4 * 64 * 8, dtype=BF16, device=device) if self.stem4_ok else None


class _SplitWeights(object):
    """Weight-side plane layouts of one parameter set for the fp32-accurate forward path (csrc/split.cu):
    per conv / linear a bf16 [Cout, taps * T * Cpad] matrix; with want_dgrad (fp32-accurate backward, online set) also
    the dgrad layout [Cin, taps * T * Cout] of every layer whose input gradient is needed."""

    def __init__(self, units, device, T, want_dgrad=False):
        self.T = T
        sizes = [u.cout * u.k * u.k * T * u.cpad for u in units]
        self.pool = torch.empty(sum(sizes), dtype=BF16, device=device)
        self.w, off = [], 0
        for u, n in zip(units, sizes):
            self.w.append(self.pool[off:off + n].view(u.cout, u.k * u.k * T * u.cpad))
            off += n
        self.wd = [None] * len(units)
        if want_dgrad:
            dsizes = [u.cin * u.k * u.k * T * u.cout if u.want_dgrad else 0 for u in units]
            self.pool_d = torch.empty(sum(dsizes), dtype=BF16, device=device)
            off = 0
            for u, n in zip(units, dsizes):
                if n:
                    self.wd[u.idx] = self.pool_d[off:off + n].view(u.cin, u.k * u.k * T * u.cout)
                off += n

    def prepare(self, units, flat):
        for u in units:
            w = flat[u.w_off:u.w_off + u.w_numel].view(u.cout, u.cin, u.k * u.k)
            ops.prep_weight_planes(w, self.T, u.cpad, self.w[u.idx])
            if self.wd[u.idx] is not None:
                ops.prep_weight_dgrad_planes(w, self.T, self.wd[u.idx])


class _Pool(object):
    """Bump allocator over one fp32 tensor (one memset / allocation per pass instead of one per layer)."""

    def __init__(self, n, device, zero):
        self.buf = torch.zeros(n, dtype=F32, device=device) if zero else torch.empty(n, dtype=F32, device=device)
        self.off = 0

    def take(self, n):
        t = self.buf[self.off:self.off + n]
        self.off += n
        assert self.off <= self.buf.numel()
        return t


class _GraphedStep(object):
    """One captured training step: fixed buffers + the forward / backward CUDA graphs (see Engine.graphed_step)."""
    __slots__ = ("inputs", "saved", "outs", "logits", "d_pred", "fwd", "bwd", "pool", "fwd_launches", "bwd_launches",
                 "mean_ptr", "pending", "cls_planes")


class Engine(object):
    def __init__(self, model):
        self.model = model
        self.device = None
        self.ready = False
        self._bwd_cb_queued = False
        self._side_stream = None
        self._side_used = False
        self._side_refs = []
        self._lane_streams = None
        self._fin_events = None
        self._group_order = 0
        self._bwd_channel = 0
        # BYOL_B200_GRAPHS=0 keeps every launch eager (debugging / profiling single kernels)
        self.use_graphs = os.environ.get("BYOL_B200_GRAPHS", "1") != "0"
        self.graphs = {}
        # forward precision: 0 = bf16 operands (fast path); 3 / 6 = fp32 operands split into 3 / 6 bf16 product
        # terms (~16 / 24 mantissa bits), fp32 conv outputs, fp64 BatchNorm statistics (csrc/split.cu)
        self.T = 0
        # backward precision: False = bf16 operands; True (needs T) = the split scheme on every backward GEMM, fp32
        # gradients between layers, fp64 BatchNorm-backward sums (_backward_group_split)
        self.bwd32 = False
        self.cls_planes = None
        self.s_online = self.s_target = None
        # weight layouts of representations(): apart from the training step's, so that a call between a captured
        # forward and its backward leaves every buffer the graphs read untouched (allocated on first use)
        self.w_eval = self.s_eval = None
        self._mlp_bar = None
        # activation recomputation (recompute_plan): per geometry the set of blocks whose online lanes keep only the
        # block input, the BN coefficients and the output mask; _recompute_now is the set of the running forward
        self._plans = {}
        self._recompute_now = frozenset()
        self._mem_budget = None     # bytes: replaces the device's free memory in recompute_plan (tests)

    # ------------------------------------------------------------------------------------------
    # flat buffers
    # ------------------------------------------------------------------------------------------
    def flatten(self):
        """(Re)build the flat parameter / gradient buffers and re-point every Parameter at its slice
        (flat order = registration order, the reference's parameters_to_vector order, main.py:212,223)."""
        model = self.model
        params = list(model.parameters())
        dev = params[0].device
        if dev.type != "cuda":
            raise RuntimeError("byol_b200.BYOL runs on CUDA only (sm_90a kernels; no CPU path): move the model "
                               "to the GPU with .cuda() before calling it")
        total = sum(p.numel() for p in params)
        theta = torch.empty(total, dtype=F32, device=dev)
        grad = torch.zeros(total, dtype=F32, device=dev)
        self.offsets = {}
        off = 0
        for p in params:
            n = p.numel()
            theta[off:off + n].copy_(p.detach().reshape(-1).to(F32))
            p.data = theta[off:off + n].view(p.shape)
            p.grad = None
            self.offsets[id(p)] = off
            off += n
        self.params = params
        self.theta = theta
        self.grad = grad
        self.total = total
        self.device = dev
        ema = model.target_network
        if ema.mean is None or ema.mean.numel() != total or ema.mean.device != dev:
            ema.mean = torch.zeros(total, dtype=F32, device=dev) if ema.mean is None or ema.mean.numel() != total \
                else ema.mean.to(dev)

    def is_flat(self):
        if self.device is None:
            return False
        base = self.theta.data_ptr()
        for p in self.params:
            if p.data_ptr() != base + 4 * self.offsets[id(p)]:
                return False
        return True

    def attach_grads(self):
        """Make p.grad a view into the flat gradient buffer (zeroing it first if grads were set to None)."""
        if self.params[0].grad is None or self.params[0].grad.data_ptr() != self.grad.data_ptr():
            self.grad.zero_()
            for p in self.params:
                off = self.offsets[id(p)]
                p.grad = self.grad[off:off + p.numel()].view(p.shape)

    def _gview(self, off, n):
        return self.grad[off:off + n]

    # ------------------------------------------------------------------------------------------
    # plan
    # ------------------------------------------------------------------------------------------
    def _unit(self, mod, bn, name):
        u = _Unit()
        u.idx = len(self.units)
        u.name = name
        if isinstance(mod, nn.Conv2d):
            assert mod.kernel_size[0] == mod.kernel_size[1] and mod.stride[0] == mod.stride[1]
            assert mod.dilation[0] == 1 and mod.bias is None, "unsupported conv: %s" % name
            u.kind, u.cin, u.cout = "conv", mod.in_channels, mod.out_channels
            u.k, u.stride, u.pad = mod.kernel_size[0], mod.stride[0], mod.padding[0]
            u.groups = mod.groups     # > 1: grouped 3x3 (model.check_grouped_convs ran at construction)
            u.b_off = -1
        else:
            u.kind, u.cin, u.cout, u.k, u.stride, u.pad = "linear", mod.in_features, mod.out_features, 1, 1, 0
            u.groups = 1
            u.b_off = self.offsets[id(mod.bias)] if mod.bias is not None else -1
        u.cpad = (u.cin + 7) // 8 * 8
        # stem (3 input channels, 7x7): folded weight layout [Cout][KH*64] (see byol_prep_weight_fold)
        u.fold = u.kind == "conv" and u.cpad == 8 and 1 < u.k <= 8
        # grouped: one 64-channel k-block per tap (byol_prep_weights_grouped)
        u.kcols = u.k * 64 if u.fold else u.k * u.k * (64 if u.groups > 1 else u.cpad)
        u.w_off = self.offsets[id(mod.weight)]
        u.w_numel = mod.weight.numel()
        u.bn = bn
        u.gn = None
        u.ws = getattr(mod, "standardized", False)     # WSConv2d (model.py): weight-standardised conv
        u.ws_off = -1
        if isinstance(bn, nn.GroupNorm):
            assert bn.affine and bn.num_groups == ops.GN_GROUPS, "unsupported GroupNorm: %s" % name
            u.bn, u.gn = None, bn
            u.g_off, u.beta_off = self.offsets[id(bn.weight)], self.offsets[id(bn.bias)]
        elif bn is not None:
            assert bn.affine and bn.track_running_stats and bn.momentum is not None, "unsupported BN: %s" % name
            u.g_off, u.beta_off = self.offsets[id(bn.weight)], self.offsets[id(bn.bias)]
        u.want_dgrad = u.cout % 8 == 0 and u.cin % 8 == 0
        self.units.append(u)
        return u

    def build_plan(self):
        self.walk_layers()
        self.module_key = self._module_key()
        self.bn_modules = [u.bn for u in self.units if u.bn is not None]
        self.bn_channels = sum(u.cout for u in self.units if u.bn is not None)
        self.sync = any(isinstance(b, nn.SyncBatchNorm) for b in self.bn_modules)
        self.group_norm = any(u.gn is not None for u in self.units)
        if self.T and (self.group_norm or self.ws_rows):
            raise ValueError("byol_b200: GroupNorm / weight-standardised layers run with bf16 operands only")
        ws = (self.ws_numel, self.ws_rows) if self.ws_rows else None
        self.ws_desc = None
        if ws is not None:
            self.ws_desc = torch.tensor([[u.w_off, u.ws_off, u.cout, u.w_numel // u.cout, r] for u, r in
                                         self._ws_units], dtype=torch.int64, device=self.device)
        self._side_stream = torch.cuda.Stream(device=self.device)
        # the same two streams serve the forward lane pairs and the backward views: every extra stream is an extra
        # caching-allocator pool, and pools do not share their cached blocks
        self._lane_streams = [torch.cuda.Stream(device=self.device) for _ in range(2)]
        self.w_online = _Weights(self.units, self.device, True, ws)
        self.w_target = _Weights(self.units, self.device, False, ws)
        self.graphs = {}           # captured steps point into the old buffers
        self._plans = {}
        self.s_online = self.s_target = None
        self.w_eval = self.s_eval = None
        if self.T:
            self.s_online = _SplitWeights(self.units, self.device, self.T, want_dgrad=self.bwd32)
            self.s_target = _SplitWeights(self.units, self.device, self.T)
        self.ready = True

    def walk_layers(self):
        """Units and blocks of the module tree (geometry and flat offsets).  Needs no device: before flatten() the
        offsets are those flatten() will assign."""
        model = self.model
        if not self.is_flat():
            self.offsets, off = {}, 0
            for p in model.parameters():
                self.offsets[id(p)] = off
                off += p.numel()
        self.units, self.blocks = [], []
        children = list(model.base_network.children())
        convs = [c for c in children if isinstance(c, nn.Conv2d)]
        bns = [c for c in children if isinstance(c, (nn.modules.batchnorm._BatchNorm, nn.GroupNorm))]
        pools = [c for c in children if isinstance(c, nn.MaxPool2d)]
        assert len(convs) == 1 and len(bns) == 1 and len(pools) == 1, "unexpected ResNet stem"
        self.stem = self._unit(convs[0], bns[0], "stem")
        self.stem.want_dgrad = False
        mp = pools[0]
        self.pool_k, self.pool_s, self.pool_p = mp.kernel_size, mp.stride, mp.padding
        for layer in [c for c in children if isinstance(c, nn.Sequential)]:
            for blk in layer.children():
                b = _Block()
                b.kind = "bottleneck" if hasattr(blk, "conv3") else "basic"
                b.c1 = self._unit(blk.conv1, blk.bn1, "conv1")
                b.c2 = self._unit(blk.conv2, blk.bn2, "conv2")
                b.c3 = self._unit(blk.conv3, blk.bn3, "conv3") if b.kind == "bottleneck" else None
                b.down = None
                if blk.downsample is not None:
                    d = list(blk.downsample.children())
                    b.down = self._unit(d[0], d[1], "down")
                b.idx = len(self.blocks)
                self.blocks.append(b)
        self.rep_dim = (self.blocks[-1].c3 or self.blocks[-1].c2).cout
        self.mlps = []
        for seq in (model.head, model.predictor):
            l1, bn, _, l2 = list(seq.children())
            self.mlps.append((self._unit(l1, bn, "l1"), self._unit(l2, None, "l2")))
        self.cls = self._unit(model.linear_classifier, None, "classifier")
        self.cls.want_dgrad = False
        # weight-standardised convs: offsets of their standardised weights (and gradients) and their first row
        self._ws_units, self.ws_numel, self.ws_rows = [], 0, 0
        for u in self.units:
            if u.ws:
                u.ws_off = self.ws_numel
                self._ws_units.append((u, self.ws_rows))
                self.ws_numel += u.w_numel
                self.ws_rows += u.cout
        # Tensor-core layouts: bf16 activations are moved by TMA (16-byte row pitch), so every layer width on the
        # path must be a multiple of 8 — except the 3-channel image (padded on conversion) and the classifier's
        # class count (fp32 logits, pitched gradient), so that any dataset's label space works (main.py:208).
        for u in self.units:
            bad_in = u.cin % 8 != 0 and u is not self.stem
            bad_out = u.cout % 8 != 0 and u is not self.cls
            if bad_in or bad_out:
                raise ValueError("byol_b200: layer %s (%s %d -> %d): channel / feature counts on the tensor-core path "
                                 "must be multiples of 8 (only the image channels and the number of classes are free)"
                                 % (u.name, u.kind, u.cin, u.cout))

    def _module_key(self):
        """Identity of every sub-module: module surgery after the first forward (e.g. convert_sync_batchnorm, which
        re-uses the Parameters but replaces the BatchNorm modules) must rebuild the plan."""
        return tuple(id(m) for m in self.model.modules())

    def plan_is_current(self):
        return self.ready and self.is_flat() and self.module_key == self._module_key()

    def _nccl_statistics(self):
        """True if this model's SyncBatchNorm statistics go over NCCL: then the fused MLP, the two-stream schedule
        and graph capture are off.  A model without SyncBatchNorm never reaches comm.peer_exchange (collective on
        its first call, so every rank must reach it at the same point)."""
        return self.sync and comm.uses_nccl_for_statistics(self.device)

    def _sum_over_ranks(self, stats, rows, channel=0, want_local=False):
        """SyncBatchNorm: SUM the per-channel statistics `stats` (covering `rows` rows here) in place over the ranks
        on exchange `channel`.  Returns (the row count the sums cover, this rank's own sums if want_local else None)."""
        if not (self.sync and comm.world_size() > 1):
            return rows, None
        local = torch.empty_like(stats) if want_local else None
        comm.allreduce_sum_(stats, local_out=local, channel=channel)
        return rows * comm.world_size(), local

    def prep_weights(self, flat, wset, want_dgrad):
        """fp32 master (flat vector) -> bf16 tensor-core layouts of every conv / linear, one launch.  A
        weight-standardised net first standardises its conv weights (ws_fwd, one launch) and converts those."""
        with_d = want_dgrad and wset.pool_d is not None
        src = flat
        if wset.ws_w is not None:
            ops.ws_fwd(flat, self.ws_desc, self.ws_rows, wset.ws_w, wset.ws_stats)
            src = wset.ws_w
            if wset.ws_desc_fprop_only is not None:
                ops.prep_weights_multi(src, wset.pool_f, wset.pool_d,
                                       wset.ws_desc_with_dgrad if with_d else wset.ws_desc_fprop_only,
                                       wset.ws_prep_blocks)
        desc = wset.desc_with_dgrad if with_d else wset.desc_fprop_only
        if desc is not None:
            ops.prep_weights_multi(flat, wset.pool_f, wset.pool_d, desc, wset.prep_blocks)
        if wset.grouped_max_c:
            ops.prep_weights_grouped(src, wset.pool_f, wset.pool_d,
                                     wset.gdesc_with_dgrad if with_d else wset.gdesc_fprop_only, wset.grouped_max_c)
        if wset.stem4_ok:
            st = self.stem
            off = st.ws_off if st.ws else st.w_off
            ops.prep_weight_stem4((src if st.ws else flat)[off:off + st.w_numel].view(st.cout, st.cin, st.k, st.k),
                                  out=wset.w_stem4)

    # ------------------------------------------------------------------------------------------
    # activation recomputation: a memory model of one bf16 training step from the layer shapes, and the blocks whose
    # online lanes keep only their input, BN coefficients and output mask (the backward pass rebuilds the rest)
    # ------------------------------------------------------------------------------------------
    # The measured bf16 steps reserved 1.23-1.29x their peak allocated bytes (profiles/): under CUDA graphs a stream
    # does not reuse what another stream freed.  MARGIN covers what the model leaves out: LARS momentum, loss,
    # classifier, a training loop's prefetched input batches.
    RESERVE_FACTOR = 1.3
    MARGIN = 3 << 30

    def memory_model(self, n, h, w, lanes=2, target=True, mlps=True):
        """Bytes of one bf16 training step with n images per view at h x w, `lanes` online lanes (one view each) that
        save activations, the target pair's lanes if `target`, the projector and predictor if `mlps`.  The defaults
        are the BYOL step; the fine-tune step (finetune.py) is one lane without target pair or MLPs.
        Per block: "stored" / "kept" = what one
        online lane saves for it without / with recompute (the block output and its mask are kept either way),
        "dy" = the backward gradients one view holds until the weight-gradient join, "work" = one view's other backward
        transients of the block (a recomputed block adds stored - kept), "flops" = its recompute.  "first_input" is the first block's input
        (saved by each online lane), "fixed" the step's other activations (stem, MLPs, input layouts); "lanes" and
        "target" describe the step to step_need."""
        cs = ops.conv_out_size

        def conv(u, hi, wi):
            ho, wo = cs(hi, u.k, u.stride, u.pad), cs(wi, u.k, u.stride, u.pad)
            e = n * ho * wo * u.cout
            return ho, wo, e, 2 * e * (u.cin // u.groups) * u.k * u.k

        st = self.stem
        h0, w0, e0, _ = conv(st, h, w)
        H, W = cs(h0, self.pool_k, self.pool_s, self.pool_p), cs(w0, self.pool_k, self.pool_s, self.pool_p)
        first = 2 * n * H * W * st.cout
        blocks = []
        for b in self.blocks:
            h1, w1, e1, f1 = conv(b.c1, H, W)
            h2, w2, e2, f2 = conv(b.c2, h1, w1)
            e3 = f3 = ea2 = 0
            hl, wl, eo = h2, w2, e2
            if b.kind == "bottleneck":
                ea2 = e2
                hl, wl, eo, f3 = conv(b.c3, h2, w2)
                e3 = eo
            ed = fd = exs = 0
            if b.down is not None:
                _, _, ed, fd = conv(b.down, H, W)
                if self._down_as_gemm(b.down, H, W):
                    exs = n * (H // 2) * (W // 2) * b.down.cin
            kept = 2 * eo + eo // 8
            stored = kept + 2 * (e1 + e1 + e2 + ea2 + e3 + ed + exs)       # y1 a1 y2 a2 y3 yd xsub
            dy = 2 * (e1 + e2 + e3 + ed)
            blocks.append({"stored": stored, "kept": kept, "dy": dy, "flops": f1 + f2 + f3 + fd,
                           "work": dy + 2 * (eo + n * H * W * b.c1.cin)})
            H, W = hl, wl
        mlp = sum(2 * n * (l1.cin + 2 * l1.cout) for l1, _ in self.mlps) if mlps else 0   # x, h, a
        fixed = lanes * (2 * e0 + first // 2 + mlp + 2 * n * h * w * 8)   # per lane: y0, pool index, MLPs, its image
        return {"blocks": blocks, "first_input": first, "fixed": fixed, "lanes": lanes, "target": target}

    @staticmethod
    def lane_bytes(mm, plan):
        """Activation bytes one online lane saves in its block dicts under `plan`."""
        return mm["first_input"] + sum(blk["kept" if i in plan else "stored"] for i, blk in enumerate(mm["blocks"]))

    def step_need(self, mm, plan):
        """Device bytes one training step needs under `plan`: the peak of the forward (the online lanes' saved set,
        the target pair's largest block when the step has one) and of the backward (the saved set, the gradients of
        the stored blocks held for the side-stream weight gradients, one block's transients), scaled by
        RESERVE_FACTOR, plus MARGIN.  The step's lanes and target pair are those of `mm` (memory_model)."""
        blocks = mm["blocks"]
        saved = mm["lanes"] * self.lane_bytes(mm, plan)
        fwd = saved + (2 * max(blk["stored"] for blk in blocks) if mm["target"] else 0)
        bwd = saved + sum(blk["dy"] for i, blk in enumerate(blocks) if i not in plan) + \
            max(blk["work"] + (blk["stored"] - blk["kept"] if i in plan else 0) for i, blk in enumerate(blocks))
        return int(self.RESERVE_FACTOR * (max(fwd, bwd) + mm["fixed"])) + self.MARGIN

    def plan_blocks(self, mm, budget):
        """The fewest blocks to recompute so that the step needs at most `budget` bytes, taken in order of saved
        bytes per recomputed FLOP (ties: the earlier block); all blocks if even that does not fit; empty if the
        stored step fits."""
        blocks = mm["blocks"]
        order = sorted(range(len(blocks)),
                       key=lambda i: (-(blocks[i]["stored"] - blocks[i]["kept"]) / blocks[i]["flops"], i))
        plan = []
        for i in order:
            if self.step_need(mm, plan) <= budget:
                break
            plan.append(i)
        return frozenset(plan)

    def recompute_plan(self, n, h, w, lanes=2, target=True, mlps=True):
        """Blocks whose online lanes recompute their activations in the backward pass, for n images per view at h x w
        in a step of `lanes` saving lanes, with or without the target pair and the MLPs (memory_model): empty when
        the stored step fits in what the device can give (its free memory plus the allocator's unused
        cache, read once per geometry: the GPU may be shared).  Only the bf16 path recomputes."""
        if self.T:
            return frozenset()
        key = (n, h, w, lanes, target, mlps, comm.world_size(), self._mem_budget)
        plan = self._plans.get(key)
        if plan is None:
            budget = self._mem_budget
            if budget is None:
                free, _ = torch.cuda.mem_get_info(self.device)
                budget = free + torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)
            plan = self._plans[key] = self.plan_blocks(self.memory_model(n, h, w, lanes, target, mlps), budget)
        return plan

    # ------------------------------------------------------------------------------------------
    # forward building blocks (lists are per lane)
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _down_as_gemm(u, h, w):
        return u.k == 1 and u.stride == 2 and u.pad == 0 and h % 2 == 0 and w % 2 == 0

    def _conv_gn(self, u, xs, lanes, stem4=None, unit_stride=None):
        """raw conv outputs + GroupNorm coefficients (_GN) per lane.  The statistics are per image: train and eval
        compute the same thing, and nothing is exchanged between ranks."""
        C = u.cout
        ys, cs = [], []
        for i, (flat, wset, _) in enumerate(lanes):
            if stem4 is not None:
                y = ops.stem_conv_fprop(stem4[0][i], wset.w_stem4, stem4[1][i][0], stem4[1][i][1])
            else:
                y = self._conv(u, xs[i], wset, unit_stride)
            ys.append(y)
            cs.append(_GN(flat[u.g_off:u.g_off + C], flat[u.beta_off:u.beta_off + C], ops.gn_stats(y, u.gn.eps)))
        return ys, cs

    def _conv_bn(self, u, xs, lanes, train, stem4=None, unit_stride=None):
        """raw conv/linear outputs + BN coefficients [scale, shift, mean, invstd] per lane."""
        if u.gn is not None:
            return self._conv_gn(u, xs, lanes, stem4, unit_stride)
        L, C = len(lanes), u.cout
        stats = self._zpool.take(L * 2 * C) if train else None
        ys = []
        for i, (flat, wset, _) in enumerate(lanes):
            st = stats[i * 2 * C:(i + 1) * 2 * C] if train else None
            bias = flat[u.b_off:u.b_off + C] if u.b_off >= 0 else None
            x = xs[i]
            if stem4 is not None:
                y = ops.stem_conv_fprop(stem4[0][i], wset.w_stem4, stem4[1][i][0], stem4[1][i][1], stats=st)
            elif u.kind == "linear":
                y = ops.linear_fprop(x, wset.wf[u.idx], bias=bias, stats=st)
            else:
                y = self._conv(u, x, wset, unit_stride, stats=st)
            ys.append(y)
        coeffs = self._cpool.take(L * 4 * C).view(L, 4, C)
        bn = u.bn
        if train:
            count, _ = self._sum_over_ranks(stats, ys[0].numel() // C, channel=self._group_order)
            fin = self._fin_events
            if fin is not None and self._group_order == 1:
                torch.cuda.current_stream().wait_event(fin[u.idx])     # running stats: online pair first
            ops.bn_finalize_lanes(stats, count, [flat[u.g_off:u.g_off + C] for flat, _, _ in lanes],
                                  [flat[u.beta_off:u.beta_off + C] for flat, _, _ in lanes], bn.running_mean,
                                  bn.running_var, bn.momentum, bn.eps, coeffs)
            if fin is not None and self._group_order == 0:
                fin[u.idx] = torch.cuda.Event()
                fin[u.idx].record(torch.cuda.current_stream())
        else:
            for i, (flat, _, _) in enumerate(lanes):
                ops.bn_eval_coeffs(flat[u.g_off:u.g_off + C], flat[u.beta_off:u.beta_off + C], bn.running_mean,
                                   bn.running_var, bn.eps, coeffs[i])
        return ys, coeffs

    @staticmethod
    def _conv(u, x, wset, unit_stride=None, stats=None):
        """Raw conv output of a block conv.  The fused statistics do not change the stored y (the epilogue sums the
        bf16 values it stores), so _rebuild calls this without them and gets the forward's bits."""
        return ops.conv_fprop(x, wset.wf[u.idx], u.k, u.k, unit_stride or u.stride, u.pad, stats=stats)

    @staticmethod
    def _apply(y, c, relu, resid=None, rc=None, mask=None):
        if isinstance(c, _GN):
            return ops.gn_apply(y, c.gamma, c.beta, c.stats, relu, resid=resid, rgn=rc, mask_out=mask)
        C = y.shape[-1]
        out = torch.empty_like(y)
        ops.bn_apply(y.view(-1, C), c[0], c[1], relu, resid=None if resid is None else resid.view(-1, C),
                     rscale=None if rc is None else rc[0], rshift=None if rc is None else rc[1], out=out.view(-1, C),
                     mask_out=mask)
        return out

    def _block_fwd(self, b, xs, lanes, train):
        L = len(lanes)
        y1, c1 = self._conv_bn(b.c1, xs, lanes, train)
        a1 = [self._apply(y1[i], c1[i], True) for i in range(L)]
        y2, c2 = self._conv_bn(b.c2, a1, lanes, train)
        if b.kind == "bottleneck":
            a2 = [self._apply(y2[i], c2[i], True) for i in range(L)]
            y3, c3 = self._conv_bn(b.c3, a2, lanes, train)
            ylast, clast = y3, c3
        else:
            a2, y3, c3 = None, None, None
            ylast, clast = y2, c2
        # block output: the backward pass reads the ReLU mask as bits (1/16 of the activation's bytes)
        masks = [torch.empty(ylast[i].numel() // 8, dtype=torch.uint8, device=ylast[i].device)
                 if lanes[i][2] is not None else None for i in range(L)]
        xsub = None
        if b.down is not None:
            # 1x1 / stride-2 downsample: compact the pixels it reads, then it is a plain TMA-fed GEMM (fprop + wgrad)
            if self._down_as_gemm(b.down, xs[0].shape[1], xs[0].shape[2]):
                xsub = [ops.subsample2(x) for x in xs]
            yd, cd = self._conv_bn(b.down, xsub if xsub is not None else xs, lanes, train, unit_stride=1 if xsub else None)
            outs = [self._apply(ylast[i], clast[i], True, resid=yd[i], rc=cd[i], mask=masks[i]) for i in range(L)]
        else:
            yd, cd = None, None
            outs = [self._apply(ylast[i], clast[i], True, resid=xs[i], mask=masks[i]) for i in range(L)]
        recompute = b.idx in self._recompute_now
        for i, (_, _, saved) in enumerate(lanes):
            if saved is not None and recompute:
                # y1 .. yd are freed on return; _block_bwd rebuilds them from x and these coefficients (_rebuild)
                saved["blocks"].append({
                    "recompute": True, "mask": masks[i], "x": xs[i], "c1": c1[i], "c2": c2[i],
                    "c3": c3[i] if c3 is not None else None, "cd": cd[i] if cd is not None else None, "out": outs[i]})
            elif saved is not None:
                saved["blocks"].append({
                    "mask": masks[i], "xsub": xsub[i] if xsub is not None else None,
                    "x": xs[i], "y1": y1[i], "c1": c1[i], "a1": a1[i], "y2": y2[i], "c2": c2[i],
                    "a2": a2[i] if a2 is not None else None, "y3": y3[i] if y3 is not None else None,
                    "c3": c3[i] if c3 is not None else None, "yd": yd[i] if yd is not None else None,
                    "cd": cd[i] if cd is not None else None, "out": outs[i]})
        return outs

    def _mlp_fused_ok(self, mlp, b):
        l1, l2 = mlp
        if self._nccl_statistics():
            return False            # the in-kernel statistics exchange needs the peer-memory channel
        return l1.bn is not None and l1.b_off >= 0 and l2.b_off >= 0 and \
            ops.mlp_fused_supported(b, l1.cin, l1.cout, l2.cout)

    def _mlp_fwd_fused(self, mlp, xs, lanes, train, key):
        """Linear -> BatchNorm1d -> ReLU -> Linear as ONE cooperative kernel per lane (csrc/mlp_fused.cu): the hidden
        activation stays in shared memory between the two GEMMs; the BatchNorm statistics cross the grid
        (and, under SyncBatchNorm, the ranks) inside the kernel."""
        l1, l2 = mlp
        H, bn = l1.cout, l1.bn
        ch = self._group_order
        if self._mlp_bar is None:
            self._mlp_bar = torch.zeros((comm.NUM_CHANNELS, 2), dtype=torch.int32, device=self.device)
        peer, world = None, 1
        if train and self.sync and comm.world_size() > 1:
            peer, world = comm.peer_exchange(self.device)[ch], comm.world_size()
        fin = self._fin_events
        if train and fin is not None and ch == 1:
            torch.cuda.current_stream().wait_event(fin[l1.idx])      # running statistics: online pair first
        outs_f, outs_b = [], []
        for i, (flat, wset, saved) in enumerate(lanes):
            stats = self._zpool.take(2 * H) if train else None
            coeffs = self._cpool.take(4 * H).view(4, H)
            o, h, a = ops.mlp_fused_fwd(
                xs[i], wset.wf[l1.idx], flat[l1.b_off:l1.b_off + H], flat[l1.g_off:l1.g_off + H],
                flat[l1.beta_off:l1.beta_off + H], wset.wf[l2.idx], flat[l2.b_off:l2.b_off + l2.cout], stats,
                bn.running_mean, bn.running_var, bn.momentum, bn.eps, xs[i].shape[0] * world, coeffs, self._mlp_bar[ch],
                train, saved is not None, peer)
            outs_f.append(o)
            outs_b.append(ops.cast_bf16(o))
            if saved is not None:
                saved[key] = {"x": xs[i], "h": h, "c": coeffs, "a": a}
        if train and fin is not None and ch == 0:
            fin[l1.idx] = torch.cuda.Event()
            fin[l1.idx].record(torch.cuda.current_stream())
        return outs_f, outs_b

    def _mlp_fwd(self, mlp, xs, lanes, train, key):
        if self._mlp_fused_ok(mlp, xs[0].shape[0]):
            return self._mlp_fwd_fused(mlp, xs, lanes, train, key)
        l1, l2 = mlp
        L = len(lanes)
        h, c = self._conv_bn(l1, xs, lanes, train)
        a = [self._apply(h[i], c[i], True) for i in range(L)]
        outs_f, outs_b = [], []
        for i, (flat, wset, saved) in enumerate(lanes):
            o = ops.linear_fprop(a[i], wset.wf[l2.idx], bias=flat[l2.b_off:l2.b_off + l2.cout], out_fp32=True)
            outs_f.append(o)
            outs_b.append(ops.cast_bf16(o))
            if saved is not None:
                saved[key] = {"x": xs[i], "h": h[i], "c": c[i], "a": a[i]}
        return outs_f, outs_b

    def convert_inputs(self, augs, outs=None):
        """fp32 NCHW images -> the stem's input layout, once per distinct tensor (the online and the target lane of a
        view share it).  Returns per lane (nhwc8 | None, stem4 | None, H, W); `outs` (a previous result) is
        overwritten in place (CUDA-graph replays read these fixed buffers)."""
        st = self.stem
        conv, res = {}, []
        for i, a in enumerate(augs):
            if id(a) not in conv:
                # padded NHWC4 for the dedicated stem kernels, NHWC8 for the generic path (e.g. 384x384 images)
                use4 = self.w_online.stem4_ok and ops.stem4_supported(st.cin, st.cout, a.shape[2], a.shape[3], st.k,
                                                                      st.stride, st.pad)
                o = outs[i] if outs is not None else (None, None, 0, 0, None)
                pl = ops.nchw_to_planes(a, self.T, st.cpad, out=o[4]) if self.T else None
                conv[id(a)] = (None, ops.nchw_to_stem4(a, out=o[1]), a.shape[2], a.shape[3], pl) if use4 else \
                    (ops.nchw_to_nhwc8(a, out=o[0]), None, a.shape[2], a.shape[3], pl)
            res.append(conv[id(a)])
        return res

    def forward_lanes(self, augs, lanes, train, rep_bf16_out=None, x8=None, reps_only=False):
        """augs: fp32 NCHW inputs per lane; lanes: (flat params, weight set, saved dict or None) per lane.
        Returns per lane (representation fp32, projection fp32, prediction fp32); with reps_only (encoder-only
        evaluation, see representations) the forward stops after the average pool and returns (representation,).

        With four lanes (online x2, target x2) the two pairs run on two CUDA streams forked from / joined into the
        caller's stream: the HBM-bound BatchNorm kernels of one pair overlap the tensor-core convolutions of the
        other.  BN running statistics keep the reference's per-layer update order (online pair before target pair)
        through one event per layer."""
        L = len(lanes)
        main = torch.cuda.current_stream()
        if x8 is None:
            x8 = self.convert_inputs(augs)
        if self.T:
            res, reps_b = self._forward_split(x8, lanes, train, rep_bf16_out or [None] * L, reps_only)
            if train:
                torch._foreach_add_([b.num_batches_tracked for b in self.bn_modules], L)
            return res, reps_b
        if rep_bf16_out is None:
            rep_bf16_out = [None] * L
        saving = sum(lane[2] is not None for lane in lanes)
        if train and saving:
            img = x8[0][0] if x8[0][0] is not None else x8[0][1]
            # the lanes that save nothing are the target pair
            self._recompute_now = self.recompute_plan(img.shape[0], x8[0][2], x8[0][3], saving, L > saving,
                                                      not reps_only)
            if self._recompute_now and self.group_norm:
                self._recompute_now = frozenset()
                raise RuntimeError("byol_b200: a GroupNorm net at %d images per view and %dx%d does not fit in device "
                                   "memory with stored activations, and GroupNorm nets do not recompute activations: "
                                   "use a smaller batch size" % (img.shape[0], x8[0][2], x8[0][3]))
        # under SyncBatchNorm over NCCL the per-layer all-reduces serialise the lane pairs anyway: run all four lanes
        # lock-step on one stream there, which halves the number of (latency-bound) NCCL calls.  The peer-memory
        # exchange (comm.PeerExchange) has one channel per stream, so the two-stream schedule stays.
        two = L == 4 and not self._nccl_statistics()
        groups = [(list(range(0, 2)), self._lane_streams[0]), (list(range(2, 4)), self._lane_streams[1])] if two \
            else [(list(range(L)), main)]
        self._fin_events = {} if (two and train) else None
        results = [None] * L
        reps_b_all = [None] * L
        if two:
            ev = torch.cuda.Event()
            ev.record(main)
        for order, (idxs, stream) in enumerate(groups):
            if two:
                stream.wait_event(ev)
            self._group_order = order
            with torch.cuda.stream(stream):
                res, rb = self._forward_group([x8[i] for i in idxs], [lanes[i] for i in idxs], train,
                                              [rep_bf16_out[i] for i in idxs], reps_only)
            for j, i in enumerate(idxs):
                results[i], reps_b_all[i] = res[j], rb[j]
        if two:
            for _, stream in groups:
                e2 = torch.cuda.Event()
                e2.record(stream)
                main.wait_event(e2)
        self._fin_events = None
        self._group_order = 0
        self._recompute_now = frozenset()
        if train:
            torch._foreach_add_([b.num_batches_tracked for b in self.bn_modules], L)
        return results, reps_b_all

    def _forward_group(self, x8, lanes, train, rep_bf16_out, reps_only=False):
        L = len(lanes)
        st = self.stem
        self._zpool = _Pool(L * 2 * self.bn_channels, self.device, zero=True) if train else None
        self._cpool = _Pool(L * 4 * self.bn_channels, self.device, zero=False)
        xs4 = [x[1] for x in x8]
        hw = [(x[2], x[3]) for x in x8]
        x8 = [x[0] for x in x8]
        y0, c0 = self._conv_bn(st, x8, lanes, train, stem4=(xs4, hw) if xs4[0] is not None else None)
        xs = []
        for i, (_, _, saved) in enumerate(lanes):
            # stem: BN-apply + ReLU + max-pool fused (the normalised 112x112 map is never written)
            if st.gn is not None:
                p, idx = ops.gn_relu_maxpool_fwd(y0[i], *c0[i], k=self.pool_k, s=self.pool_s, p=self.pool_p,
                                                 want_idx=saved is not None)
            else:
                p, idx = ops.bn_relu_maxpool_fwd(y0[i], c0[i][0], c0[i][1], self.pool_k, self.pool_s, self.pool_p,
                                                 want_idx=saved is not None)
            xs.append(p)
            if saved is not None:
                saved.update({"x8": x8[i] if xs4[i] is None else (xs4[i], hw[i][0], hw[i][1]),
                              "y0": y0[i], "c0": c0[i], "a0_shape": tuple(y0[i].shape), "pool_idx": idx,
                              "blocks": []})
        for b in self.blocks:
            xs = self._block_fwd(b, xs, lanes, train)
        reps_f, reps_b = [], []
        for i in range(L):
            out_b = rep_bf16_out[i]
            n, h, w, c = xs[i].shape
            yf = torch.empty((n, c), dtype=F32, device=self.device)
            yb = out_b if out_b is not None else torch.empty((n, c), dtype=BF16, device=self.device)
            ops.check(ops.lib.byol_avgpool_fwd(xs[i].data_ptr(), yf.data_ptr(), yb.data_ptr(), n, h * w, c,
                                               ops._stream()), "byol_avgpool_fwd")
            reps_f.append(yf)
            reps_b.append(yb)
            if lanes[i][2] is not None:
                lanes[i][2]["final_shape"] = (n, h, w, c)
        if reps_only:
            return [(r,) for r in reps_f], reps_b
        # Under SyncBatchNorm the fused MLP kernels are cooperative (most of the GPU each) AND wait for their peer
        # ranks: two of them from different streams must never be schedulable in different orders on different ranks
        # (rank X resident with stream A's kernel, rank Y with stream B's -> circular wait).  So the second lane pair
        # enters its MLP section only after the first pair has left it: A-head, A-pred, B-head, B-pred everywhere.
        gate = train and self.sync and comm.world_size() > 1 and self._fin_events is not None and \
            self._mlp_fused_ok(self.mlps[0], reps_b[0].shape[0])
        if gate and self._group_order == 1:
            torch.cuda.current_stream().wait_event(self._fin_events["mlp_gate"])
        proj_f, proj_b = self._mlp_fwd(self.mlps[0], reps_b, lanes, train, "head")
        pred_f, _ = self._mlp_fwd(self.mlps[1], proj_b, lanes, train, "pred")
        if gate and self._group_order == 0:
            self._fin_events["mlp_gate"] = torch.cuda.Event()
            self._fin_events["mlp_gate"].record(torch.cuda.current_stream())
        return [(reps_f[i], proj_f[i], pred_f[i]) for i in range(L)], reps_b

    # ------------------------------------------------------------------------------------------
    # fp32-accurate forward ("split-bf16", csrc/split.cu): same layer walk, fp32 conv outputs, fp64 statistics.
    # Lanes run lock-step on the caller's stream.  For the online lanes the bf16 tensors the (bf16) backward pass
    # needs are written alongside, under the same keys as the fast path.
    # ------------------------------------------------------------------------------------------
    def _split_set(self, lane):
        """The plane layouts a lane runs on: its own weight set when it carries _SplitWeights (representations),
        else the online or target set by its parameter vector."""
        if isinstance(lane[1], _SplitWeights):
            return lane[1]
        return self.s_online if lane[0] is self.theta else self.s_target

    def _conv_bn_split(self, u, xs, lanes, train, is_linear=False):
        L, C, T = len(lanes), u.cout, self.T
        stats = torch.zeros(L * 2 * C, dtype=torch.float64, device=self.device) if train else None
        ys = []
        for i, (flat, _, _) in enumerate(lanes):
            wset = self._split_set(lanes[i])
            bias = flat[u.b_off:u.b_off + C] if u.b_off >= 0 else None
            if u.kind == "linear":
                y = ops.linear_fprop(xs[i], wset.w[u.idx], bias=bias, out_fp32=True)
            else:
                y = ops.conv_fprop(xs[i], wset.w[u.idx], u.k, u.k, u.stride, u.pad, out_fp32=True)
            if train:
                ops.stats_f32(y.view(-1, C), stats[i * 2 * C:(i + 1) * 2 * C])
            ys.append(y)
        coeffs = torch.empty((L, 4, C), dtype=F32, device=self.device)
        bn = u.bn
        if train:
            count, _ = self._sum_over_ranks(stats, ys[0].numel() // C)
            ops.bn_finalize_lanes_f64(stats, count, [flat[u.g_off:u.g_off + C] for flat, _, _ in lanes],
                                      [flat[u.beta_off:u.beta_off + C] for flat, _, _ in lanes], bn.running_mean,
                                      bn.running_var, bn.momentum, bn.eps, coeffs)
        else:
            for i, (flat, _, _) in enumerate(lanes):
                ops.bn_eval_coeffs(flat[u.g_off:u.g_off + C], flat[u.beta_off:u.beta_off + C], bn.running_mean,
                                   bn.running_var, bn.eps, coeffs[i])
        return ys, coeffs

    def _act_split(self, y, c, keep, resid=None, rc=None, block_out=False, want_mask=None):
        """BN-apply (+ residual) + ReLU of one lane's fp32 conv output -> (fp32 | None, planes NHWC, bf16 copy, mask).
        keep: write the bf16 copy; want_mask (default keep): the ReLU mask bits of a block output."""
        C = y.shape[-1]
        want_mask = keep if want_mask is None else want_mask
        o32, pl, cp, mask = ops.bn_apply_f32(y.view(-1, C), c[0], c[1], True, self.T,
                                             resid=None if resid is None else resid.view(-1, C),
                                             rscale=None if rc is None else rc[0],
                                             rshift=None if rc is None else rc[1], want_out32=block_out,
                                             want_planes=True, want_copy=keep, want_mask=want_mask and block_out)
        shp = tuple(y.shape[:-1])
        return (None if o32 is None else o32.view(shp + (C,)), pl.view(shp + (self.T * C,)),
                None if cp is None else cp.view(shp + (C,)), mask)

    def _block_fwd_split(self, b, X, lanes, train):
        """X: per lane (fp32 block input, its planes, its bf16 copy or None)."""
        L = len(lanes)
        save = [lanes[i][2] is not None for i in range(L)]
        # bf16 copies only for the bf16 backward; the fp32 backward keeps the fp32 tensors and recomputes the planes
        keep = [s and not self.bwd32 for s in save]
        xs_p = [x[1] for x in X]
        y1, c1 = self._conv_bn_split(b.c1, xs_p, lanes, train)
        a1 = [self._act_split(y1[i], c1[i], keep[i]) for i in range(L)]
        y2, c2 = self._conv_bn_split(b.c2, [a[1] for a in a1], lanes, train)
        if b.kind == "bottleneck":
            a2 = [self._act_split(y2[i], c2[i], keep[i]) for i in range(L)]
            y3, c3 = self._conv_bn_split(b.c3, [a[1] for a in a2], lanes, train)
            ylast, clast = y3, c3
        else:
            a2, y3, c3 = None, None, None
            ylast, clast = y2, c2
        if b.down is not None:
            yd, cd = self._conv_bn_split(b.down, xs_p, lanes, train)
            outs = [self._act_split(ylast[i], clast[i], keep[i], resid=yd[i], rc=cd[i], block_out=True,
                                    want_mask=save[i]) for i in range(L)]
        else:
            yd, cd = None, None
            outs = [self._act_split(ylast[i], clast[i], keep[i], resid=X[i][0], block_out=True, want_mask=save[i])
                    for i in range(L)]
        for i, (_, _, saved) in enumerate(lanes):
            if saved is not None and self.bwd32:
                saved["blocks"].append({
                    "mask": outs[i][3], "x": X[i][0], "y1": y1[i], "c1": c1[i], "y2": y2[i], "c2": c2[i],
                    "y3": y3[i] if y3 is not None else None, "c3": c3[i] if c3 is not None else None,
                    "yd": yd[i] if yd is not None else None, "cd": cd[i] if cd is not None else None})
            elif saved is not None:
                cb = ops.cast_bf16
                saved["blocks"].append({
                    "mask": outs[i][3], "xsub": None, "x": X[i][2], "y1": cb(y1[i]), "c1": c1[i], "a1": a1[i][2],
                    "y2": cb(y2[i]), "c2": c2[i], "a2": a2[i][2] if a2 is not None else None,
                    "y3": cb(y3[i]) if y3 is not None else None, "c3": c3[i] if c3 is not None else None,
                    "yd": cb(yd[i]) if yd is not None else None, "cd": cd[i] if cd is not None else None,
                    "out": outs[i][2]})
        return [(o[0], o[1], o[2]) for o in outs]

    def _mlp_fwd_split(self, mlp, X, lanes, train, key):
        """X: per lane (planes [b, T*in], bf16 copy [b, in] | None, fp32 [b, in]); returns fp32 outputs [b, out]."""
        l1, l2 = mlp
        L = len(lanes)
        h, c = self._conv_bn_split(l1, [x[0] for x in X], lanes, train)
        outs = []
        for i, (flat, _, saved) in enumerate(lanes):
            wset = self._split_set(lanes[i])
            _, ap, ab, _ = ops.bn_apply_f32(h[i], c[i][0], c[i][1], True, self.T, want_planes=True,
                                            want_copy=saved is not None and not self.bwd32)
            outs.append(ops.linear_fprop(ap, wset.w[l2.idx], bias=flat[l2.b_off:l2.b_off + l2.cout], out_fp32=True))
            if saved is not None and self.bwd32:
                saved[key] = {"x": X[i][2], "h": h[i], "c": c[i]}
            elif saved is not None:
                saved[key] = {"x": X[i][1], "h": ops.cast_bf16(h[i]), "c": c[i], "a": ab}
        return outs

    def _forward_split(self, x8, lanes, train, rep_bf16_out, reps_only=False):
        L, T = len(lanes), self.T
        st = self.stem
        keep = [lanes[i][2] is not None for i in range(L)]
        y0, c0 = self._conv_bn_split(st, [x[4] for x in x8], lanes, train)
        X = []
        for i, (_, _, saved) in enumerate(lanes):
            C = st.cout
            a0, _, _, _ = ops.bn_apply_f32(y0[i].view(-1, C), c0[i][0], c0[i][1], True, T, want_out32=True,
                                           want_planes=False)
            p32, idx = ops.maxpool_f32(a0.view(y0[i].shape), self.pool_k, self.pool_s, self.pool_p, want_idx=keep[i])
            pl, cp = ops.split_planes(p32.view(-1, C), T, want_copy=keep[i] and not self.bwd32)
            shp = tuple(p32.shape[:-1])
            X.append((p32, pl.view(shp + (T * C,)), None if cp is None else cp.view(shp + (C,))))
            if saved is not None and self.bwd32:
                saved.update({"x8": x8[i][4], "y0": y0[i], "c0": c0[i], "a0_shape": tuple(y0[i].shape),
                              "pool_idx": idx, "blocks": []})
            elif saved is not None:
                saved.update({"x8": x8[i][0] if x8[i][1] is None else (x8[i][1], x8[i][2], x8[i][3]),
                              "y0": ops.cast_bf16(y0[i]), "c0": c0[i], "a0_shape": tuple(y0[i].shape),
                              "pool_idx": idx, "blocks": []})
        for b in self.blocks:
            X = self._block_fwd_split(b, X, lanes, train)
        reps_f, reps_b, M = [], [], []
        if reps_only:
            return [(ops.avgpool_f32(X[i][0]),) for i in range(L)], [None] * L
        for i in range(L):
            n, h, w, c = X[i][0].shape
            rep = ops.avgpool_f32(X[i][0])
            pl, cp = ops.split_planes(rep, T, want_copy=True, copy_out=rep_bf16_out[i])
            reps_f.append(rep)
            reps_b.append(cp)
            M.append((pl, cp, rep))
            if keep[i]:
                lanes[i][2]["final_shape"] = (n, h, w, c)
        proj = self._mlp_fwd_split(self.mlps[0], M, lanes, train, "head")
        M2 = [ops.split_planes(p, T, want_copy=keep[i] and not self.bwd32) + (p,) for i, p in enumerate(proj)]
        pred = self._mlp_fwd_split(self.mlps[1], M2, lanes, train, "pred")
        return [(reps_f[i], proj[i], pred[i]) for i in range(L)], reps_b

    # ------------------------------------------------------------------------------------------
    # backward building blocks (online lanes only)
    # ------------------------------------------------------------------------------------------
    def _gn_bwd(self, u, gs, ys, cs, mask_mode, acts=None, want_dz=False):
        C = u.cout
        dys, dzs = [], []
        for i, c in enumerate(cs):
            act = None if acts is None else acts[i]
            s12 = torch.zeros((ys[i].shape[0], ops.GN_GROUPS, 2), dtype=F32, device=self.device)
            ops.gn_bwd_reduce(gs[i], ys[i], c.gamma, c.beta, c.stats, s12, mask_mode, act=act,
                              dgamma=self._gview(u.g_off, C), dbeta=self._gview(u.beta_off, C))
            dz = torch.empty_like(ys[i]) if want_dz else None
            dys.append(ops.gn_bwd_apply(gs[i], ys[i], c.gamma, c.beta, c.stats, s12, mask_mode, act=act, dz_out=dz))
            dzs.append(dz)
        return dys, dzs

    def _bn_bwd(self, u, gs, ys, cs, mask_mode, acts=None, want_dz=False):
        if u.gn is not None:
            return self._gn_bwd(u, gs, ys, cs, mask_mode, acts, want_dz)
        L, C = len(gs), u.cout
        s12 = self._bpool.take(L * 2 * C)
        for i in range(L):
            ops.bn_bwd_reduce(gs[i].view(-1, C), ys[i].view(-1, C), cs[i], s12[i * 2 * C:(i + 1) * 2 * C], mask_mode,
                              act=None if acts is None else (acts[i] if mask_mode == 3 else acts[i].view(-1, C)))
        count, local = self._sum_over_ranks(s12, ys[0].numel() // C, channel=self._bwd_channel, want_local=True)
        gamma = self.theta[u.g_off:u.g_off + C]
        dys, dzs = [], []
        for i in range(L):
            dz = torch.empty_like(ys[i]) if want_dz else None
            dy = torch.empty_like(ys[i])
            ops.bn_bwd_apply(gs[i].view(-1, C), ys[i].view(-1, C), cs[i], gamma, s12[i * 2 * C:(i + 1) * 2 * C], count,
                             mask_mode, act=None if acts is None else (acts[i] if mask_mode == 3 else acts[i].view(-1, C)),
                             dy=dy.view(-1, C),
                             dz_out=None if dz is None else dz.view(-1, C),
                             s12_local=None if local is None else local[i * 2 * C:(i + 1) * 2 * C],
                             dgamma=self._gview(u.g_off, C), dbeta=self._gview(u.beta_off, C))
            dys.append(dy)
            dzs.append(dz)
        return dys, dzs

    def _wgrad(self, u, xs, dys, unit_stride=None, planes=False):
        """dW += dY^T * im2col(X) on the side stream: the weight-gradient GEMMs only feed the flat gradient buffer, so
        they overlap with the HBM-bound BatchNorm-backward kernels of the next layer on the main stream.
        planes: xs / dys are split-operand planes (fp32-accurate backward)."""
        if u.ws:      # the gradient of the standardised weight; ws_bwd maps it to the parameter's
            dw = self.w_online.ws_grad[u.ws_off:u.ws_off + u.w_numel].view(u.cout, u.cin // u.groups, u.k, u.k)
        else:
            dw = self._gview(u.w_off, u.w_numel).view(u.cout, u.cin // u.groups, u.k, u.k)
        launch = self._launch_wgrad_planes if planes else self._launch_wgrad
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self._side_stream.wait_event(ev)
        with torch.cuda.stream(self._side_stream):
            launch(u, xs, dys, dw, unit_stride)
        # keep the operands alive until the launching stream has joined the side stream (no record_stream: that would
        # add an allocator event per tensor); after the join, reuse by the owning stream is ordered behind the reads
        self._side_refs.append((xs, dys))
        self._side_used = True

    def _launch_wgrad(self, u, xs, dys, dw, unit_stride=None):
        for x, dy in zip(xs, dys):
            if isinstance(x, tuple):      # stem: (padded NHWC4 image, H, W) -> dedicated kernel
                ops.stem_conv_wgrad(x[0], dy, dw, x[1], x[2])
            elif u.kind == "linear":
                ops.conv_wgrad(x.view(x.shape[0], 1, 1, -1), dy.view(dy.shape[0], 1, 1, -1), dw, 1, 1, 1, 0)
            else:
                ops.conv_wgrad(x, dy, dw, u.k, u.k, unit_stride or u.stride, u.pad)

    def _launch_wgrad_planes(self, u, xps, dyps, dw, unit_stride=None):
        for xp, dyp in zip(xps, dyps):
            if u.kind == "linear":
                ops.conv_wgrad_planes(xp.view(xp.shape[0], 1, 1, -1), dyp.view(dyp.shape[0], 1, 1, -1), dw, 1, 1, 1, 0,
                                      self.T)
            else:
                ops.conv_wgrad_planes(xp, dyp, dw, u.k, u.k, u.stride, u.pad, self.T)

    def _join_side_stream(self):
        if self._side_used:
            ev = torch.cuda.Event()
            ev.record(self._side_stream)
            torch.cuda.current_stream().wait_event(ev)
            self._side_used = False
            self._side_refs = []

    def _dgrad(self, u, dys, in_shapes, resids=None, resid_masks=None, resid_up=False, unit_stride=None):
        wd = self.w_online.wd[u.idx]
        outs = []
        for i, dy in enumerate(dys):
            n, h, w, _ = in_shapes[i]
            outs.append(ops.conv_dgrad(dy, wd, h, w, u.k, u.k, unit_stride or u.stride, u.pad,
                                       resid=None if resids is None else resids[i],
                                       resid_mask=None if resid_masks is None else resid_masks[i],
                                       resid_up=resid_up))
        return outs

    def _rebuild(self, b, s):
        """The saved dict of a block the forward recomputes: y1, a1, y2, a2, y3, xsub, yd again from its input and the
        forward's scale / shift, by the forward's kernels with the forward's arguments, on the current stream.  No
        statistics, running-statistic update or SyncBatchNorm exchange: the bits equal the forward's."""
        w, x = self.w_online, s["x"]
        r = {k: v for k, v in s.items() if k != "recompute"}
        r["y1"] = self._conv(b.c1, x, w)
        r["a1"] = self._apply(r["y1"], s["c1"], True)
        r["y2"] = self._conv(b.c2, r["a1"], w)
        r["a2"] = r["y3"] = r["xsub"] = r["yd"] = None
        if b.kind == "bottleneck":
            r["a2"] = self._apply(r["y2"], s["c2"], True)
            r["y3"] = self._conv(b.c3, r["a2"], w)
        if b.down is not None:
            if self._down_as_gemm(b.down, x.shape[1], x.shape[2]):
                r["xsub"] = ops.subsample2(x)
                r["yd"] = self._conv(b.down, r["xsub"], w, unit_stride=1)
            else:
                r["yd"] = self._conv(b.down, x, w)
        return r

    def _block_bwd(self, b, S, gs):
        if S[0].get("recompute"):
            out = self._block_bwd(b, [self._rebuild(b, s) for s in S], gs)
            # the weight gradients read the rebuilt tensors on the side stream: join, so that they are freed here
            self._join_side_stream()
            return out
        L = len(gs)
        outs = [s["out"] for s in S]
        xs = [s["x"] for s in S]
        xshapes = [tuple(x.shape) for x in xs]
        last = b.c3 if b.kind == "bottleneck" else b.c2
        ylast = [s["y3"] if b.kind == "bottleneck" else s["y2"] for s in S]
        clast = [s["c3"] if b.kind == "bottleneck" else s["c2"] for s in S]
        masks = [s["mask"] for s in S]
        # identity blocks whose first conv is 1x1: the masked gradient of the residual branch is never materialised,
        # the dgrad epilogue of that conv adds gs where the mask bit is set
        fuse_resid = b.down is None and b.c1.k == 1
        dyl, dzs = self._bn_bwd(last, gs, ylast, clast, 3, acts=masks, want_dz=b.down is None and not fuse_resid)
        resid_masks = None
        resid_up = False
        if b.down is not None:
            dyd, _ = self._bn_bwd(b.down, gs, [s["yd"] for s in S], [s["cd"] for s in S], 3, acts=masks)
            if S[0].get("xsub") is not None:
                self._wgrad(b.down, [s["xsub"] for s in S], dyd, unit_stride=1)
            else:
                self._wgrad(b.down, xs, dyd)
            if S[0].get("xsub") is not None and b.c1.k == 1 and b.c1.stride == 1:
                # plain GEMM on the strided pixels only; the conv1 dgrad epilogue scatters the compact result to the
                # even pixels (the 3/4-zero dense gradient map of the downsample branch is never written)
                resid = self._dgrad(b.down, dyd, [tuple(s["xsub"].shape) for s in S], unit_stride=1)
                resid_up = True
            else:
                resid = self._dgrad(b.down, dyd, xshapes)
        elif fuse_resid:
            resid, resid_masks = gs, masks
        else:
            resid = dzs
        if b.kind == "bottleneck":
            self._wgrad(b.c3, [s["a2"] for s in S], dyl)
            g2 = self._dgrad(b.c3, dyl, [tuple(s["a2"].shape) for s in S])
            dy2, _ = self._bn_bwd(b.c2, g2, [s["y2"] for s in S], [s["c2"] for s in S], 1)
        else:
            dy2 = dyl
        self._wgrad(b.c2, [s["a1"] for s in S], dy2)
        g1 = self._dgrad(b.c2, dy2, [tuple(s["a1"].shape) for s in S])
        dy1, _ = self._bn_bwd(b.c1, g1, [s["y1"] for s in S], [s["c1"] for s in S], 1)
        self._wgrad(b.c1, xs, dy1)
        return self._dgrad(b.c1, dy1, xshapes, resids=resid, resid_masks=resid_masks, resid_up=resid_up)

    def _mlp_bwd(self, mlp, S, douts):
        """douts: per lane fp32 or bf16 [b, out] gradient of the MLP output; returns bf16 grads of its input."""
        l1, l2 = mlp
        L = len(S)
        dbs = []
        for i in range(L):
            d = douts[i]
            ops.col_sum(d, self._gview(l2.b_off, l2.cout))
            dbs.append(ops.cast_bf16(d) if d.dtype == F32 else d)
        self._wgrad(l2, [s["a"] for s in S], dbs)
        das = [ops.linear_dgrad(dbs[i], self.w_online.wd[l2.idx]) for i in range(L)]
        dhs, _ = self._bn_bwd(l1, das, [s["h"] for s in S], [s["c"] for s in S], 1)
        for i in range(L):
            ops.col_sum(dhs[i], self._gview(l1.b_off, l1.cout))
        self._wgrad(l1, [s["x"] for s in S], dhs)
        return [ops.linear_dgrad(dhs[i], self.w_online.wd[l1.idx]) for i in range(L)]

    # ------------------------------------------------------------------------------------------
    # fp32-accurate backward (backward_precision="fp32"): the layer walk of _backward_group with the split scheme on
    # every GEMM (dY planes x weight planes for dgrad, dY planes x input planes for wgrad, T product terms, fp32
    # outputs), fp32 gradients between layers and fp64 BatchNorm-backward sums.  The online views run lock-step on
    # the caller's stream (like the split forward), not on one stream each as in the bf16 backward: dgamma / dbeta
    # then get the fp64 sum over both views with one rounding and no atomics, at the cost of the view-level overlap.
    # The weight gradients run on the side stream, joined after every block so that the recomputed planes they read
    # are freed block by block.
    # ------------------------------------------------------------------------------------------
    def _bn_bwd_f32(self, u, gs, ys, cs, mask_mode, masks=None, want_dz=False, want_f32=False):
        """-> per lane (dy planes, fp32 dy | None, fp32 dz | None)."""
        L, C = len(gs), u.cout
        s12 = torch.zeros(L * 2 * C, dtype=torch.float64, device=self.device)
        for i in range(L):
            ops.bn_bwd_reduce_f32(gs[i].view(-1, C), ys[i].view(-1, C), cs[i], s12[i * 2 * C:(i + 1) * 2 * C],
                                  mask_mode, mask=None if masks is None else masks[i])
        count, local = self._sum_over_ranks(s12, ys[0].numel() // C, want_local=True)
        gamma = self.theta[u.g_off:u.g_off + C]
        # dgamma / dbeta: the lanes' rank-local fp64 sums are added first, so the flat gradient takes ONE fp32 rounding
        # (by the last lane's apply kernel)
        loc = (s12 if local is None else local).view(L, 2 * C)
        loc = loc[0] if L == 1 else loc.sum(0)
        res = []
        for i in range(L):
            sl = slice(i * 2 * C, (i + 1) * 2 * C)
            last = i == L - 1
            pl, d32, dz = ops.bn_bwd_apply_f32(gs[i].view(-1, C), ys[i].view(-1, C), cs[i], gamma, s12[sl], count,
                                               mask_mode, self.T, mask=None if masks is None else masks[i],
                                               want_f32=want_f32, want_dz=want_dz, s12_local=loc if last else None,
                                               dgamma=self._gview(u.g_off, C) if last else None,
                                               dbeta=self._gview(u.beta_off, C) if last else None)
            shp = tuple(ys[i].shape[:-1])
            res.append((pl.view(shp + (self.T * C,)), d32, None if dz is None else dz.view(ys[i].shape)))
        return res

    def _planes(self, x):
        """fp32 [..., C] -> activation-pattern planes [..., T*C]."""
        C = x.shape[-1]
        return ops.split_planes(x.reshape(-1, C), self.T)[0].view(tuple(x.shape[:-1]) + (self.T * C,))

    def _act_planes(self, y, c):
        """relu(bn(y)) of a saved fp32 conv output, recomputed as planes (the input of the next layer)."""
        C = y.shape[-1]
        return ops.bn_apply_f32(y.view(-1, C), c[0], c[1], True, self.T)[1].view(tuple(y.shape[:-1]) + (self.T * C,))

    def _wgrad_split(self, u, xps, dyps):
        self._wgrad(u, xps, dyps, planes=True)

    def _dgrad_split(self, u, dyps, in_shapes, resids=None):
        wd = self.s_online.wd[u.idx]
        return [ops.conv_dgrad_planes(dyp, wd, in_shapes[i][1], in_shapes[i][2], u.k, u.k, u.stride, u.pad, self.T,
                                      resid=None if resids is None else resids[i]) for i, dyp in enumerate(dyps)]

    def _block_bwd_split(self, b, S, gs):
        """gs: per lane fp32 gradient of the block output; returns the fp32 gradient of the block input."""
        xs = [s["x"] for s in S]
        xshapes = [tuple(x.shape) for x in xs]
        xps = [self._planes(x) for x in xs]
        last = b.c3 if b.kind == "bottleneck" else b.c2
        key = "3" if b.kind == "bottleneck" else "2"
        masks = [s["mask"] for s in S]
        rl = self._bn_bwd_f32(last, gs, [s["y" + key] for s in S], [s["c" + key] for s in S], 3, masks=masks,
                              want_dz=b.down is None)
        dyl = [r[0] for r in rl]
        if b.down is not None:
            dyd = [r[0] for r in self._bn_bwd_f32(b.down, gs, [s["yd"] for s in S], [s["cd"] for s in S], 3,
                                                  masks=masks)]
            self._wgrad_split(b.down, xps, dyd)
            resid = self._dgrad_split(b.down, dyd, xshapes)
        else:
            resid = [r[2] for r in rl]
        if b.kind == "bottleneck":
            a2 = [self._act_planes(s["y2"], s["c2"]) for s in S]
            self._wgrad_split(b.c3, a2, dyl)
            g2 = self._dgrad_split(b.c3, dyl, [tuple(s["y2"].shape) for s in S])
            dy2 = [r[0] for r in self._bn_bwd_f32(b.c2, g2, [s["y2"] for s in S], [s["c2"] for s in S], 1)]
        else:
            dy2 = dyl
        a1 = [self._act_planes(s["y1"], s["c1"]) for s in S]
        self._wgrad_split(b.c2, a1, dy2)
        g1 = self._dgrad_split(b.c2, dy2, [tuple(s["y1"].shape) for s in S])
        dy1 = [r[0] for r in self._bn_bwd_f32(b.c1, g1, [s["y1"] for s in S], [s["c1"] for s in S], 1)]
        self._wgrad_split(b.c1, xps, dy1)
        out = self._dgrad_split(b.c1, dy1, xshapes, resids=resid)
        self._join_side_stream()
        return out

    def _mlp_bwd_split(self, mlp, S, douts):
        """douts: per lane fp32 [b, out] gradient of the MLP output; returns fp32 grads of its input."""
        l1, l2 = mlp
        L, T = len(S), self.T
        dps = []
        for i in range(L):
            ops.col_sum(douts[i], self._gview(l2.b_off, l2.cout))
            dps.append(ops.split_planes(douts[i], T)[0])
        self._wgrad_split(l2, [self._act_planes(s["h"], s["c"]) for s in S], dps)
        das = [ops.linear_dgrad_planes(dps[i], self.s_online.wd[l2.idx], T) for i in range(L)]
        rh = self._bn_bwd_f32(l1, das, [s["h"] for s in S], [s["c"] for s in S], 1, want_f32=True)
        for i in range(L):
            ops.col_sum(rh[i][1], self._gview(l1.b_off, l1.cout))
        dhs = [r[0] for r in rh]
        self._wgrad_split(l1, [self._planes(s["x"]) for s in S], dhs)
        out = [ops.linear_dgrad_planes(dhs[i], self.s_online.wd[l1.idx], T) for i in range(L)]
        self._join_side_stream()
        return out

    def _backward_group_split(self, saved, d_reps, d_projs, d_preds):
        L = len(saved)
        if all(d is None for d in d_preds) and all(d is None for d in d_projs) and all(d is None for d in d_reps):
            return
        zero = lambda ref: torch.zeros_like(ref)
        head_in = None
        if any(d is not None for d in d_preds):
            ref = [d for d in d_preds if d is not None][0]
            dq = [(d if d is not None else zero(ref)).contiguous() for d in d_preds]
            head_in = self._mlp_bwd_split(self.mlps[1], [s["pred"] for s in saved], dq)
        if any(d is not None for d in d_projs):
            ref = [d for d in d_projs if d is not None][0]
            extra = [(d if d is not None else zero(ref)).contiguous() for d in d_projs]
            head_in = extra if head_in is None else [head_in[i] + e for i, e in enumerate(extra)]
        rep_g = None
        if head_in is not None:
            rep_g = self._mlp_bwd_split(self.mlps[0], [s["head"] for s in saved], head_in)
        if rep_g is None and all(d is None for d in d_reps):
            return
        gs = []
        for i, s in enumerate(saved):
            n, h, w, c = s["final_shape"]
            du = d_reps[i].contiguous() if d_reps[i] is not None else None
            gs.append(ops.avgpool_bwd_f32(None if rep_g is None else rep_g[i], du, n, h, w, c))
        for bi in range(len(self.blocks) - 1, -1, -1):
            gs = self._block_bwd_split(self.blocks[bi], [s["blocks"][bi] for s in saved], gs)
        g0 = []
        for i, s in enumerate(saved):
            n, h, w, c = s["a0_shape"]
            g0.append(ops.maxpool_bwd_f32(gs[i], s["pool_idx"], h, w, self.pool_k, self.pool_s, self.pool_p))
        dy0 = [r[0] for r in self._bn_bwd_f32(self.stem, g0, [s["y0"] for s in saved], [s["c0"] for s in saved], 1)]
        self._wgrad_split(self.stem, [s["x8"] for s in saved], dy0)
        self._join_side_stream()

    def backward_online(self, saved, d_reps, d_projs, d_preds, notify=True):
        """Backward of the online views.  Each view runs on its own CUDA stream (forked from / joined into the
        caller's stream) so that one view's HBM-bound BatchNorm-backward kernels overlap the other's GEMMs; both
        accumulate into the same flat gradient buffer with atomic reductions."""
        if notify:
            self.notify_backward()
        L = len(saved)
        if self.bwd32:
            self._backward_group_split(saved, d_reps, d_projs, d_preds)
            return
        ws = self.w_online.ws_grad
        if ws is not None:
            ws.zero_()
        if L != 2 or self._nccl_statistics():
            self._bwd_channel = 0
            self._backward_group(saved, d_reps, d_projs, d_preds)
        else:
            self._backward_views(saved, d_reps, d_projs, d_preds)
        if ws is not None:
            # after both views and their weight gradients: the parameter gradient of every standardised conv weight
            w = self.w_online
            ops.ws_bwd(ws, w.ws_w, w.ws_stats, self.ws_desc, self.ws_rows, self.grad)

    def _backward_views(self, saved, d_reps, d_projs, d_preds):
        L = len(saved)
        main = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(main)
        for i in range(L):
            stream = self._lane_streams[i]
            stream.wait_event(ev)
            with torch.cuda.stream(stream):
                self._bwd_channel = i      # one exchange channel per view / stream
                self._backward_group([saved[i]], [d_reps[i]], [d_projs[i]], [d_preds[i]])
        for i in range(L):
            e2 = torch.cuda.Event()
            e2.record(self._lane_streams[i])
            main.wait_event(e2)

    def _backward_group(self, saved, d_reps, d_projs, d_preds):
        """saved: per online view the dict filled by forward_lanes; d_*: fp32 grads (or None) of the outputs."""
        L = len(saved)
        self._bpool = _Pool(L * 2 * self.bn_channels, self.device, zero=True)
        zero = lambda ref: torch.zeros_like(ref)
        # predictor
        if all(d is None for d in d_preds) and all(d is None for d in d_projs) and all(d is None for d in d_reps):
            return
        head_in = None
        if any(d is not None for d in d_preds):
            dq = [d if d is not None else zero(d_preds[[j for j in range(L) if d_preds[j] is not None][0]])
                  for d in d_preds]
            head_in = self._mlp_bwd(self.mlps[1], [s["pred"] for s in saved], [d.contiguous() for d in dq])
        if any(d is not None for d in d_projs):
            ref = [d for d in d_projs if d is not None][0]
            extra = [d if d is not None else zero(ref) for d in d_projs]
            head_in = [e.contiguous() if head_in is None else (head_in[i].float() + e) for i, e in enumerate(extra)]
        rep_g = None
        if head_in is not None:
            rep_g = self._mlp_bwd(self.mlps[0], [s["head"] for s in saved], head_in)
        if rep_g is None and all(d is None for d in d_reps):
            self._join_side_stream()
            return
        gs = []
        for i, s in enumerate(saved):
            n, h, w, c = s["final_shape"]
            du = d_reps[i].contiguous() if d_reps[i] is not None else None
            if du is not None and du.dtype == BF16:
                # the fine-tune step's bf16 classifier dgrad (finetune.py) takes the kernel's bf16 input: the kernel adds
                # either input to 0.f, so the result has the bits of du.float() passed as the fp32 input
                assert rep_g is None
                gs.append(ops.avgpool_bwd(du, None, n, h, w, c))
                continue
            gs.append(ops.avgpool_bwd(None if rep_g is None else rep_g[i], du, n, h, w, c))
        for bi in range(len(self.blocks) - 1, -1, -1):
            gs = self._block_bwd(self.blocks[bi], [s["blocks"][bi] for s in saved], gs)
        # (folding the pool backward into both BatchNorm-backward passes was measured ~2 ms/step SLOWER: the window
        # search runs twice and costs more than the saved write + two reads of the 112x112 gradient map)
        g0 = []
        for i, s in enumerate(saved):
            n, h, w, c = s["a0_shape"]
            g0.append(ops.maxpool_bwd(gs[i], s["pool_idx"], h, w, self.pool_k, self.pool_s, self.pool_p))
        dy0, _ = self._bn_bwd(self.stem, g0, [s["y0"] for s in saved], [s["c0"] for s in saved], 1)
        self._wgrad(self.stem, [s["x8"] for s in saved], dy0)
        self._join_side_stream()

    # ------------------------------------------------------------------------------------------
    # CUDA-graph replay of the training step (forward of the 4 lanes + classifier, backward of the 2 online views)
    # ------------------------------------------------------------------------------------------
    def graph_key(self, a1):
        return (tuple(a1.shape), comm.world_size(), bool(self.sync), self.theta.data_ptr(), self.T, self.bwd32,
                self.recompute_plan(a1.shape[0], a1.shape[2], a1.shape[3]))

    def prep_step(self, mean, training):
        """All weight layouts one forward (+ backward) needs, from the fp32 masters."""
        self.prep_weights(self.theta, self.w_online, want_dgrad=training)
        if self.T:
            self.s_online.prepare(self.units, self.theta)
            self.s_target.prepare(self.units, mean)
        else:
            self.prep_weights(mean, self.w_target, want_dgrad=False)

    def representations(self, images, flat):
        """Encoder-only eval-mode forward of fp32 NCHW `images` at the parameter vector `flat` (theta or the EMA mean):
        the average-pooled encoder output, fp32 [B, rep_dim].  One lane on the caller's stream with eval BatchNorm
        (running statistics); nothing is saved or updated.  It runs the kernels of the eval forward's representation
        lanes on the same inputs, so the result has their bits.  Its weight layouts live in their own buffers
        (w_eval / s_eval, encoder layers only): the captured training step's buffers are neither read nor written."""
        enc = self.units[:self.mlps[0][0].idx]      # walk_layers lists the encoder's units first
        if self.T:
            if self.s_eval is None:
                self.s_eval = _SplitWeights(enc, self.device, self.T)
            self.s_eval.prepare(enc, flat)
            wset = self.s_eval
        else:
            if self.w_eval is None:
                self.w_eval = _Weights(enc, self.device, False, (self.ws_numel, self.ws_rows) if self.ws_rows else None)
            self.prep_weights(flat, self.w_eval, want_dgrad=False)
            wset = self.w_eval
        res, _ = self.forward_lanes([images], [(flat, wset, None)], False, reps_only=True)
        return res[0][0]

    def graphed_step(self, model, a1, a2):
        """Returns the captured step for this input geometry, or None while it is still warming up / if graphs are
        disabled.  First call with a new geometry: eager (sets kernel attributes, sizes the allocator).  Second call:
        capture — all ~1000 launches of the forward pass go into one graph and those of the backward pass into a
        second one, both in one private memory pool; the activations saved for the backward pass, the inputs, the
        outputs and the incoming prediction gradients are fixed buffers.  From then on a step costs two graph
        launches plus a handful of small eager kernels (input layout, loss, EMA, LARS) on the host."""
        if not self.use_graphs:
            return None
        if self._nccl_statistics():
            return None          # per-layer NCCL collectives stay eager; the peer-memory exchange is capturable
        key = self.graph_key(a1)
        st = self.graphs.get(key)
        if st is None:
            self.graphs = {key: "warm"}      # one geometry at a time: a captured step pins its activations
            return None
        if st == "warm":
            st = self._capture_step(model, a1, a2)
            self.graphs[key] = st
        return st

    def _capture_step(self, model, a1, a2):
        from ._lib import launch_count
        st = _GraphedStep()
        st.pending = False
        b = a1.shape[0]
        # fixed input buffers (written by the eager layout kernels before every replay)
        st.inputs = self.convert_inputs([a1]) + self.convert_inputs([a2])
        st.saved = [{}, {}]
        mean = model.target_network.mean
        lanes = [(self.theta, self.w_online, st.saved[0]), (self.theta, self.w_online, st.saved[1]),
                 (mean, self.w_target, None), (mean, self.w_target, None)]
        st.mean_ptr = mean.data_ptr()
        rep_cat = model._rep_cat
        torch.cuda.synchronize()
        # A dead model that is part of a reference cycle still owns its captured graphs until Python's cycle collector
        # runs.  If that happened during this capture, destroying those graphs (cudaGraphExecDestroy) would be an
        # unsafe call from the capturing thread and would invalidate the capture.  So collect first and keep the
        # collector off until both graphs are captured.
        gc.collect()
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            pool = torch.cuda.graph_pool_handle()
            st.fwd = torch.cuda.CUDAGraph()
            n0 = launch_count[0]
            with torch.cuda.graph(st.fwd, pool=pool, capture_error_mode="thread_local"):
                self.prep_step(mean, True)
                outs, _ = self.forward_lanes(None, lanes, True, rep_bf16_out=[rep_cat[:b], rep_cat[b:], None, None],
                                             x8=[st.inputs[0], st.inputs[1], st.inputs[0], st.inputs[1]])
                st.logits = self.classifier_forward(rep_cat, [outs[0][0], outs[1][0]])
            st.cls_planes = self.cls_planes
            st.fwd_launches = launch_count[0] - n0
            st.outs = [t for o in outs for t in o]
            # backward for the usual gradient pattern: only the two online predictions receive a gradient
            # (objective.py:23-24 detaches the targets; main.py:601 adds the classifier loss, which is stop-grad)
            st.d_pred = [torch.zeros_like(st.outs[2]), torch.zeros_like(st.outs[5])]
            st.bwd = torch.cuda.CUDAGraph()
            n0 = launch_count[0]
            with torch.cuda.graph(st.bwd, pool=pool, capture_error_mode="thread_local"):
                self.backward_online(st.saved, [None, None], [None, None], st.d_pred, notify=False)
            st.bwd_launches = launch_count[0] - n0
        finally:
            if gc_was_enabled:
                gc.enable()
        st.pool = pool
        return st

    # classifier (stop-grad input; main.py:250-252)
    def classifier_forward(self, rep_cat_b, reps_f32=None):
        u = self.cls
        flat = self.theta
        bias = flat[u.b_off:u.b_off + u.cout]
        self.cls_planes = None
        if self.T and reps_f32 is not None:
            pl = torch.cat([ops.split_planes(r, self.T)[0] for r in reps_f32], 0)
            if self.bwd32:
                self.cls_planes = pl      # the fp32 backward's weight gradient reads the representation planes
            return ops.linear_fprop(pl, self.s_online.w[u.idx], bias=bias, out_fp32=True)
        return ops.linear_fprop(rep_cat_b, self.w_online.wf[u.idx], bias=bias, out_fp32=True)

    def classifier_backward(self, rep_cat_b, d_logits, planes=None):
        """planes: the representation planes classifier_forward kept (fp32-accurate backward), else None."""
        self.notify_backward()
        u = self.cls
        d = d_logits.contiguous().float()
        ops.col_sum(d, self._gview(u.b_off, u.cout))
        cpad = (u.cout + 7) // 8 * 8
        if planes is not None:
            self._wgrad(u, [planes], [ops.split_planes(d, self.T, cpad=cpad)[0]], planes=True)
            self._join_side_stream()
            return
        # any class count: the bf16 gradient gets a 16-byte row pitch, the GEMM reads only the first `cout` columns
        db = ops.cast_bf16(d) if u.cout % 8 == 0 else ops.cast_bf16_pitched(d, cpad)
        self._wgrad(u, [rep_cat_b], [db])
        self._join_side_stream()

    # ------------------------------------------------------------------------------------------
    # DDP: one flat gradient all-reduce (mean) when the backward pass finishes (main.py:440-443, 617)
    # ------------------------------------------------------------------------------------------
    def notify_backward(self):
        self.attach_grads()
        if not self._bwd_cb_queued:
            self._bwd_cb_queued = True
            torch.autograd.Variable._execution_engine.queue_callback(self._finish_backward)

    def _finish_backward(self):
        self._bwd_cb_queued = False
        self._join_side_stream()
        comm.allreduce_mean_(self.grad)
