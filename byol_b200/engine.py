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
import os

import torch
import torch.nn as nn

from . import comm, ops

BF16 = torch.bfloat16
F32 = torch.float32


class _Unit(object):
    """One conv/linear (+ optional BN) layer: static geometry plus offsets into the flat parameter vector."""
    __slots__ = ("idx", "kind", "cin", "cout", "cpad", "k", "stride", "pad", "w_off", "w_numel", "b_off", "bn",
                 "g_off", "beta_off", "name", "want_dgrad", "fold", "kcols")


class _Block(object):
    __slots__ = ("kind", "c1", "c2", "c3", "down")


class _Weights(object):
    """bf16 tensor-core layouts of one weight set (online or target)."""

    def __init__(self, units, device, want_dgrad):
        nf = sum(u.cout * u.kcols for u in units)
        self.pool_f = torch.empty(nf, dtype=BF16, device=device)
        self.pool_d = None
        self.wf, self.wd = [], []
        self.off_f, self.off_d = [], []
        off = 0
        for u in units:
            n = u.cout * u.kcols
            self.wf.append(self.pool_f[off:off + n].view(u.cout, u.kcols))
            self.off_f.append(off)
            off += n
        if want_dgrad:
            nd = sum(u.cin * u.k * u.k * u.cout for u in units if u.want_dgrad)
            self.pool_d = torch.empty(nd, dtype=BF16, device=device)
            off = 0
            for u in units:
                if u.want_dgrad:
                    n = u.cin * u.k * u.k * u.cout
                    self.wd.append(self.pool_d[off:off + n].view(u.cin, u.k * u.k * u.cout))
                    self.off_d.append(off)
                    off += n
                else:
                    self.wd.append(None)
                    self.off_d.append(-1)
        else:
            self.wd = [None] * len(units)
            self.off_d = [-1] * len(units)
        # descriptor tables for the one-launch weight conversion (with and without the dgrad layouts)
        rows_d, rows_n = [], []
        for u in units:
            fold = (u.k * 16 + u.k) if u.fold else 0
            base = [u.w_off, self.off_f[u.idx], -1, u.cout, u.cin, u.cpad, u.k * u.k, fold]
            rows_n.append(list(base))
            base[2] = self.off_d[u.idx] if (u.want_dgrad and not u.fold) else -1
            rows_d.append(base)
        self.desc_with_dgrad = torch.tensor(rows_d, dtype=torch.int64, device=device)
        self.desc_fprop_only = torch.tensor(rows_n, dtype=torch.int64, device=device)
        self.prep_blocks = ops.prep_blocks(rows_n)      # same shapes in both tables
        # dedicated stem kernel layout ([7][4][64][8]) when the first conv is the torchvision 7x7/2 stem
        st = units[0]
        self.stem4_ok = (st.kind == "conv" and st.k == 7 and st.stride == 2 and st.pad == 3 and st.cin <= 4 and
                         st.cout == 64)
        self.w_stem4 = torch.empty(7 * 4 * 64 * 8, dtype=BF16, device=device) if self.stem4_ok else None


class _SplitWeights(object):
    """Weight-side plane layouts of one parameter set for the fp32-accurate forward path (csrc/split.cu):
    per conv / linear a bf16 [Cout, taps * T * Cpad] matrix."""

    def __init__(self, units, device, T):
        self.T = T
        sizes = [u.cout * u.k * u.k * T * u.cpad for u in units]
        self.pool = torch.empty(sum(sizes), dtype=BF16, device=device)
        self.w, off = [], 0
        for u, n in zip(units, sizes):
            self.w.append(self.pool[off:off + n].view(u.cout, u.k * u.k * T * u.cpad))
            off += n

    def prepare(self, units, flat):
        for u in units:
            w = flat[u.w_off:u.w_off + u.w_numel].view(u.cout, u.cin, u.k * u.k)
            ops.prep_weight_planes(w, self.T, u.cpad, self.w[u.idx])


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
                 "mean_ptr", "pending")


class Engine(object):
    def __init__(self, model):
        self.model = model
        self.device = None
        self.ready = False
        self._bwd_cb_queued = False
        self._side_stream = None
        self._side_used = False
        self._side_refs = []
        self.overlap_wgrad = os.environ.get("BYOL_B200_OVERLAP_WGRAD", "1") != "0"
        self.multi_stream = os.environ.get("BYOL_B200_MULTI_STREAM", "1") != "0"
        self._fwd_streams = None
        self._bwd_streams = None
        self._fin_events = None
        self._group_order = 0
        self._bwd_channel = 0
        # BYOL_B200_GRAPHS=0 keeps every launch eager (debugging / profiling single kernels)
        self.use_graphs = os.environ.get("BYOL_B200_GRAPHS", "1") != "0"
        self.graphs = {}
        # forward precision: 0 = bf16 operands (fast path); 3 / 6 = fp32 operands split into 3 / 6 bf16 product
        # terms (~16 / 24 mantissa bits), fp32 conv outputs, fp64 BatchNorm statistics (csrc/split.cu)
        self.T = 0
        self.s_online = self.s_target = None
        # block-output BatchNorm fused into the expanding 1x1 GEMMs (see _fuse3).  OFF by default: the statistics pass
        # re-runs the GEMM, so the fused form moves more work than the unfused conv + BN-apply kernels
        # (tools/time_fused.py times both).  It saves 7-14 GB of activations per 512 images; BYOL_B200_FUSE3=1
        # enables it.
        self.fuse3 = os.environ.get("BYOL_B200_FUSE3", "0") == "1"
        self.fuse3_max_planes = int(os.environ.get("BYOL_B200_FUSE3_MAX_PLANES", "128"))
        # projector / predictor forward as one cooperative kernel per lane (csrc/mlp_fused.cu); =0: four launches
        self.fused_mlp = os.environ.get("BYOL_B200_FUSED_MLP", "1") != "0"
        self._mlp_bar = None

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
            assert mod.groups == 1 and mod.dilation[0] == 1 and mod.bias is None, "unsupported conv: %s" % name
            u.kind, u.cin, u.cout = "conv", mod.in_channels, mod.out_channels
            u.k, u.stride, u.pad = mod.kernel_size[0], mod.stride[0], mod.padding[0]
            u.b_off = -1
        else:
            u.kind, u.cin, u.cout, u.k, u.stride, u.pad = "linear", mod.in_features, mod.out_features, 1, 1, 0
            u.b_off = self.offsets[id(mod.bias)] if mod.bias is not None else -1
        u.cpad = (u.cin + 7) // 8 * 8
        # stem (3 input channels, 7x7): folded weight layout [Cout][KH*64] (see byol_prep_weight_fold)
        u.fold = u.kind == "conv" and u.cpad == 8 and 1 < u.k <= 8
        u.kcols = u.k * 64 if u.fold else u.k * u.k * u.cpad
        u.w_off = self.offsets[id(mod.weight)]
        u.w_numel = mod.weight.numel()
        u.bn = bn
        if bn is not None:
            assert bn.affine and bn.track_running_stats and bn.momentum is not None, "unsupported BN: %s" % name
            u.g_off, u.beta_off = self.offsets[id(bn.weight)], self.offsets[id(bn.bias)]
        u.want_dgrad = u.cout % 8 == 0 and u.cin % 8 == 0
        self.units.append(u)
        return u

    def build_plan(self):
        model = self.model
        self.units, self.blocks = [], []
        children = list(model.base_network.children())
        convs = [c for c in children if isinstance(c, nn.Conv2d)]
        bns = [c for c in children if isinstance(c, nn.modules.batchnorm._BatchNorm)]
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
                self.blocks.append(b)
        self.rep_dim = (self.blocks[-1].c3 or self.blocks[-1].c2).cout
        self.mlps = []
        for seq in (model.head, model.predictor):
            l1, bn, _, l2 = list(seq.children())
            self.mlps.append((self._unit(l1, bn, "l1"), self._unit(l2, None, "l2")))
        self.cls = self._unit(model.linear_classifier, None, "classifier")
        self.cls.want_dgrad = False
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
        self.module_key = self._module_key()
        self.bn_modules = [u.bn for u in self.units if u.bn is not None]
        self.bn_channels = sum(u.cout for u in self.units if u.bn is not None)
        self.sync = any(isinstance(b, nn.SyncBatchNorm) for b in self.bn_modules)
        self._side_stream = torch.cuda.Stream(device=self.device) if self.overlap_wgrad else None
        # the same two streams serve the forward lane pairs and the backward views: every extra stream is an extra
        # caching-allocator pool, and pools do not share their cached blocks
        self._fwd_streams = [torch.cuda.Stream(device=self.device) for _ in range(2)]
        self._bwd_streams = self._fwd_streams
        self.w_online = _Weights(self.units, self.device, True)
        self.w_target = _Weights(self.units, self.device, False)
        self.graphs = {}           # captured steps point into the old buffers
        self.s_online = self.s_target = None
        if self.T:
            self.s_online = _SplitWeights(self.units, self.device, self.T)
            self.s_target = _SplitWeights(self.units, self.device, self.T)
        self.ready = True

    def _module_key(self):
        """Identity of every sub-module: module surgery after the first forward (e.g. convert_sync_batchnorm, which
        re-uses the Parameters but replaces the BatchNorm modules) must rebuild the plan."""
        return tuple(id(m) for m in self.model.modules())

    def plan_is_current(self):
        return self.ready and self.is_flat() and self.module_key == self._module_key()

    def world(self):
        return comm.world_size()

    def prep_weights(self, flat, wset, want_dgrad):
        """fp32 master (flat vector) -> bf16 tensor-core layouts of every conv / linear, one launch."""
        desc = wset.desc_with_dgrad if (want_dgrad and wset.pool_d is not None) else wset.desc_fprop_only
        ops.prep_weights_multi(flat, wset.pool_f, wset.pool_d, desc, wset.prep_blocks)
        if wset.stem4_ok:
            st = self.stem
            ops.prep_weight_stem4(flat[st.w_off:st.w_off + st.w_numel].view(st.cout, st.cin, st.k, st.k),
                                  out=wset.w_stem4)

    # ------------------------------------------------------------------------------------------
    # forward building blocks (lists are per lane)
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _down_as_gemm(u, x):
        return u.k == 1 and u.stride == 2 and u.pad == 0 and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0

    def _conv_bn(self, u, xs, lanes, train, stem4=None, unit_stride=None, stats_only=False):
        """raw conv/linear outputs + BN coefficients [scale, shift, mean, invstd] per lane.
        stats_only (1x1 / stride-1 convolutions): the GEMM runs for its column statistics only (nothing is written;
        in eval mode nothing runs at all) — pass 1 of the fused block-output BatchNorm, see _block_fwd."""
        L, C = len(lanes), u.cout
        stats = self._zpool.take(L * 2 * C) if train else None
        ys = []
        rows = xs[0].numel() // xs[0].shape[-1] if stats_only else None
        for i, (flat, wset, _) in enumerate(lanes):
            st = stats[i * 2 * C:(i + 1) * 2 * C] if train else None
            bias = flat[u.b_off:u.b_off + C] if u.b_off >= 0 else None
            x = xs[i]
            if stats_only:
                if train:
                    ops.gemm_fused(x.view(-1, x.shape[-1]), wset.wf[u.idx], stats=st, no_store=True)
                continue
            if stem4 is not None:
                y = ops.stem_conv_fprop(stem4[0][i], wset.w_stem4, stem4[1][i][0], stem4[1][i][1], stats=st)
            elif u.kind == "linear":
                y = ops.linear_fprop(x, wset.wf[u.idx], bias=bias, stats=st)
            else:
                y = ops.conv_fprop(x, wset.wf[u.idx], u.k, u.k, unit_stride or u.stride, u.pad, stats=st)
            ys.append(y)
        coeffs = self._cpool.take(L * 4 * C).view(L, 4, C)
        bn = u.bn
        if train:
            if rows is None:
                rows = ys[0].numel() // C
            count = rows
            if self.sync and self.world() > 1:
                comm.allreduce_sum_(stats, channel=self._group_order)
                count = rows * self.world()
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
    def _apply(y, c, relu, resid=None, rc=None, mask=None):
        C = y.shape[-1]
        out = torch.empty_like(y)
        ops.bn_apply(y.view(-1, C), c[0], c[1], relu, resid=None if resid is None else resid.view(-1, C),
                     rscale=None if rc is None else rc[0], rshift=None if rc is None else rc[1], out=out.view(-1, C),
                     mask_out=mask)
        return out

    def _fuse3(self, b, x):
        """Bottleneck blocks whose expanding 1x1 convolution (conv3: planes -> 4 x planes) and 1x1 downsample branch
        are plain GEMMs: their BatchNorm + residual + ReLU runs in the GEMM epilogue ("statistics pass + recompute"),
        so the 4 x planes wide raw outputs y3 / yd are never written or re-read.  The second GEMM pass costs tensor
        time, so the trade pays where the block is HBM-bound: planes <= fuse3_max_planes (stages 1-2 of ResNet-50)."""
        if not self.fuse3 or b.kind != "bottleneck" or b.c3.k != 1 or b.c3.stride != 1 or b.c3.pad != 0:
            return False
        if b.c3.cin > self.fuse3_max_planes:
            return False
        if b.down is not None:
            d = b.down
            if d.k != 1 or d.pad != 0 or not (d.stride == 1 or self._down_as_gemm(d, x)):
                return False
        return True

    def _block_fwd_fused3(self, b, xs, lanes, train):
        L = len(lanes)
        y1, c1 = self._conv_bn(b.c1, xs, lanes, train)
        a1 = [self._apply(y1[i], c1[i], True) for i in range(L)]
        y2, c2 = self._conv_bn(b.c2, a1, lanes, train)
        a2 = [self._apply(y2[i], c2[i], True) for i in range(L)]
        C3 = b.c3.cout
        _, c3 = self._conv_bn(b.c3, a2, lanes, train, stats_only=True)
        n, h, w, _ = a2[0].shape
        masks = [torch.empty(n * h * w * C3 // 8, dtype=torch.uint8, device=self.device)
                 if lanes[i][2] is not None else None for i in range(L)]
        xsub, cd = None, None
        if b.down is not None:
            d = b.down
            xsub = [ops.subsample2(x) for x in xs] if d.stride == 2 else None
            xin = xsub if xsub is not None else xs
            _, cd = self._conv_bn(d, xin, lanes, train, stats_only=True)
            # the normalised residual branch bn_d(conv_d(x)) straight from the GEMM epilogue
            resid = [ops.gemm_fused(xin[i].view(-1, d.cin), lanes[i][1].wf[d.idx], colscale=cd[i][0], bias=cd[i][1])
                     for i in range(L)]
        else:
            resid = [x.view(-1, C3) for x in xs]
        outs = []
        for i in range(L):
            o = ops.gemm_fused(a2[i].view(-1, b.c3.cin), lanes[i][1].wf[b.c3.idx], colscale=c3[i][0], bias=c3[i][1],
                               resid=resid[i], relu=True, mask_out=masks[i])
            outs.append(o.view(n, h, w, C3))
        for i, (_, _, saved) in enumerate(lanes):
            if saved is not None:
                saved["blocks"].append({
                    "fused3": True, "mask": masks[i], "xsub": xsub[i] if xsub is not None else None,
                    "x": xs[i], "y1": y1[i], "c1": c1[i], "a1": a1[i], "y2": y2[i], "c2": c2[i], "a2": a2[i],
                    "y3": None, "c3": c3[i], "yd": None, "cd": cd[i] if cd is not None else None, "out": outs[i]})
        return outs

    def _block_fwd(self, b, xs, lanes, train):
        if self._fuse3(b, xs[0]):
            return self._block_fwd_fused3(b, xs, lanes, train)
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
            if self._down_as_gemm(b.down, xs[0]):
                xsub = [ops.subsample2(x) for x in xs]
            yd, cd = self._conv_bn(b.down, xsub if xsub is not None else xs, lanes, train, unit_stride=1 if xsub else None)
            outs = [self._apply(ylast[i], clast[i], True, resid=yd[i], rc=cd[i], mask=masks[i]) for i in range(L)]
        else:
            yd, cd = None, None
            outs = [self._apply(ylast[i], clast[i], True, resid=xs[i], mask=masks[i]) for i in range(L)]
        for i, (_, _, saved) in enumerate(lanes):
            if saved is not None:
                saved["blocks"].append({
                    "mask": masks[i], "xsub": xsub[i] if xsub is not None else None,
                    "x": xs[i], "y1": y1[i], "c1": c1[i], "a1": a1[i], "y2": y2[i], "c2": c2[i],
                    "a2": a2[i] if a2 is not None else None, "y3": y3[i] if y3 is not None else None,
                    "c3": c3[i] if c3 is not None else None, "yd": yd[i] if yd is not None else None,
                    "cd": cd[i] if cd is not None else None, "out": outs[i]})
        return outs

    def _mlp_fused_ok(self, mlp, b):
        l1, l2 = mlp
        if not self.fused_mlp or (self.sync and comm.uses_nccl_for_statistics(self.device)):
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
        if train and self.sync and self.world() > 1:
            peer, world = comm.peer_exchange(self.device)[ch], self.world()
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

    def forward_lanes(self, augs, lanes, train, rep_bf16_out=None, x8=None):
        """augs: fp32 NCHW inputs per lane; lanes: (flat params, weight set, saved dict or None) per lane.
        Returns per lane (representation fp32, projection fp32, prediction fp32).

        With four lanes (online x2, target x2) the two pairs run on two CUDA streams forked from / joined into the
        caller's stream: the HBM-bound BatchNorm kernels of one pair overlap the tensor-core convolutions of the
        other.  BN running statistics keep the reference's per-layer update order (online pair before target pair)
        through one event per layer."""
        L = len(lanes)
        main = torch.cuda.current_stream()
        if x8 is None:
            x8 = self.convert_inputs(augs)
        if self.T:
            res, reps_b = self._forward_split(x8, lanes, train, rep_bf16_out or [None] * L)
            if train:
                torch._foreach_add_([b.num_batches_tracked for b in self.bn_modules], L)
            return res, reps_b
        if rep_bf16_out is None:
            rep_bf16_out = [None] * L
        # under SyncBatchNorm over NCCL the per-layer all-reduces serialise the lane pairs anyway: run all four lanes
        # lock-step on one stream there, which halves the number of (latency-bound) NCCL calls.  The peer-memory
        # exchange (comm.PeerExchange) has one channel per stream, so the two-stream schedule stays.
        two = self.multi_stream and L == 4 and not (self.sync and comm.uses_nccl_for_statistics(self.device))
        groups = [(list(range(0, 2)), self._fwd_streams[0]), (list(range(2, 4)), self._fwd_streams[1])] if two \
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
                                              [rep_bf16_out[i] for i in idxs])
            for j, i in enumerate(idxs):
                results[i], reps_b_all[i] = res[j], rb[j]
        if two:
            for _, stream in groups:
                e2 = torch.cuda.Event()
                e2.record(stream)
                main.wait_event(e2)
        self._fin_events = None
        self._group_order = 0
        if train:
            torch._foreach_add_([b.num_batches_tracked for b in self.bn_modules], L)
        return results, reps_b_all

    def _forward_group(self, x8, lanes, train, rep_bf16_out):
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
        # Under SyncBatchNorm the fused MLP kernels are cooperative (most of the GPU each) AND wait for their peer
        # ranks: two of them from different streams must never be schedulable in different orders on different ranks
        # (rank X resident with stream A's kernel, rank Y with stream B's -> circular wait).  So the second lane pair
        # enters its MLP section only after the first pair has left it: A-head, A-pred, B-head, B-pred everywhere.
        gate = train and self.sync and self.world() > 1 and self._fin_events is not None and \
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
    def _conv_bn_split(self, u, xs, lanes, train, is_linear=False):
        L, C, T = len(lanes), u.cout, self.T
        stats = torch.zeros(L * 2 * C, dtype=torch.float64, device=self.device) if train else None
        ys = []
        for i, (flat, _, _) in enumerate(lanes):
            wset = self.s_online if flat is self.theta else self.s_target
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
            rows = ys[0].numel() // C
            count = rows
            if self.sync and self.world() > 1:
                comm.allreduce_sum_(stats)
                count = rows * self.world()
            ops.bn_finalize_lanes_f64(stats, count, [flat[u.g_off:u.g_off + C] for flat, _, _ in lanes],
                                      [flat[u.beta_off:u.beta_off + C] for flat, _, _ in lanes], bn.running_mean,
                                      bn.running_var, bn.momentum, bn.eps, coeffs)
        else:
            for i, (flat, _, _) in enumerate(lanes):
                ops.bn_eval_coeffs(flat[u.g_off:u.g_off + C], flat[u.beta_off:u.beta_off + C], bn.running_mean,
                                   bn.running_var, bn.eps, coeffs[i])
        return ys, coeffs

    def _act_split(self, y, c, keep, resid=None, rc=None, block_out=False):
        """BN-apply (+ residual) + ReLU of one lane's fp32 conv output -> (fp32 | None, planes NHWC, bf16 copy, mask)."""
        C = y.shape[-1]
        o32, pl, cp, mask = ops.bn_apply_f32(y.view(-1, C), c[0], c[1], True, self.T,
                                             resid=None if resid is None else resid.view(-1, C),
                                             rscale=None if rc is None else rc[0],
                                             rshift=None if rc is None else rc[1], want_out32=block_out,
                                             want_planes=True, want_copy=keep, want_mask=keep and block_out)
        shp = tuple(y.shape[:-1])
        return (None if o32 is None else o32.view(shp + (C,)), pl.view(shp + (self.T * C,)),
                None if cp is None else cp.view(shp + (C,)), mask)

    def _block_fwd_split(self, b, X, lanes, train):
        """X: per lane (fp32 block input, its planes, its bf16 copy or None)."""
        L = len(lanes)
        keep = [lanes[i][2] is not None for i in range(L)]
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
            outs = [self._act_split(ylast[i], clast[i], keep[i], resid=yd[i], rc=cd[i], block_out=True)
                    for i in range(L)]
        else:
            yd, cd = None, None
            outs = [self._act_split(ylast[i], clast[i], keep[i], resid=X[i][0], block_out=True) for i in range(L)]
        for i, (_, _, saved) in enumerate(lanes):
            if saved is not None:
                cb = ops.cast_bf16
                saved["blocks"].append({
                    "mask": outs[i][3], "xsub": None, "x": X[i][2], "y1": cb(y1[i]), "c1": c1[i], "a1": a1[i][2],
                    "y2": cb(y2[i]), "c2": c2[i], "a2": a2[i][2] if a2 is not None else None,
                    "y3": cb(y3[i]) if y3 is not None else None, "c3": c3[i] if c3 is not None else None,
                    "yd": cb(yd[i]) if yd is not None else None, "cd": cd[i] if cd is not None else None,
                    "out": outs[i][2]})
        return [(o[0], o[1], o[2]) for o in outs]

    def _mlp_fwd_split(self, mlp, X, lanes, train, key):
        """X: per lane (planes [b, T*in], bf16 copy [b, in]); returns fp32 outputs [b, out]."""
        l1, l2 = mlp
        L = len(lanes)
        h, c = self._conv_bn_split(l1, [x[0] for x in X], lanes, train)
        outs = []
        for i, (flat, _, saved) in enumerate(lanes):
            wset = self.s_online if flat is self.theta else self.s_target
            _, ap, ab, _ = ops.bn_apply_f32(h[i], c[i][0], c[i][1], True, self.T, want_planes=True,
                                            want_copy=saved is not None)
            outs.append(ops.linear_fprop(ap, wset.w[l2.idx], bias=flat[l2.b_off:l2.b_off + l2.cout], out_fp32=True))
            if saved is not None:
                saved[key] = {"x": X[i][1], "h": ops.cast_bf16(h[i]), "c": c[i], "a": ab}
        return outs

    def _forward_split(self, x8, lanes, train, rep_bf16_out):
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
            pl, cp = ops.split_planes(p32.view(-1, C), T, want_copy=keep[i])
            shp = tuple(p32.shape[:-1])
            X.append((p32, pl.view(shp + (T * C,)), None if cp is None else cp.view(shp + (C,))))
            if saved is not None:
                saved.update({"x8": x8[i][0] if x8[i][1] is None else (x8[i][1], x8[i][2], x8[i][3]),
                              "y0": ops.cast_bf16(y0[i]), "c0": c0[i], "a0_shape": tuple(y0[i].shape),
                              "pool_idx": idx, "blocks": []})
        for b in self.blocks:
            X = self._block_fwd_split(b, X, lanes, train)
        reps_f, reps_b, M = [], [], []
        for i in range(L):
            n, h, w, c = X[i][0].shape
            rep = ops.avgpool_f32(X[i][0])
            pl, cp = ops.split_planes(rep, T, want_copy=True, copy_out=rep_bf16_out[i])
            reps_f.append(rep)
            reps_b.append(cp)
            M.append((pl, cp))
            if keep[i]:
                lanes[i][2]["final_shape"] = (n, h, w, c)
        proj = self._mlp_fwd_split(self.mlps[0], M, lanes, train, "head")
        M2 = [ops.split_planes(p, T, want_copy=keep[i]) for i, p in enumerate(proj)]
        pred = self._mlp_fwd_split(self.mlps[1], M2, lanes, train, "pred")
        return [(reps_f[i], proj[i], pred[i]) for i in range(L)], reps_b

    # ------------------------------------------------------------------------------------------
    # backward building blocks (online lanes only)
    # ------------------------------------------------------------------------------------------
    def _bn_bwd(self, u, gs, ys, cs, mask_mode, acts=None, want_dz=False):
        L, C = len(gs), u.cout
        s12 = self._bpool.take(L * 2 * C)
        for i in range(L):
            ops.bn_bwd_reduce(gs[i].view(-1, C), ys[i].view(-1, C), cs[i], s12[i * 2 * C:(i + 1) * 2 * C], mask_mode,
                              act=None if acts is None else (acts[i] if mask_mode == 3 else acts[i].view(-1, C)))
        rows = ys[0].numel() // C
        count, local = rows, None
        if self.sync and self.world() > 1:
            local = torch.empty_like(s12)
            comm.allreduce_sum_(s12, local_out=local, channel=self._bwd_channel)
            count = rows * self.world()
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

    def _wgrad(self, u, xs, dys, unit_stride=None):
        """dW += dY^T * im2col(X) on the side stream: the weight-gradient GEMMs only feed the flat gradient buffer, so
        they overlap with the HBM-bound BatchNorm-backward kernels of the next layer on the main stream."""
        dw = self._gview(u.w_off, u.w_numel).view(u.cout, u.cin, u.k, u.k)
        main = torch.cuda.current_stream()
        side = self._side_stream
        if side is None:
            self._launch_wgrad(u, xs, dys, dw, unit_stride)
            return
        ev = torch.cuda.Event()
        ev.record(main)
        side.wait_event(ev)
        with torch.cuda.stream(side):
            self._launch_wgrad(u, xs, dys, dw, unit_stride)
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

    def _join_side_stream(self):
        if self._side_stream is not None and self._side_used:
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

    def _bn_bwd_recompute(self, u, gs, xs2d, cs, masks):
        """BatchNorm backward of a block-output BN whose input y = x2d @ W^T was never stored (_block_fwd_fused3):
        both passes recompute y on the tensor cores — (1) sum dz, sum dz*xhat in the GEMM epilogue, (2) after the
        cross-rank exchange, dy = A*dz + B*y + Cc written straight from the epilogue.  dz = gs masked by the ReLU bits."""
        L, C = len(gs), u.cout
        wf = self.w_online.wf[u.idx]
        s12 = self._bpool.take(L * 2 * C)
        for i in range(L):
            prep = ops.bn_bwd_prep(cs[i][2], cs[i][3])
            ops.gemm_fused(xs2d[i], wf, colscale=prep[:C], bias=prep[C:], resid=gs[i].view(-1, C), resid_mask=masks[i],
                           stats=s12[i * 2 * C:(i + 1) * 2 * C], bwd_reduce=True)
        rows = xs2d[0].shape[0]
        count, local = rows, None
        if self.sync and self.world() > 1:
            local = torch.empty_like(s12)
            comm.allreduce_sum_(s12, local_out=local, channel=self._bwd_channel)
            count = rows * self.world()
        gamma = self.theta[u.g_off:u.g_off + C]
        dys = []
        for i in range(L):
            sl = slice(i * 2 * C, (i + 1) * 2 * C)
            abc = ops.bn_bwd_coeffs(s12[sl], cs[i], gamma, count, s12_local=None if local is None else local[sl],
                                    dgamma=self._gview(u.g_off, C), dbeta=self._gview(u.beta_off, C))
            dy = ops.gemm_fused(xs2d[i], wf, colscale=abc[:C], bias=abc[C:2 * C], resid=gs[i].view(-1, C),
                                resid_mask=masks[i], resid_colscale=abc[2 * C:])
            dys.append(dy.view(gs[i].shape))
        return dys

    def _block_bwd_fused3(self, b, S, gs):
        L = len(gs)
        xs = [s["x"] for s in S]
        xshapes = [tuple(x.shape) for x in xs]
        masks = [s["mask"] for s in S]
        a2 = [s["a2"] for s in S]
        dy3 = self._bn_bwd_recompute(b.c3, gs, [a.view(-1, b.c3.cin) for a in a2], [s["c3"] for s in S], masks)
        resid_masks, resid_up = None, False
        if b.down is not None:
            d = b.down
            xin = [s["xsub"] if s["xsub"] is not None else s["x"] for s in S]
            dyd = self._bn_bwd_recompute(d, gs, [x.view(-1, d.cin) for x in xin], [s["cd"] for s in S], masks)
            self._wgrad(d, xin, dyd, unit_stride=1)
            if S[0]["xsub"] is not None and b.c1.k == 1 and b.c1.stride == 1:
                resid = self._dgrad(d, dyd, [tuple(x.shape) for x in xin], unit_stride=1)
                resid_up = True
            elif S[0]["xsub"] is not None:
                raise RuntimeError("fused downsample branch needs a 1x1 / stride-1 conv1")   # not a torchvision net
            else:
                resid = self._dgrad(d, dyd, xshapes, unit_stride=1)
        else:
            resid, resid_masks = gs, masks          # masked residual gradient added by the conv1 dgrad epilogue
        self._wgrad(b.c3, a2, dy3)
        g2 = self._dgrad(b.c3, dy3, [tuple(a.shape) for a in a2])
        dy2, _ = self._bn_bwd(b.c2, g2, [s["y2"] for s in S], [s["c2"] for s in S], 1)
        self._wgrad(b.c2, [s["a1"] for s in S], dy2)
        g1 = self._dgrad(b.c2, dy2, [tuple(s["a1"].shape) for s in S])
        dy1, _ = self._bn_bwd(b.c1, g1, [s["y1"] for s in S], [s["c1"] for s in S], 1)
        self._wgrad(b.c1, xs, dy1)
        return self._dgrad(b.c1, dy1, xshapes, resids=resid, resid_masks=resid_masks, resid_up=resid_up)

    def _block_bwd(self, b, S, gs):
        if S[0].get("fused3"):
            return self._block_bwd_fused3(b, S, gs)
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

    def backward_online(self, saved, d_reps, d_projs, d_preds, notify=True):
        """Backward of the online views.  Each view runs on its own CUDA stream (forked from / joined into the
        caller's stream) so that one view's HBM-bound BatchNorm-backward kernels overlap the other's GEMMs; both
        accumulate into the same flat gradient buffer with atomic reductions."""
        if notify:
            self.notify_backward()
        L = len(saved)
        main = torch.cuda.current_stream()
        if not (self.multi_stream and L == 2) or (self.sync and comm.uses_nccl_for_statistics(self.device)):
            self._bwd_channel = 0
            self._backward_group(saved, d_reps, d_projs, d_preds)
            return
        ev = torch.cuda.Event()
        ev.record(main)
        for i in range(L):
            stream = self._bwd_streams[i]
            stream.wait_event(ev)
            with torch.cuda.stream(stream):
                self._bwd_channel = i      # one exchange channel per view / stream
                self._backward_group([saved[i]], [d_reps[i]], [d_projs[i]], [d_preds[i]])
        for i in range(L):
            e2 = torch.cuda.Event()
            e2.record(self._bwd_streams[i])
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
        return (tuple(a1.shape), self.world(), bool(self.sync), self.theta.data_ptr(), self.multi_stream,
                self.overlap_wgrad, self.T, self.fuse3, self.fuse3_max_planes, self.fused_mlp)

    def prep_step(self, mean, training):
        """All weight layouts one forward (+ backward) needs, from the fp32 masters."""
        self.prep_weights(self.theta, self.w_online, want_dgrad=training)
        if self.T:
            self.s_online.prepare(self.units, self.theta)
            self.s_target.prepare(self.units, mean)
        else:
            self.prep_weights(mean, self.w_target, want_dgrad=False)

    def graphed_step(self, model, a1, a2):
        """Returns the captured step for this input geometry, or None while it is still warming up / if graphs are
        disabled.  First call with a new geometry: eager (sets kernel attributes, sizes the allocator).  Second call:
        capture — all ~1000 launches of the forward pass go into one graph and those of the backward pass into a
        second one, both in one private memory pool; the activations saved for the backward pass, the inputs, the
        outputs and the incoming prediction gradients are fixed buffers.  From then on a step costs two graph
        launches plus a handful of small eager kernels (input layout, loss, EMA, LARS) on the host."""
        if not self.use_graphs:
            return None
        if self.sync and comm.uses_nccl_for_statistics(self.device):
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
        pool = torch.cuda.graph_pool_handle()
        st.fwd = torch.cuda.CUDAGraph()
        n0 = launch_count[0]
        with torch.cuda.graph(st.fwd, pool=pool, capture_error_mode="thread_local"):
            self.prep_step(mean, True)
            outs, _ = self.forward_lanes(None, lanes, True, rep_bf16_out=[rep_cat[:b], rep_cat[b:], None, None],
                                         x8=[st.inputs[0], st.inputs[1], st.inputs[0], st.inputs[1]])
            st.logits = self.classifier_forward(rep_cat, [outs[0][0], outs[1][0]])
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
        st.pool = pool
        return st

    # classifier (stop-grad input; main.py:250-252)
    def classifier_forward(self, rep_cat_b, reps_f32=None):
        u = self.cls
        flat = self.theta
        bias = flat[u.b_off:u.b_off + u.cout]
        if self.T and reps_f32 is not None:
            pl = torch.cat([ops.split_planes(r, self.T)[0] for r in reps_f32], 0)
            return ops.linear_fprop(pl, self.s_online.w[u.idx], bias=bias, out_fp32=True)
        return ops.linear_fprop(rep_cat_b, self.w_online.wf[u.idx], bias=bias, out_fp32=True)

    def classifier_backward(self, rep_cat_b, d_logits):
        self.notify_backward()
        u = self.cls
        d = d_logits.contiguous().float()
        ops.col_sum(d, self._gview(u.b_off, u.cout))
        # any class count: the bf16 gradient gets a 16-byte row pitch, the GEMM reads only the first `cout` columns
        db = ops.cast_bf16(d) if u.cout % 8 == 0 else ops.cast_bf16_pitched(d, (u.cout + 7) // 8 * 8)
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
