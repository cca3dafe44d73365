"""LARS — drop-in for /root/reference/optimizers/lars.py (same class name, constructor, proxy API).

``step()`` replaces the reference's per-parameter Python loop (~7 launches and 2 host syncs per tensor,
lars.py:96-111) and the wrapped ``torch.optim.SGD.step`` (lars.py:121) by one fused multi-tensor pass pair
(`byol_lars_sgd_step`): per-tensor ||p||, ||g + wd p||, then g' = (g + wd p) * trust*||p||/(||g||+eps),
buf = momentum*buf + g', p -= lr*buf — no host synchronisation.
"""
import torch
from torch.optim.optimizer import Optimizer

from . import ops

__all__ = ['LARS']

_CHUNK = 32768


def chunk_table(lengths, dev):
    """The work items of the multi-tensor kernels (byol_lars_sgd_step, byol_sgd_nesterov_step) over tensors of the
    given lengths: chunk j covers elements [chunk_start[j], chunk_start[j] + chunk_len[j]) of tensor chunk_tensor[j],
    chunks of at most 32 768 elements; tensor t's chunks are [tensor_first_chunk[t], tensor_first_chunk[t + 1])."""
    cs, cl, ct, first = [], [], [], []
    for t, n in enumerate(lengths):
        first.append(len(cs))
        for s in range(0, n, _CHUNK):
            cs.append(s)
            cl.append(min(_CHUNK, n - s))
            ct.append(t)
    first.append(len(cs))
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)
    return {"chunk_start": torch.tensor(cs, dtype=torch.int64, device=dev), "chunk_len": i32(cl),
            "chunk_tensor": i32(ct), "tensor_first_chunk": i32(first)}


class LARS(Optimizer):
    """Wraps a ``torch.optim.SGD`` (the reference wraps arbitrary optimizers; its configurations only ever use
    SGD / SGD-momentum, main.py:316,332-340).  Param groups may carry the ``'ignore'`` flag set by
    ``helpers.layers.add_weight_decay`` (lars.py:88,99-100)."""

    def __init__(self, optimizer, eps=1e-8, trust_coef=0.001):
        if eps < 0.0:
            raise ValueError('invalid epsilon value: , %f' % eps)
        if trust_coef < 0.0:
            raise ValueError("invalid trust coefficient: %f" % trust_coef)
        if not isinstance(optimizer, torch.optim.SGD):
            raise NotImplementedError("byol_b200.LARS fuses LARS with torch.optim.SGD only, got %r" % type(optimizer))
        self.optim = optimizer
        self.eps = eps
        self.trust_coef = trust_coef
        self._table = None
        self._key = None

    def __getstate__(self):
        return (self.optim, {'eps': self.eps, 'trust_coef': self.trust_coef})

    def __setstate__(self, state):
        self.optim, lars_dict = state
        self.eps = lars_dict['eps']
        self.trust_coef = lars_dict['trust_coef']
        self._table, self._key = None, None

    def __repr__(self):
        return '%s(%r)' % (self.__class__.__name__, self.optim)

    @property
    def param_groups(self):
        return self.optim.param_groups

    @property
    def state(self):
        return self.optim.state

    def state_dict(self):
        return self.optim.state_dict()

    def load_state_dict(self, state_dict):
        self.optim.load_state_dict(state_dict)
        self._table, self._key = None, None

    def zero_grad(self, set_to_none=True):
        self.optim.zero_grad(set_to_none=set_to_none)

    def add_param_group(self, param_group):
        self.optim.add_param_group(param_group)
        self._table, self._key = None, None

    # ------------------------------------------------------------------------------------------
    def _build(self, entries, dev):
        """entries: list of (param, group).  One flat momentum buffer; per-param views live in optimizer state
        under the same key torch.optim.SGD uses ('momentum_buffer'), so state_dict() stays compatible."""
        total = sum(p.numel() for p, _ in entries)
        use_mom = any(g['momentum'] != 0 for _, g in entries)
        flat_m = torch.zeros(total, dtype=torch.float32, device=dev) if use_mom else None
        m_ptrs = []
        off = 0
        for p, g in entries:
            n = p.numel()
            if use_mom:
                view = flat_m[off:off + n].view(p.shape)
                st = self.optim.state[p]
                old = st.get('momentum_buffer')
                if old is not None:
                    view.copy_(old)
                st['momentum_buffer'] = view
                m_ptrs.append(view.data_ptr())
            off += n
        i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=dev)
        T = len(entries)
        table = chunk_table([p.numel() for p, _ in entries], dev)
        table.update({
            "p_ptrs": i64([p.data_ptr() for p, _ in entries]), "g_ptrs": i64([p.grad.data_ptr() for p, _ in entries]),
            "m_ptrs": i64(m_ptrs) if use_mom else None, "wd": torch.zeros(T, device=dev),
            "lr": torch.zeros(T, device=dev), "ignore": torch.zeros(T, dtype=torch.int32, device=dev),
            "partial": torch.zeros(2 * table["chunk_start"].numel(), dtype=torch.float64, device=dev),
            "flat_m": flat_m, "hyper": None, "ptrs": None,
        })
        return table

    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        entries = [(p, g) for g in self.optim.param_groups for p in g['params'] if p.grad is not None]
        if not entries:
            return loss
        momentum = entries[0][1]['momentum']
        for _, g in entries:
            if g.get('dampening', 0) != 0 or g.get('nesterov', False) or g.get('maximize', False) \
                    or g['momentum'] != momentum:
                raise NotImplementedError("byol_b200.LARS: dampening / nesterov / maximize / per-group momentum")
        dev = entries[0][0].device
        if dev.type != 'cuda':
            raise RuntimeError("byol_b200.LARS.step needs CUDA parameters (no CPU path)")
        key = tuple(id(p) for p, _ in entries)
        if self._table is None or self._key != key:
            for p, _ in entries:
                # the kernel reads raw fp32 storage: anything else would be silently reinterpreted
                if p.dtype != torch.float32 or p.grad.dtype != torch.float32 or not p.is_contiguous() \
                        or not p.grad.is_contiguous() or p.device != dev or p.grad.device != dev:
                    raise NotImplementedError("byol_b200.LARS: parameters and gradients must be contiguous fp32 "
                                              "tensors on one CUDA device (got %s / %s)" % (p.dtype, p.grad.dtype))
            self._table, self._key = self._build(entries, dev), key
        tb = self._table
        ptrs = ([p.data_ptr() for p, _ in entries], [p.grad.data_ptr() for p, _ in entries])
        if tb["ptrs"] != ptrs:
            tb["p_ptrs"].copy_(torch.tensor(ptrs[0], dtype=torch.int64), non_blocking=False)
            tb["g_ptrs"].copy_(torch.tensor(ptrs[1], dtype=torch.int64), non_blocking=False)
            tb["ptrs"] = ptrs
        # ignore is None (group not made by add_weight_decay) => lars.py:100 skips the scaling too
        hyper = ([float(g['weight_decay']) for _, g in entries], [float(g['lr']) for _, g in entries],
                 [0 if (g.get('ignore', None) is not None and not g['ignore']) else 1 for _, g in entries])
        if tb["hyper"] != hyper:
            tb["wd"].copy_(torch.tensor(hyper[0], dtype=torch.float32))
            tb["lr"].copy_(torch.tensor(hyper[1], dtype=torch.float32))
            tb["ignore"].copy_(torch.tensor(hyper[2], dtype=torch.int32))
            tb["hyper"] = hyper
        # momentum buffers start at zero, so "buf = momentum*buf + g" reproduces SGD's first-step "buf = g" exactly
        ops.lars_sgd_step(tb, self.trust_coef, self.eps, momentum, first_step=False)
        return loss
