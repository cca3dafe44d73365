"""GPU: the BYOL paper's loss (objective.loss_function(..., variant="byol"); loss_rows_* kernels in csrc/optim.cu)
exactly against its fp32 restatement and within stated bounds of float64.

Definition.  r(x) = max(sum_d x_d^2, eps)^(-1/2) with eps = fp32(1e-12), x^ = r(x) x, l(q, z) = sum_d (q^_d - z^_d)^2,
L = (1/B) sum_i [l(q1_i, z2_i) + l(q2_i, z1_i)].  With u = q^ - z^ and delta = [sum q^2 > eps],
dL/dq = (go / B) 2 r(q) (u - delta (q^.u) q^).  A row whose sum of squares is NaN or +inf has r = NaN.

* Exact operands.  Predictions and targets are integers in [-8, 8] times 2^-4, so every per-row sum of squares is exact
  whatever the order (below 2^24 grid units at D = 2048).  What follows is restated in numpy in the kernels' order:
    - loss_rows_fwd_kernel: lane l of a sample's warp takes the float4s l, l + 32, ... of a row in order and adds
      x, y, z, w by FFMA (s = fma(x, x, s)); a butterfly (xor 16, 8, 4, 2, 1) of FADDs adds the lane sums.
      r = 1 / sqrt(max(s, eps)) by the IEEE square root and division (FMNMX, then MUFU.RSQ / MUFU.RCP with their
      correction steps, which round correctly).  Pass 2: q^ = rn(r(q) q), u = rn(q^ - rn(r(z) z)), then l = fma(u, u, l)
      and p = fma(q^, u, p) per element in the same lane order and butterfly.  c = p, or 0 when s(q) <= eps.
    - block slot = sum over the block's 8 samples, in order, of (double)l12 + (double)l21 (fp64, from 0.0).
    - loss_rows_finalize_kernel: lane l adds slots l, l + 32, ... in fp64, a fp64 butterfly, loss = fp32(S / B).
    - loss_rows_bwd_kernel: k = rn(rn(2 go) / B), a = rn(k r(q)), dq = rn(a * fma(-c, q^, u)).
  The kernels write every fp32 operation as an intrinsic (__fmul_rn, __fsub_rn, __fdiv_rn, __fsqrt_rn) or fmaf, so
  `cuobjdump -sass` shows no contraction beyond those fmaf: the FFMAs in the SASS are the explicit ones plus the
  division and square-root sequences.  Loss, the saved scalars and dq1 / dq2 must equal the restatement bit for bit.
* float64 bounds (in units of 2^-24): the loss within LOSS_ULPS of (1/B) sum_i sum_d |u_d| (|q^_d| + |z^_d|) +
  l_i (T + 6), T = the float4s per lane; dq within DQ_ULPS of |a| (|q^| + |z^| + |q^| (T + 9)).
* Row scale invariance, batch-split independence, float64 autograd, run to run and two training-step comparisons.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.exact import NO_EVENTS, byol_kernel_sequence, check_in_fresh_process, expect_bits, expect_within
from tests.util import fma32, gen, ints

pytestmark = pytest.mark.gpu
F32, F64 = torch.float32, torch.float64
f32 = np.float32
EPS = f32(1e-12)
LOSS_ULPS = 16
DQ_ULPS = 16
NAN = float("nan")


# ------------------------------------------------------------------------------------------------------------------
# restatement of the kernels
# ------------------------------------------------------------------------------------------------------------------
def _lanes(x):
    """[B, D] -> [B, T, 32, 4]: element (t, l, c) is component c of float4 l + 32 t; zero padded."""
    b, d = x.shape
    d4 = d // 4
    t = -(-d4 // 32)
    out = np.zeros((b, t * 32, 4), dtype=np.float32)
    out[:, :d4] = x.reshape(b, d4, 4)
    valid = np.zeros((t * 32, 4), dtype=bool)
    valid[:d4] = True
    return out.reshape(b, t, 32, 4), valid.reshape(t, 32, 4)


def _butterfly(v):
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, np.arange(32) ^ o]
    return v[:, 0]


def _rnorm(s):
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        r = f32(1) / np.sqrt(np.maximum(s, EPS))
    return np.where(s < np.inf, r, f32(NAN)).astype(np.float32)


def _pair(q, z):
    """(r(q), r(z), c, l, s(q)) per row of one pair."""
    qa, valid = _lanes(q)
    za, _ = _lanes(z)
    b, t = qa.shape[:2]
    with np.errstate(invalid="ignore", over="ignore"):
        sq, sz = np.zeros((b, 32), np.float32), np.zeros((b, 32), np.float32)
        for i in range(t):
            for c in range(4):
                sq = fma32(qa[:, i, :, c], qa[:, i, :, c], sq)
                sz = fma32(za[:, i, :, c], za[:, i, :, c], sz)
        sq, sz = _butterfly(sq), _butterfly(sz)
        rq, rz = _rnorm(sq), _rnorm(sz)
        l, p = np.zeros((b, 32), np.float32), np.zeros((b, 32), np.float32)
        for i in range(t):
            for c in range(4):
                m = valid[i, :, c]
                qh = rq[:, None] * qa[:, i, :, c]
                u = qh - rz[:, None] * za[:, i, :, c]
                l = np.where(m, fma32(u, u, l), l)
                p = np.where(m, fma32(qh, u, p), p)
        l, p = _butterfly(l), _butterfly(p)
    return rq, rz, np.where(sq > EPS, p, f32(0)).astype(np.float32), l, sq


def restated(q1, q2, z1, z2, go):
    """(loss, saved [B, 8], dq1, dq2) as the kernels compute them, from fp32 numpy operands."""
    b = q1.shape[0]
    a = _pair(q1, z2)
    c = _pair(q2, z1)
    saved = np.stack([a[0], a[1], a[2], a[3], c[0], c[1], c[2], c[3]], 1).astype(np.float32)
    lrow = a[3].astype(np.float64) + c[3].astype(np.float64)
    nb = -(-b // 8)
    part = np.zeros(nb)
    for blk in range(nb):
        s = 0.0
        for v in lrow[8 * blk:8 * blk + 8]:
            s = s + v
        part[blk] = s
    lanes = np.zeros((1, 32))
    for i in range(nb):
        lanes[0, i % 32] = lanes[0, i % 32] + part[i]
    with np.errstate(invalid="ignore"):
        loss = f32(_butterfly(lanes)[0] / b)
        k = (f32(go) * f32(2)) / f32(b)
        dq = []
        for q, z, rq, rz, cc in ((q1, z2, a[0], a[1], a[2]), (q2, z1, c[0], c[1], c[2])):
            qh = rq[:, None] * q
            u = qh - rz[:, None] * z
            dq.append((k * rq)[:, None] * fma32(-cc[:, None], qh, u))
    return loss, saved, dq[0].astype(np.float32), dq[1].astype(np.float32)


def float64_reference(q1, q2, z1, z2, go, b=None):
    """The definition in float64 on the same fp32 operands: (loss, per-pair dict of r, u, q^, z^, c, a, l, dq), with
    eps = fp32(1e-12).  b: the batch size the gradient divides by (default: these rows)."""
    b = q1.shape[0] if b is None else b
    pairs = []
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for q, z in ((q1, z2), (q2, z1)):
            q, z = q.astype(np.float64), z.astype(np.float64)
            sq, sz = (q * q).sum(1), (z * z).sum(1)
            rq, rz = 1 / np.sqrt(np.maximum(sq, float(EPS))), 1 / np.sqrt(np.maximum(sz, float(EPS)))
            qh, zh = rq[:, None] * q, rz[:, None] * z
            u = qh - zh
            c = np.where(sq > float(EPS), (qh * u).sum(1), 0.0)
            a = 2.0 * float(f32(go)) / b * rq
            pairs.append(dict(r=rq, rz=rz, u=u, qh=qh, zh=zh, c=c, a=a, l=(u * u).sum(1),
                              dq=a[:, None] * (u - c[:, None] * qh)))
    return (pairs[0]["l"] + pairs[1]["l"]).mean(), pairs


def check_against_float64(name, loss, saved, dq1, dq2, q1, q2, z1, z2, go, b=None):
    """loss: of these rows; b: the batch size of the launch (default: these rows)."""
    t = -(-q1.shape[1] // 128)
    L, pairs = float64_reference(q1, q2, z1, z2, go, b)
    mag = sum((np.abs(p["u"]) * (np.abs(p["qh"]) + np.abs(p["zh"]))).sum(1) + p["l"] * (t + 6) for p in pairs)
    with np.errstate(invalid="ignore"):
        expect_within(name + " loss vs float64", loss, [L], LOSS_ULPS * 2.0 ** -24 * mag.mean())
    sv = saved.detach().cpu().numpy()
    for j, p in enumerate(pairs):
        expect_within(name + " r(q) vs float64", sv[:, 4 * j], p["r"], 4 * 2.0 ** -24 * np.abs(p["r"]))
        expect_within(name + " r(z) vs float64", sv[:, 4 * j + 1], p["rz"], 4 * 2.0 ** -24 * np.abs(p["rz"]))
    for j, (got, p) in enumerate(((dq1, pairs[0]), (dq2, pairs[1]))):
        qh = np.abs(p["qh"])
        with np.errstate(invalid="ignore"):
            tol = DQ_ULPS * 2.0 ** -24 * np.abs(p["a"])[:, None] * (qh + np.abs(p["zh"]) + qh * (t + 9))
        expect_within("%s dq%d vs float64" % (name, j + 1), got.reshape(-1), p["dq"].reshape(-1),
                      np.nan_to_num(tol.reshape(-1)))


# ------------------------------------------------------------------------------------------------------------------
# exact cases
# ------------------------------------------------------------------------------------------------------------------
K = 4                       # operands on the 2^-4 grid, |x| <= 1/2


def _operands(dev, g, b, d):
    q1 = ints((b, d), dev, g, 8) * 2.0 ** -K
    q2 = ints((b, d), dev, g, 8) * 2.0 ** -K
    # targets correlated with the predictions, as in training: the pair losses stay well inside [0, 4]
    z2 = q1 + ints((b, d), dev, g, 4) * 2.0 ** -K
    z1 = q2 + ints((b, d), dev, g, 4) * 2.0 ** -K
    return [x.float() for x in (q1, q2, z1, z2)]


def _edit_rows(ops_, b, d):
    """Zero, clamped, NaN, inf and overflowing rows (B >= 7); returns {operand index: rows with a non-finite r}."""
    q1, q2, z1, z2 = ops_
    q1[0].zero_()                               # a zero prediction: r = eps^-1/2, delta = 0
    z1[1].zero_()                               # a zero target
    q2[2].zero_(); q2[2, 3] = 2.0 ** -21        # 0 < sum q^2 = 2^-42 <= eps: clamped
    z2[2].zero_(); z2[2, 1] = -2.0 ** -21
    q1[3, d // 2] = NAN                         # only this row's loss and gradient are NaN
    q2[4, 1] = float("inf")
    z1[5, 0] = -float("inf")                    # a non-finite target: its pair's gradient row is NaN
    q1[6] = 1e20 / d ** 0.5                     # finite, norm 1e20: sum of squares overflows to +inf
    return {0: [3, 6], 1: [4, 5]}


def run_loss(q1, q2, z1, z2, go):
    from byol_b200 import ops
    b = q1.shape[0]
    loss = torch.full((1,), NAN, device=q1.device)
    saved = torch.full((b, 8), NAN, device=q1.device)
    ops.loss_rows_fwd(q1, q2, z1, z2, loss, saved)
    dq1, dq2 = torch.full_like(q1, NAN), torch.full_like(q2, NAN)
    gout = None if go is None else torch.full((1,), go, device=q1.device)
    ops.loss_rows_bwd(q1, q2, z1, z2, saved, gout, dq1, dq2)
    return loss, saved, dq1, dq2


CASES = [(b, d, go, edits) for b in (1, 7, 512, 4096) for d in (8, 256, 2048) for go in (0.75, None)
         for edits in ((False, True) if b >= 7 else (False,))]


@pytest.mark.parametrize("b,d,go,edits", CASES)
def test_exact_against_restatement(cuda, b, d, go, edits):
    g = gen(cuda, 1000 * b + d + (7 if go is None else 0) + (1 if edits else 0))
    ops_ = _operands(cuda, g, b, d)
    bad = _edit_rows(ops_, b, d) if edits else {0: [], 1: []}
    loss, saved, dq1, dq2 = run_loss(*ops_, go)
    torch.cuda.synchronize()
    np_ = [x.cpu().numpy() for x in ops_]
    gv = 1.0 if go is None else go
    r_loss, r_saved, r_dq1, r_dq2 = restated(*np_, gv)
    name = "B=%d D=%d go=%s%s" % (b, d, go, " edited" if edits else "")
    expect_bits(name + " loss", loss, [r_loss])
    expect_bits(name + " saved", saved, r_saved)
    expect_bits(name + " dq1", dq1, r_dq1)
    expect_bits(name + " dq2", dq2, r_dq2)
    if edits:
        assert torch.isnan(loss).all()
        for j, dq in enumerate((dq1, dq2)):
            nan_rows = torch.isnan(dq).any(1).nonzero().flatten().tolist()
            assert nan_rows == bad[j], "dq%d: NaN rows %s, expected %s" % (j + 1, nan_rows, bad[j])
            assert torch.isnan(dq[bad[j]]).all(), "a non-finite row's gradient is NaN throughout"
        # the overflowing row must not read as a zero row (r = 0 would give a finite loss and gradient)
        assert torch.isnan(saved[6, 0])
        keep = [i for i in range(b) if i not in (3, 4, 5, 6)]
        check_against_float64(name + " (finite rows)", _mean_of_rows(saved, keep), saved[keep],
                              dq1[keep], dq2[keep], *[x[keep] for x in np_], gv, b=b)
    else:
        check_against_float64(name, loss, saved, dq1, dq2, *np_, gv)


def _mean_of_rows(saved, rows):
    """The loss of a subset of rows, from the per-row pair losses the kernel saved (float64 mean)."""
    s = saved[rows].double()
    return [float((s[:, 3] + s[:, 7]).mean())]


# ------------------------------------------------------------------------------------------------------------------
# scale, batch split, autograd, run to run
# ------------------------------------------------------------------------------------------------------------------
def _randn_operands(dev, seed, b, d):
    g = torch.Generator(device=dev).manual_seed(seed)
    q1, q2 = (torch.randn(b, d, generator=g, device=dev) for _ in range(2))
    z2 = q1 * 0.5 + torch.randn(b, d, generator=g, device=dev) * 0.5
    z1 = q2 * 0.5 + torch.randn(b, d, generator=g, device=dev) * 0.5
    return [q1, q2, z1, z2]


def test_row_scale_invariance(cuda):
    """Scaling one row of q and one of z by 2^k (k in [-20, 20]; every sum stays >= eps and no square goes subnormal)
    leaves the loss bits unchanged and scales that row of dq by exactly 2^-k."""
    b, d = 64, 256
    base = _randn_operands(cuda, 3, b, d)
    assert float(min(x.abs().min() for x in base)) * 2.0 ** -20 > 2.0 ** -63, "a square would go subnormal"
    l0, _, d10, d20 = run_loss(*base, 0.75)
    for k in range(-20, 21):
        i, j = (k + 20) % b, (3 * k + 41) % b
        xs = [x.clone() for x in base]
        xs[0][i] *= 2.0 ** k          # q1 row i
        xs[2][j] *= 2.0 ** -k         # z1 row j (target of q2 row j)
        xs[1][j] *= 2.0 ** k          # q2 row j
        loss, _, dq1, dq2 = run_loss(*xs, 0.75)
        expect_bits("loss, rows scaled by 2^%d" % k, loss, l0)
        want1, want2 = d10.clone(), d20.clone()
        want1[i] *= 2.0 ** -k
        want2[j] *= 2.0 ** -k
        expect_bits("dq1, rows scaled by 2^%d" % k, dq1, want1)
        expect_bits("dq2, rows scaled by 2^%d" % k, dq2, want2)
    print("loss bits and dq scaling exact for k in [-20, 20]")


def test_batch_split_independence(cuda):
    """dq of the whole batch equals 1/2 dq of each half bit for bit; the loss equals the mean of the halves' losses
    within the float64 bound."""
    b, d = 512, 256
    xs = _randn_operands(cuda, 4, b, d)
    loss, saved, dq1, dq2 = run_loss(*xs, 1.0)
    halves = [run_loss(*[x[h * 256:(h + 1) * 256].contiguous() for x in xs], 1.0) for h in (0, 1)]
    torch.cuda.synchronize()
    expect_bits("dq1 of the batch vs its halves", dq1, torch.cat([h[2] for h in halves]) * 0.5)
    expect_bits("dq2 of the batch vs its halves", dq2, torch.cat([h[3] for h in halves]) * 0.5)
    expect_bits("saved of the batch vs its halves", saved, torch.cat([h[1] for h in halves]))
    np_ = [x.cpu().numpy() for x in xs]
    L, pairs = float64_reference(*np_, 1.0)
    mag = sum((np.abs(p["u"]) * (np.abs(p["qh"]) + np.abs(p["zh"]))).sum(1) + p["l"] * 8 for p in pairs)
    mean_halves = (float(halves[0][0]) + float(halves[1][0])) / 2
    tol = LOSS_ULPS * 2.0 ** -24 * mag.mean()
    print("batch loss %.9g, mean of halves %.9g, float64 %.9g, bound %.3g" % (float(loss), mean_halves, L, tol))
    assert abs(float(loss) - mean_halves) <= 2 * tol
    assert abs(float(loss) - L) <= tol


@pytest.mark.parametrize("b,d", [(7, 8), (512, 256), (4096, 256), (64, 2048)])
def test_against_float64_autograd(cuda, b, d):
    from byol_b200.objective import loss_function
    xs = _randn_operands(cuda, 5 + b, b, d)
    q1, q2 = (x.clone().requires_grad_(True) for x in xs[:2])
    loss = loss_function(q1, q2, xs[2], xs[3], variant="byol")
    go = torch.tensor(1.25, device=cuda)
    loss.backward(go)
    r = [x.double().clone().requires_grad_(True) for x in xs]

    def nrm(x):
        return x * torch.rsqrt(torch.clamp((x * x).sum(-1, keepdim=True), min=1e-12))
    ref = (((nrm(r[0]) - nrm(r[3].detach())) ** 2).sum(-1) + ((nrm(r[1]) - nrm(r[2].detach())) ** 2).sum(-1)).mean()
    ref.backward(go.double())
    torch.cuda.synchronize()
    el = abs(float(loss) - float(ref)) / abs(float(ref))
    e1 = float((q1.grad.double() - r[0].grad).abs().max() / r[0].grad.abs().max())
    e2 = float((q2.grad.double() - r[1].grad).abs().max() / r[1].grad.abs().max())
    print("B=%d D=%d: loss %.8g rel err %.2e, dq1 %.2e, dq2 %.2e" % (b, d, float(loss), el, e1, e2))
    assert el < 1e-6 and e1 < 1e-6 and e2 < 1e-6
    assert xs[2].grad is None and xs[3].grad is None


def test_run_to_run(cuda):
    xs = _randn_operands(cuda, 6, 4096, 256)
    a, b = run_loss(*xs, 0.5), run_loss(*xs, 0.5)
    for name, x, y in zip(("loss", "saved", "dq1", "dq2"), a, b):
        expect_bits("run to run " + name, x, y)


def test_bad_arguments(cuda):
    from byol_b200 import ops
    from byol_b200._lib import ByolLibraryError
    xs = [torch.zeros(4, 6, device=cuda) for _ in range(4)]
    with pytest.raises(ByolLibraryError, match="multiple of 4"):
        ops.loss_rows_fwd(*xs, torch.empty(1, device=cuda), torch.empty(4, 8, device=cuda))
    with pytest.raises(ByolLibraryError, match="multiple of 4"):
        ops.loss_rows_bwd(*xs, torch.empty(4, 8, device=cuda), None, xs[0].clone(), xs[1].clone())
    with pytest.raises(ValueError):
        ops.loss_rows_fwd(*[torch.zeros(4, 8, device=cuda) for _ in range(3)], torch.zeros(4, 16, device=cuda),
                          torch.empty(1, device=cuda), torch.empty(4, 8, device=cuda))
    # a misaligned view is copied by the autograd Function, not rejected
    from byol_b200.objective import loss_function
    big = torch.randn(4 * 8 + 1, device=cuda)
    q = big[1:].view(4, 8)
    assert q.data_ptr() % 16 != 0
    ref = loss_function(q.clone(), q.clone(), q.clone() * 2, q.clone() * 2, variant="byol")
    assert torch.equal(loss_function(q, q, q * 2, q * 2, variant="byol"), ref)


# ------------------------------------------------------------------------------------------------------------------
# which kernels each variant launches
# ------------------------------------------------------------------------------------------------------------------
VARIANT_KERNELS = {"byol": ["loss_rows_fwd_kernel", "loss_rows_finalize_kernel", "loss_rows_bwd_kernel"],
                   "reference": ["loss_fwd_partial_kernel", "loss_finalize_kernel", "loss_bwd_kernel"]}


def _check_launches():
    from byol_b200.objective import loss_function
    dev = torch.device("cuda:0")
    xs = _randn_operands(dev, 7, 512, 256)

    def call(variant):
        q1, q2 = (x.clone().requires_grad_(True) for x in xs[:2])
        loss_function(q1, q2, xs[2], xs[3], variant=variant).backward()
        torch.cuda.synchronize()
    for v in VARIANT_KERNELS:
        call(v)
    order = ["byol", "reference", "byol"]
    got = byol_kernel_sequence([lambda v=v: call(v) for v in order])
    if not got:
        print(NO_EVENTS)
        return
    want = [k for v in order for k in VARIANT_KERNELS[v]]
    assert got == want, "launched %s, expected %s" % (got, want)
    print("both variants launched exactly their kernels: %s" % got)


def test_variants_launch_their_kernels(cuda):
    """variant="byol" launches the three loss_rows kernels and nothing else; the default launches the reference
    loss's three.  In a fresh Python process, as tests/test_gpu_optim_exact.py does."""
    check_in_fresh_process(__name__)


# ------------------------------------------------------------------------------------------------------------------
# training steps
# ------------------------------------------------------------------------------------------------------------------
def _cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def test_training_step_fp32_against_oracle(cuda):
    """One fp32 (forward and backward) ResNet-18 step at 8 x 64^2 with the paper's loss against the CPU oracle's step
    with it (tests/paper_loss_oracle.py): the BYOL loss within 1e-3 relative, the gradient norm within 10 % and the
    parameter update in direction and size."""
    from byol_b200.model import BYOL
    from byol_b200.objective import loss_function
    from byol_b200 import wiring
    from oracle import byol_oracle as O
    from tests.paper_loss_oracle import OracleBYOL
    seed, b, r, lr, total = 9, 8, 64, 0.3, 10
    torch.manual_seed(seed)
    model = BYOL(512, 256, 1000, total, arch="resnet18", precision="fp32", backward_precision="fp32")
    params, buffers = O.init_reference_state("resnet18", seed)
    theta0 = torch.cat([p.reshape(-1) for p in params.values()])
    assert torch.equal(torch.nn.utils.parameters_to_vector(model.parameters()).detach(), theta0)
    model = model.cuda().train()
    oracle = OracleBYOL("resnet18", params, buffers, total)
    opt = wiring.LARS(torch.optim.SGD(wiring.add_weight_decay(model, 1e-6), lr=lr, momentum=0.9), eps=0.0)
    g = torch.Generator().manual_seed(10)
    a1, a2 = torch.rand(b, 3, r, r, generator=g), torch.rand(b, 3, r, r, generator=g)
    lab = torch.randint(0, 1000, (b,), generator=g)
    out = model(a1.cuda(), a2.cuda())
    byol = loss_function(out["online_prediction1"], out["online_prediction2"], out["target_projection1"],
                         out["target_projection2"], variant="byol")
    ce = F.cross_entropy(out["linear_preds"], torch.cat([lab, lab]).cuda())
    opt.zero_grad()
    (byol + ce).backward()
    gflat = model._engine.grad.detach().clone()
    opt.step()
    torch.cuda.synchronize()
    ref = oracle.train_step(a1, a2, lab, lr, loss="byol")
    gref = torch.cat([x.reshape(-1) for x in ref["grads"].values()])
    ratio = float(gflat.double().norm().cpu() / gref.double().norm())
    upd, upd_ref = model._engine.theta.cpu() - theta0, oracle.flat_params() - theta0
    uc, ur = _cos(upd, upd_ref), float(upd.double().norm() / upd_ref.double().norm())
    print("byol loss %.7f oracle %.7f; gradient norm ratio %.4f cosine %.5f; update cosine %.5f norm ratio %.4f" % (
        byol.item(), ref["byol_loss"].item(), ratio, _cos(gflat, gref), uc, ur))
    assert 0.0 <= byol.item() <= 8.0
    assert abs(byol.item() - ref["byol_loss"].item()) < 1e-3 * abs(ref["byol_loss"].item())
    assert 0.9 < ratio < 1.1
    assert uc > 0.99 and 0.9 < ur < 1.1


def test_graphed_steps_match_eager(cuda):
    """20 bf16 ResNet-18 steps through wiring.train_step(..., loss_variant="byol"), CUDA-graphed and eager: losses and
    parameters bit-identical, every BYOL loss finite and in [0, 8]."""
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    b, r = 8, 64
    g = torch.Generator().manual_seed(12)
    batches = [(torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda(),
                torch.randint(0, 1000, (b,), generator=g).cuda()) for _ in range(4)]
    res = {}
    for mode in ("eager", "graph"):
        torch.manual_seed(13)
        model = BYOL(512, 256, 1000, 40, arch="resnet18").cuda().train()
        model._engine.use_graphs = mode == "graph"
        opt = wiring.build_optimizer(model, global_batch_size=256)
        stats = [wiring.train_step(model, opt, *batches[s % 4], loss_variant="byol") for s in range(20)]
        torch.cuda.synchronize()
        captured = [v for v in model._engine.graphs.values() if v != "warm"]
        assert (len(captured) == 1) == (mode == "graph")
        res[mode] = (torch.stack([s["loss_mean"] for s in stats]), torch.stack([s["byol_loss_mean"] for s in stats]),
                     model._engine.theta.clone())
        model = opt = None
    byol = res["eager"][1].cpu()
    print("byol losses %s" % byol.tolist())
    assert torch.isfinite(byol).all() and bool(((byol >= 0) & (byol <= 8)).all())
    for name, x, y in zip(("loss", "byol loss", "theta"), res["eager"], res["graph"]):
        assert torch.equal(x, y), "%s differs between graphed and eager steps" % name
