"""GPU: semi-supervised evaluation (byol_b200.finetune) and its kernel, byol_sgd_nesterov_step (csrc/optim.cu).

* The Nesterov-SGD kernel is bit-exact over 20 steps against the fp32 restatement of its operation order, on ragged and
  misaligned ranges, close to torch.optim.SGD(nesterov=True), and leaves the gradients zeroed.
* The encoder gradient of one fine-tune step is bit-equal to the gradient the BYOL training step computes when the
  same d_rep enters its online_representation1, with stored and with recomputed activations.
* One step agrees with fp32 torch autograd (loss, classifier gradients, running statistics), and its encoder gradient
  as well as torch's bf16 autocast does.
* A run gives the same bits alone or in a sweep, and on every call.
* Fine-tuning a random ResNet-18 separates colour / stripe classes; an lr = 0 run does not move.
* finetune_accuracy runs both subset modes and the target network, never selects a diverged run, and leaves the model
  and graphed training untouched.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from tests import linear_oracle as O
from tests.image_folder import loader_kwargs, make_image_folder

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float(a @ b / (a.norm() * b.norm()))


# ---- the kernel ----
def test_sgd_nesterov_kernel_bit_exact_over_20_steps(cuda):
    from byol_b200 import ops
    from byol_b200.lars import chunk_table
    from byol_b200.linear_eval import cosine_factor
    rng = np.random.default_rng(0)
    # ragged lengths (not multiples of 4, one over two chunks) and one range starting off the 16-byte phase
    lengths, offsets = [5, 2 * 32768 + 3, 37, 4096], [0, 8, 1, 3]
    lrs, wds, mu = [0.1, 0.05, 0.0, 0.3], [0.0, 1e-3, 1e-2, 5e-4], 0.9
    store = [torch.zeros(3, off + n + 8, dtype=torch.float32, device=cuda) for off, n in zip(offsets, lengths)]
    p = [s[0, off:off + n] for s, off, n in zip(store, offsets, lengths)]
    g = [s[1, off:off + n] for s, off, n in zip(store, offsets, lengths)]
    m = [s[2, off:off + n] for s, off, n in zip(store, offsets, lengths)]
    w0 = [rng.standard_normal(n).astype(np.float32) for n in lengths]
    for t, v in zip(p, w0):
        t.copy_(torch.from_numpy(v))
    i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=cuda)
    table = chunk_table(lengths, cuda)
    table.update({"p_ptrs": i64([t.data_ptr() for t in p]), "g_ptrs": i64([t.data_ptr() for t in g]),
                  "m_ptrs": i64([t.data_ptr() for t in m]),
                  "lr": torch.tensor(lrs, dtype=torch.float32, device=cuda),
                  "wd": torch.tensor(wds, dtype=torch.float32, device=cuda)})
    w, buf = [v.copy() for v in w0], [np.zeros(n, np.float32) for n in lengths]
    tp = [torch.nn.Parameter(torch.from_numpy(v.copy()).to(cuda)) for v in w0]
    opt = torch.optim.SGD([{"params": [t], "lr": 0.0, "weight_decay": wd} for t, wd in zip(tp, wds)], lr=0.0,
                          momentum=mu, nesterov=True)
    sentinel = [s.clone() for s in store]
    for step in range(20):
        scale = cosine_factor(step, 20)
        grads = [(rng.standard_normal(n) * 0.01).astype(np.float32) for n in lengths]
        for t, v in zip(g, grads):
            t.copy_(torch.from_numpy(v))
        ops.sgd_nesterov_step(table, scale, mu)
        for k in range(len(lengths)):
            lr_k = np.float32(np.float32(lrs[k]) * scale)
            w[k], buf[k] = O.sgd(w[k], buf[k], grads[k], lr_k, np.float32(wds[k]), mu)
            assert np.array_equal(p[k].cpu().numpy().view(np.int32), w[k].view(np.int32)), (step, k)
            assert np.array_equal(m[k].cpu().numpy().view(np.int32), buf[k].view(np.int32)), (step, k)
            assert not g[k].cpu().numpy().any(), (step, k)
            opt.param_groups[k]["lr"] = float(lr_k)
            tp[k].grad = torch.from_numpy(grads[k]).to(cuda)
        opt.step()
    for s, s0, off, n in zip(store, sentinel, offsets, lengths):      # nothing outside the ranges was written
        assert torch.equal(s[:, :off], s0[:, :off]) and torch.equal(s[:, off + n:], s0[:, off + n:])
    assert np.array_equal(w[2], w0[2])                                 # lr = 0: the init, exactly
    for k in range(len(lengths)):
        theirs = tp[k].detach().cpu().numpy()
        assert np.abs(w[k] - theirs).max() <= 1e-6 * max(np.abs(theirs).max(), 1e-3), k


# ---- one step against the BYOL step and against torch ----
def _model(arch, d, classes=10):
    from byol_b200.model import BYOL
    torch.manual_seed(21)
    return BYOL(d, 64, classes, 10, arch=arch, head_latent_size=128).cuda().train()


NETS = [("resnet18", 512, 12), ("resnet:bottleneck:1,1,1,1", 2048, 8)]


@pytest.mark.parametrize("recompute", [False, True])
@pytest.mark.parametrize("arch,d,b", NETS)
def test_encoder_gradient_equals_the_byol_step(cuda, arch, d, b, recompute):
    """The fine-tune step hands its bf16 d_rep to the average-pool backward's bf16 input; the BYOL step gets the same
    values as fp32.  The kernel adds either to 0.f, so both walk the same kernels on the same operands: equal bits."""
    from byol_b200.finetune import FineTune
    model = _model(arch, d)
    ft = FineTune(model, 5, 0.1, seed=1)
    for eng in (ft.eng, model._engine):
        eng._mem_budget = 0 if recompute else 1 << 62
    g = torch.Generator().manual_seed(5)
    x = torch.rand(b, 3, 64, 64, generator=g).cuda()
    lab = torch.randint(0, 5, (b,), generator=g).cuda()
    _, d_rep = ft.gradients(x, lab)
    n_enc = sum(p.numel() for p in ft.model.base_network.parameters())
    nblk = len(ft.eng.blocks)
    assert ft.eng.recompute_plan(b, 64, 64, 1, False, False) == (frozenset(range(nblk)) if recompute else frozenset())
    out = model(x, torch.rand(b, 3, 64, 64, generator=g).cuda())
    out["online_representation1"].backward(d_rep.float())
    torch.cuda.synchronize()
    assert model._engine.recompute_plan(b, 64, 64) == (frozenset(range(nblk)) if recompute else frozenset())
    mine, theirs = ft.eng.grad[:n_enc], model._engine.grad[:n_enc]
    assert mine.abs().max() > 0
    assert torch.equal(_bits(mine), _bits(theirs))


def _ref_grads(arch, state, x, W, bias, lab, autocast):
    """(loss, gradients of the encoder parameters, the module after the step) of torch autograd on an fp32 copy of the
    encoder in train mode; autocast: the convolutions in bf16 under torch.autocast."""
    from byol_b200.model import _resnet
    ref = torch.nn.Sequential(*list(_resnet(arch).children())[:-1]).cuda().train()
    ref.load_state_dict(state)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        f = ref(x).flatten(1).float()
    loss = Fn.cross_entropy(f @ W.t() + bias, lab)
    loss.backward()
    return loss.item(), [p.grad for p in ref.parameters()], ref


@pytest.mark.parametrize("arch,d,b", NETS)
def test_step_against_fp32_autograd(cuda, arch, d, b):
    """Loss within 1e-2 of fp32 autograd.  The gradients and running statistics are held to what torch's own bf16
    autocast reaches against fp32 on the same step, since a bf16 forward already moves the features by a few percent
    on these random-init nets: the encoder gradient's cosine sits at 0.92-0.93 for the whole encoder and >= 0.915 for
    every convolution for both (measured on an H100 for 8-64 images at 64 and 128 px), so 0.99 / 0.95 would be out of
    reach for any bf16-operand backward.  The classifier gradients and the running statistics are within twice
    autocast's largest error (and always within 2^-7 of the largest value)."""
    from byol_b200.finetune import FineTune
    model = _model(arch, d)
    C = 5
    ft = FineTune(model, C, 0.1, seed=2)
    state = {k: v.clone() for k, v in ft.model.base_network.state_dict().items()}
    W = ft.classifier_weight.clone().requires_grad_(True)
    bias = ft.classifier_bias.clone().requires_grad_(True)
    tracked = [m.num_batches_tracked.item() for m in ft.model.base_network.modules() if hasattr(m, "num_batches_tracked")]
    g = torch.Generator().manual_seed(6)
    x = torch.rand(b, 3, 64, 64, generator=g).cuda()
    lab = torch.randint(0, C, (b,), generator=g).cuda()
    loss_sum, _ = ft.gradients(x, lab)
    xb = x.bfloat16().float()
    ref_loss, ref_g, ref = _ref_grads(arch, state, xb, W, bias, lab, False)
    cls_g = (W.grad.clone(), bias.grad.clone())
    W.grad = bias.grad = None
    _, ac_g, ref_ac = _ref_grads(arch, state, xb, W, bias, lab, True)
    ac_cls_g = (W.grad.clone(), bias.grad.clone())
    torch.cuda.synchronize()
    loss = loss_sum.item() / b
    assert abs(loss - ref_loss) <= 1e-2 * abs(ref_loss), (loss, ref_loss)
    eng = ft.eng
    n_enc = sum(p.numel() for p in ref.parameters())
    whole, whole_ac = _cos(eng.grad[:n_enc], torch.cat([t.reshape(-1) for t in ref_g])), \
        _cos(torch.cat([t.reshape(-1) for t in ac_g]), torch.cat([t.reshape(-1) for t in ref_g]))
    print("%s: whole-encoder gradient cosine %.4f (torch autocast %.4f)" % (arch, whole, whole_ac))
    assert whole >= 0.9 and whole >= whole_ac - 0.01
    off = 0
    for (name, p), t, t_ac in zip(ref.named_parameters(), ref_g, ac_g):
        if p.dim() == 4:
            c, c_ac = _cos(eng.grad[off:off + p.numel()], t), _cos(t_ac, t)
            assert c >= 0.9 and c >= c_ac - 0.01, (name, c, c_ac)
        off += p.numel()
    def close(mine, theirs, ac, what):
        err, err_ac = float((mine - theirs).abs().max()), float((ac - theirs).abs().max())
        assert err <= max(2 * err_ac, 2 ** -7 * float(theirs.abs().max())) + 1e-6, (what, err, err_ac)

    u = eng.cls
    close(eng.grad[u.w_off:u.w_off + u.w_numel].view(C, d), cls_g[0], ac_cls_g[0], "classifier weight")
    close(eng.grad[u.b_off:u.b_off + C], cls_g[1], ac_cls_g[1], "classifier bias")
    stats = lambda m: [(n, t) for n, t in m.state_dict().items() if "running_" in n]
    for (n, a), (_, r), (_, r_ac) in zip(stats(ft.model.base_network), stats(ref), stats(ref_ac)):
        close(a, r, r_ac, n)
    after = [m.num_batches_tracked.item() for m in ft.model.base_network.modules() if hasattr(m, "num_batches_tracked")]
    assert after == [t + 1 for t in tracked]


# ---- runs are independent and reproducible ----
def test_run_alone_equals_run_in_sweep(cuda):
    from byol_b200.finetune import FineTune
    model = _model("resnet18", 512)
    g = torch.Generator().manual_seed(7)
    batches = [(torch.rand(8, 3, 64, 64, generator=g).cuda(), torch.randint(0, 4, (8,), generator=g).cuda())
               for _ in range(3)]

    def train(lrs):
        runs = [FineTune(model, 4, lr, 1e-4, seed=3) for lr in lrs]
        for t, (x, lab) in enumerate(batches):
            for r in runs:
                r.step(x, lab, 1.0 - t / 3)
        torch.cuda.synchronize()
        return [(r.eng.theta.clone(), [t.clone() for t in r.model.base_network.buffers()]) for r in runs]

    sweep = train([0.1, 0.05, 0.02])
    alone = train([0.05])[0]
    again = train([0.05])[0]
    for a, bb in ((sweep[1], alone), (alone, again)):
        assert torch.equal(_bits(a[0]), _bits(bb[0]))
        assert all(torch.equal(x, y) for x, y in zip(a[1], bb[1]))
    assert not torch.equal(sweep[0][0], sweep[1][0])


# ---- learning ----
def _stripes_folder(root, seed):
    """Four visibly different classes: reddish, greenish and bluish images, and black / white horizontal stripes."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    for split, n in (("train", 24), ("valid", 6), ("test", 8)):
        for c in range(4):
            os.makedirs(os.path.join(root, split, "k%d" % c), exist_ok=True)
            for i in range(n):
                h, w = rng.integers(56, 96, size=2)
                img = rng.integers(0, 60, size=(h, w, 3)).astype(np.uint8)
                if c < 3:
                    img[..., c] = rng.integers(180, 255)
                else:
                    img[(np.arange(h) // 6) % 2 == 0] = 230
                Image.fromarray(img).save(os.path.join(root, split, "k%d" % c, "%s%d.JPEG" % (split, i)), quality=90)


def test_finetuning_a_random_encoder_separates_classes(cuda, tmp_path):
    from byol_b200.data import get_loader
    from byol_b200.finetune import finetune_accuracy
    _stripes_folder(tmp_path, seed=1)
    loader = get_loader(**loader_kwargs(tmp_path))
    model = _model("resnet18", 512, classes=4)
    theta0 = torch.cat([p.detach().reshape(-1) for p in model.base_network.parameters()])
    acc = finetune_accuracy(model, loader, label_fraction=1.0, epochs=6, batch_size=16, lrs=(0.1, 0.02, 0.0))
    print(acc)
    assert acc["labelled"] == 96
    assert acc["lr"] != 0.0 and acc["finetune_top1"] >= 90.0, acc
    assert acc["runs"][2]["test_top1"] <= 50.0, acc                    # lr = 0: chance level for 4 classes
    assert torch.equal(theta0, torch.cat([p.detach().reshape(-1) for p in model.base_network.parameters()]))


# ---- finetune_accuracy on the image folder ----
def test_finetune_accuracy_on_image_folder(cuda, tmp_path):
    from byol_b200.data import get_loader
    from byol_b200.finetune import finetune_accuracy
    make_image_folder(tmp_path, seed=6)
    loader = get_loader(**loader_kwargs(tmp_path))
    model = _model("resnet18", 512, classes=loader.output_size)
    kw = dict(epochs=3, batch_size=2, lrs=(1e6, 0.1, 0.0), weight_decays=(0.0, 1e-4))
    acc = finetune_accuracy(model, loader, label_fraction=0.5, **kw)
    assert set(acc) == {"finetune_top1", "finetune_top5", "lr", "weight_decay", "labelled", "runs"}
    assert acc["labelled"] == 6
    assert [(r["lr"], r["weight_decay"]) for r in acc["runs"]] == [(1e6, 0.0), (1e6, 1e-4), (0.1, 0.0), (0.1, 1e-4),
                                                                   (0.0, 0.0), (0.0, 1e-4)]
    for r in acc["runs"]:
        assert set(r) == {"lr", "weight_decay", "val_top1", "val_top5", "finite", "test_top1", "test_top5"}
        assert 0.0 <= r["val_top1"] <= r["val_top5"] <= 100.0
        assert 0.0 <= r["test_top1"] <= r["test_top5"] <= 100.0
    assert not acc["runs"][0]["finite"] and not acc["runs"][1]["finite"], acc
    assert acc["lr"] != 1e6 and 0.0 <= acc["finetune_top1"] <= acc["finetune_top5"] <= 100.0
    assert acc == finetune_accuracy(model, loader, label_fraction=0.5, **kw)
    names = ["a0.JPEG", "a1.JPEG", "b0.JPEG", "b1.JPEG", "c0.JPEG", "c1.jpeg"]
    sub = finetune_accuracy(model, loader, subset=names, epochs=2, batch_size=3, lrs=(0.1,))
    assert sub["labelled"] == 6 and len(sub["runs"]) == 1 and sub["runs"][0]["finite"]
    target = finetune_accuracy(model, loader, label_fraction=0.5, network="target", epochs=1, batch_size=2,
                               lrs=(0.1, 0.05))
    assert 0.0 <= target["finetune_top1"] <= target["finetune_top5"] <= 100.0 and len(target["runs"]) == 2


def test_training_is_undisturbed(cuda, tmp_path):
    """Graphed training steps give the same bits with finetune_accuracy calls between steps and between a step's
    forward and backward; the calls change no weight, running statistic, num_batches_tracked, EMA or EMA step."""
    from byol_b200 import wiring
    from byol_b200.data import get_loader
    from byol_b200.finetune import finetune_accuracy
    from byol_b200.model import BYOL
    from tests.test_gpu_knn import _bn_state, _step
    make_image_folder(tmp_path, seed=2)
    loader = get_loader(**loader_kwargs(tmp_path))
    arch, b, r = "resnet:bottleneck:1,1,1,1", 8, 64
    g = torch.Generator().manual_seed(3)
    batches = [(torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda(),
                torch.randint(0, 10, (b,), generator=g).cuda()) for _ in range(4)]
    res = {}
    for mode in ("plain", "probed"):
        torch.manual_seed(11)
        model = BYOL(2048, 64, 10, 20, arch=arch, head_latent_size=128).cuda().train()
        opt = wiring.build_optimizer(model, global_batch_size=256)

        def probe_calls():
            before, step = _bn_state(model), model.target_network.step
            theta = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
            mean = model.target_network.mean.clone()
            for network in ("online", "target"):
                acc = finetune_accuracy(model, loader, label_fraction=0.5, epochs=1, batch_size=4, lrs=(0.1,),
                                        network=network)
                assert 0.0 <= acc["finetune_top1"] <= acc["finetune_top5"] <= 100.0
            after = _bn_state(model)
            assert all(torch.equal(x, y) for x, y in zip(before, after)) and model.target_network.step == step
            assert torch.equal(theta, torch.cat([p.detach().reshape(-1) for p in model.parameters()]))
            assert torch.equal(mean, model.target_network.mean)

        hook = probe_calls if mode == "probed" else None
        losses = []
        for bt in batches:
            losses.append(_step(model, opt, *bt, hook=hook))
            if hook is not None:
                hook()
        torch.cuda.synchronize()
        assert len([v for v in model._engine.graphs.values() if v != "warm"]) == 1     # steps 2-4 were graphed
        res[mode] = {"loss": torch.stack(losses), "theta": model._engine.theta.clone(),
                     "target": model.target_network.mean.clone(), "bn": _bn_state(model),
                     "step": model.target_network.step}
        model = opt = None
    for key in ("loss", "theta", "target"):
        assert torch.equal(res["plain"][key], res["probed"][key]), key
    assert all(torch.equal(x, y) for x, y in zip(res["plain"]["bn"], res["probed"]["bn"]))
    assert res["plain"]["step"] == res["probed"]["step"]
