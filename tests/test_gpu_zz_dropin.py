"""GPU: the byol_b200 classes dropped into the UNMODIFIED reference's own step loop.

`oracle/_ref/` holds the reference's own modules, byte-compiled by build() (oracle/build_ref.py; git-ignored).  The test
imports that `main` with the import shims of oracle/ref_shims for its three missing submodules, rebinds the four
names INTEGRATION.md tells a maintainer to re-import (BYOL, loss_function, LARS, DistributedDataParallelPassthrough)
and then calls the reference's `main.execute_graph` (/root/reference/main.py:559-662) — its loop, its
F.cross_entropy, its metrics.topk, its optimizer.zero_grad()/backward()/step() order — on cuda:0.  The returned
losses must follow the golden values the stock reference produced on the same seeds (tests/golden/*.npz).
"""
import functools
import os
import sys

import numpy as np
import pytest
import torch

from tests.test_oracle_golden import _batches, load_case

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def _import_reference_main(arch, rep, b, r):
    if not os.path.exists(os.path.join(REF, "main.pyc")):
        pytest.skip("oracle/_ref has no compiled reference (build() found no reference checkout)")
    for m in [k for k in sys.modules if k in ("main", "objective") or k.startswith(("optimizers", "helpers", "datasets", "tree"))]:
        del sys.modules[m]
    argv, path = sys.argv, list(sys.path)
    sys.argv = ["main.py", "--arch=%s" % arch, "--representation-size=%d" % rep, "--num-replicas=1",
                "--batch-size=%d" % b, "--image-size-override=%d" % r, "--debug-step"]
    sys.path[:0] = [REF, os.path.join(ROOT, "oracle", "ref_shims")]
    try:
        import main   # argparse runs at import (main.py:119); cuda is on by default on a GPU box
    finally:
        sys.argv = argv
        sys.path[:] = path
    assert os.path.realpath(main.__file__).startswith(os.path.realpath(REF))
    main.args.cuda = True
    main.args.distributed_rank = 0
    return main


@pytest.mark.parametrize("precision,first_tol,later_tol", [("fp32", 1e-3, 2e-2), ("bf16", 3e-2, 6e-2)])
def test_reference_execute_graph_with_byol_b200_classes(cuda, precision, first_tol, later_tol):
    import byol_b200.model
    import byol_b200.objective
    import byol_b200.lars
    import byol_b200.wiring
    z, arch, rep, b, r, steps, seed, lr, total = load_case("rn18_b8_r64")
    main = _import_reference_main(arch, rep, b, r)
    # --- the INTEGRATION.md edit, applied to the imported module (main.py's functions look these names up as globals)
    main.BYOL = functools.partial(byol_b200.model.BYOL, arch=main.args.arch,
                                  head_latent_size=main.args.head_latent_size, precision=precision)
    main.loss_function = byol_b200.objective.loss_function
    main.LARS = byol_b200.lars.LARS
    main.layers.DistributedDataParallelPassthrough = byol_b200.wiring.DistributedDataParallelPassthrough
    # --- the reference's wiring, unmodified: model construction order as main.build_loader_model_grapher
    # (main.py:428-436), optimizer as main.build_optimizer (main.py:321-340) with the golden run's fixed lr
    torch.manual_seed(seed)
    model = main.BYOL(base_network_output_size=rep, projection_output_size=256, classifier_output_size=1000,
                      total_training_steps=total, base_decay=0.996)
    model = model.cuda()
    groups = main.layers.add_weight_decay(model, 1e-6)
    opt = main.LARS(torch.optim.SGD(groups, lr=lr, momentum=0.9), eps=0.0)
    assert isinstance(model, byol_b200.model.BYOL) and isinstance(opt, byol_b200.lars.LARS)
    got = []
    for s, (a1, a2, lab) in enumerate(_batches(seed, steps, b, r)):
        got.append(main.execute_graph(1, model, [(a1, a2, lab)], None, optimizer=opt, prefix="train"))
    ref = [float(z["s%d_loss" % s]) for s in range(steps)]
    print("execute_graph losses (%s): %s   reference: %s" % (precision, got, ref))
    assert abs(got[0] - ref[0]) < first_tol * abs(ref[0])
    np.testing.assert_allclose(got, ref, rtol=later_tol)
    assert model.target_network.step == int(z["s%d_ema_step" % (steps - 1)])
    assert int(model.state_dict()["base_network.1.num_batches_tracked"]) == 4 * steps
    # the evaluation branch of the same function (main.py:573-575,584-598: model.eval(), no_grad, classifier on view 1)
    a1, a2, lab = _batches(seed, 1, b, r)[0]
    val = main.execute_graph(1, model, [(a1, a2, lab)], None, optimizer=None, prefix="test")
    assert np.isfinite(val) and not model.training
    assert model.target_network.step == int(z["s%d_ema_step" % (steps - 1)])      # no EMA update in eval mode
