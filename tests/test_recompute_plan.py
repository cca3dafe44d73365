"""CPU: the activation-recompute planner (Engine.memory_model / plan_blocks).  The bytes one online lane saves are
checked against sums written out from the torchvision layer shapes; the plan against budgets around the stored step's
need."""
import pytest

from byol_b200.model import BYOL

WIDTHS = (64, 128, 256, 512)      # bottleneck planes per stage; the block output has 4x planes channels


def _engine(arch, precision="bf16"):
    eng = BYOL(2048, 256, 1000, 10, arch=arch, precision=precision)._engine
    eng.walk_layers()
    return eng


def _lane_bytes(n, r, depths, inner, recompute=False):
    """Bottleneck nets (v1.5: the stride sits on conv2, the downsample is a 1x1 conv with the block's stride).
    Stored per block: y1 a1 [N,R_in,R_in,w], y2 a2 [N,R_out,R_out,w], y3 and the output [N,R_out,R_out,4p], the
    downsample's yd [N,R_out,R_out,4p] and, when it is a stride-2 GEMM, the compacted input xsub [N,R_out,R_out,Cin];
    bf16 each, plus the output's ReLU mask (1 bit per value).  With recompute only the output and its mask remain.
    The first block's input (the max-pool output [N,R/4,R/4,64]) is saved as well."""
    s = r // 4
    total = 2 * n * s * s * 64
    cin = 64
    for stage, (p, d) in enumerate(zip(WIDTHS, depths)):
        w = p * inner // 64
        for j in range(d):
            stride = 2 if (stage > 0 and j == 0) else 1
            ri, ro = s, s // stride
            y1, y2, out = n * ri * ri * w, n * ro * ro * w, n * ro * ro * 4 * p
            yd = out if j == 0 else 0
            xsub = n * ro * ro * cin if (j == 0 and stride == 2) else 0
            if recompute:
                total += 2 * out + out // 8
            else:
                total += 2 * (y1 + y1 + y2 + y2 + out + yd + xsub + out) + out // 8
            s, cin = ro, 4 * p
    return total


@pytest.mark.parametrize("arch,n,depths,inner", [
    ("resnet50", 512, (3, 4, 6, 3), 64),
    ("resnet200", 256, (3, 24, 36, 3), 64),
    ("resnext50_32x4d", 512, (3, 4, 6, 3), 128),      # 32 groups x 4 channels: inner width 2x planes
])
def test_lane_bytes_match_layer_shapes(arch, n, depths, inner):
    eng = _engine(arch)
    mm = eng.memory_model(n, 224, 224)
    everything = frozenset(range(len(eng.blocks)))
    assert len(eng.blocks) == sum(depths)
    assert eng.lane_bytes(mm, frozenset()) == _lane_bytes(n, 224, depths, inner)
    assert eng.lane_bytes(mm, everything) == _lane_bytes(n, 224, depths, inner, recompute=True)
    print("%s b%d: %.2f GB per online lane stored, %.2f GB recomputing every block" %
          (arch, n, eng.lane_bytes(mm, frozenset()) / 1e9, eng.lane_bytes(mm, everything) / 1e9))


def _order(mm):
    b = mm["blocks"]
    return sorted(range(len(b)), key=lambda i: (-(b[i]["stored"] - b[i]["kept"]) / b[i]["flops"], i))


@pytest.mark.parametrize("arch,n", [("resnet50", 512), ("resnext50_32x4d", 512), ("resnet:basic:2,2,2,2", 256)])
def test_plan_is_minimal_prefix_of_bytes_per_flop_order(arch, n):
    eng = _engine(arch)
    mm = eng.memory_model(n, 224, 224)
    order = _order(mm)
    stored = eng.step_need(mm, frozenset())
    assert eng.plan_blocks(mm, stored) == frozenset()
    assert eng.plan_blocks(mm, 10 * stored) == frozenset()
    assert eng.plan_blocks(mm, stored - 1) == frozenset(order[:1])
    for k in range(1, len(order) + 1):
        need = eng.step_need(mm, frozenset(order[:k]))
        assert need < eng.step_need(mm, frozenset(order[:k - 1]))
        assert eng.plan_blocks(mm, need) == frozenset(order[:k])              # fits with k blocks, not with k - 1
    assert eng.plan_blocks(mm, 0) == frozenset(order)                         # nothing fits: every block
    if arch == "resnet50":
        assert order[:3] == [0, 1, 2]        # the 56x56 stage saves the most bytes per recomputed FLOP


def test_recompute_plan_override_and_scope():
    eng = _engine("resnet50")
    mm = eng.memory_model(64, 128, 128)
    eng._mem_budget = eng.step_need(mm, frozenset())
    assert eng.recompute_plan(64, 128, 128) == frozenset()
    eng._mem_budget = 0
    assert eng.recompute_plan(64, 128, 128) == frozenset(range(len(eng.blocks)))
    for precision in ("fp32", "bf16x2"):                 # the split paths keep their own storage
        e = _engine("resnet50", precision)
        e._mem_budget = 0
        assert e.recompute_plan(64, 128, 128) == frozenset()
