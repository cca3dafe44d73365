"""Generate the ResNeXt-50 golden vectors (tests/golden/rnx50_b8_r64.npz) by running the UNMODIFIED reference on CPU,
with the same recipe as make_golden.py (its run_case: main.execute_graph, LARS around SGD, sampled parameters,
gradients and EMA).

    python tests/golden/make_golden_resnext.py        # writes tests/golden/rnx50_b8_r64.npz (about 10 s)

ResNeXt-50 32x4d has 32 groups of 4 channels in its first stage: the grouped 3x3 convolutions.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden  # noqa: E402

# name, arch, repr, batch, image size, steps, seed, lr
CASE = ("rnx50_b8_r64", "resnext50_32x4d", 2048, 8, 64, 2, 13, 0.3)

if __name__ == "__main__":
    torch.set_num_threads(8)
    sys.argv = sys.argv[:1]
    make_golden.run_case(CASE)
