"""GPU: the default ("reference") augmentation recipe gives the same bits as the build that recorded
tests/golden/augment_reference_bits_h100.json.

The sampler's records (dense, and ragged images sampled in chunks of one batch) and the apply / apply_ragged outputs
at a fixed seed and a few sizes (an up-scaling crop, the test transform's whole-image resize, and the pipeline without
its blur stage among them) are hashed with SHA-256.  A kernel change that keeps the reference recipe's arithmetic
gives the same digests; one that reorders a draw or a sum does not.

Regenerate (on the build whose bits are the reference):  python tests/test_gpu_augment_reference_bits.py --write [path]
"""
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FIXTURE = os.path.join(ROOT, "tests", "golden", "augment_reference_bits_h100.json")

pytestmark = pytest.mark.gpu

# ragged batch: landscape / portrait photographs, one image smaller than the output (every crop up-scales) and an
# extreme aspect ratio
RAGGED_SIZES = [(375, 500), (500, 375), (333, 500), (40, 52), (16, 200), (480, 640), (281, 300), (97, 131),
                (375, 500), (224, 224), (600, 450), (64, 48)]


def _sha(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def _images(n, hs, ws, seed):
    return torch.rand(n, 3, hs, ws, generator=torch.Generator().manual_seed(seed))


def _u8_images(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8) for h, w in sizes]


def _dense(dev, hs, ws, R, blur=True, n=8, seed=3):
    from byol_b200.augment import TwoViewAugment
    aug = TwoViewAugment(image_size=R, seed=seed, blur=blur)
    imgs = _images(n, hs, ws, hs * 1000 + ws).to(dev)
    d = {}
    for step in range(2):
        p = aug.sample_params(n, hs, ws, dev)
        v1, v2 = aug.apply(imgs, p)
        d["records_step%d" % step], d["views_step%d" % step] = _sha(p), _sha(torch.stack([v1, v2]))
    return d


def _ragged(dev, R, chunk, seed=11):
    from byol_b200.augment import TwoViewAugment
    aug = TwoViewAugment(image_size=R, seed=seed)
    imgs = [t.to(dev) for t in _u8_images(RAGGED_SIZES, seed)]
    n = len(imgs)
    parts = [aug.sample_params_ragged(RAGGED_SIZES[s:s + chunk], dev, n0=s, total=n, step=4)
             for s in range(0, n, chunk)]
    p = torch.cat(parts, dim=1).contiguous()
    v1, v2 = aug.apply_ragged(imgs, p)
    t1, t2 = aug.apply_ragged(imgs, aug.resize_params(RAGGED_SIZES, dev))
    return {"records_chunked": _sha(p), "views": _sha(torch.stack([v1, v2])),
            "resize_views": _sha(torch.stack([t1, t2]))}


def _cases():
    """name -> (function, kwargs); each function returns {part: digest}."""
    return {
        "dense_96x128_R64": (_dense, dict(hs=96, ws=128, R=64)),
        "dense_300x260_R224": (_dense, dict(hs=300, ws=260, R=224)),
        "dense_40x48_R112_upscale": (_dense, dict(hs=40, ws=48, R=112)),
        "dense_256x256_R224_noblur": (_dense, dict(hs=256, ws=256, R=224, blur=False)),
        "ragged_R224_chunk5": (_ragged, dict(R=224, chunk=5)),
        "ragged_R64_chunk4": (_ragged, dict(R=64, chunk=4)),
    }


def _digests(name, dev):
    fn, kw = _cases()[name]
    out = fn(dev, **kw)
    torch.cuda.synchronize()
    return out


def _fixture():
    with open(FIXTURE) as f:
        return json.load(f)


def test_fixture_covers_every_case():
    assert sorted(_fixture()["digests"]) == sorted(_cases())


@pytest.mark.parametrize("name", sorted(_cases()))
def test_reference_recipe_bits(cuda, name):
    assert _digests(name, cuda) == _fixture()["digests"][name]


if __name__ == "__main__":
    if not sys.argv[1:] or sys.argv[1] != "--write" or len(sys.argv) > 3:
        raise SystemExit("usage: python tests/test_gpu_augment_reference_bits.py --write [path]")
    path = sys.argv[2] if len(sys.argv) == 3 else FIXTURE
    dev = torch.device("cuda", 0)
    digests = {name: _digests(name, dev) for name in sorted(_cases())}
    again = {name: _digests(name, dev) for name in sorted(_cases())}
    assert digests == again, "the augmentation is not run-to-run reproducible"
    out = {"device": torch.cuda.get_device_name(0), "digests": digests}
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %d cases to %s" % (len(digests), path))
