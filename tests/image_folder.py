"""A small seeded image folder for the loader tests: JPEGs of mixed sizes (one smaller than 64 px, one with an extreme
aspect ratio, one grayscale) and one PNG named .JPEG, over three classes, in <root>/train and <root>/test."""
import os

import numpy as np

CLASSES = ["n01_cat", "n02_dog", "n03_fox"]
# (split, class index, file name, (H, W), kind)
FILES = [
    ("train", 0, "a0.JPEG", (120, 160), "rgb"),
    ("train", 0, "a1.JPEG", (96, 72), "rgb"),
    ("train", 0, "a2.jpg", (20, 30), "rgb"),           # smaller than the 64 px output
    ("train", 0, "a3.JPEG", (75, 100), "gray"),        # single-component JPEG
    ("train", 1, "b0.JPEG", (16, 200), "rgb"),         # extreme aspect ratio
    ("train", 1, "b1.JPEG", (130, 90), "rgb"),
    ("train", 1, "b2.JPEG", (88, 88), "png"),          # a PNG with a .JPEG name
    ("train", 1, "sub/b3.JPEG", (64, 80), "rgb"),      # nested below the class directory
    ("train", 2, "c0.JPEG", (100, 140), "rgb"),
    ("train", 2, "c1.jpeg", (140, 100), "rgb"),
    ("train", 2, "c2.JPEG", (66, 66), "rgb"),
    ("train", 2, "c3.JPEG", (50, 77), "rgb"),
    ("train", 2, "notes.txt", None, "text"),           # not an image: skipped
    ("test", 0, "t0.JPEG", (110, 90), "rgb"),
    ("test", 1, "t1.JPEG", (45, 60), "gray"),
    ("test", 2, "t2.JPEG", (90, 120), "rgb"),
    ("test", 2, "t3.JPEG", (70, 70), "png"),
    ("test", 2, "t4.JPEG", (128, 96), "rgb"),
]


def _pixels(rng, h, w, channels):
    """Smooth random content (bilinearly upsampled noise), so that JPEG keeps it well."""
    from PIL import Image
    small = rng.integers(0, 256, size=(max(2, h // 8), max(2, w // 8), channels), dtype=np.uint8)
    img = Image.fromarray(small[..., 0] if channels == 1 else small)
    return img.resize((w, h), Image.BILINEAR)


def make_image_folder(root, seed=0):
    """Writes the folder under `root`; returns {relative path: (class index, kind)} of the image files."""
    rng = np.random.default_rng(seed)
    made = {}
    for split, c, name, hw, kind in FILES:
        rel = os.path.join(split, CLASSES[c], name)
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        if kind == "text":
            with open(path, "w") as f:
                f.write("not an image\n")
            continue
        img = _pixels(rng, hw[0], hw[1], 1 if kind == "gray" else 3)
        if kind == "png":
            img.save(path, format="PNG")
        else:
            img.save(path, format="JPEG", quality=90)
        made[rel] = (c, kind)
    return made


def loader_kwargs(root, **over):
    """vars(args) of the reference's parser as the loader sees it, plus the transform lists main.py adds."""
    kw = dict(task="multi_augment_image_folder", data_dir=str(root), batch_size=4, image_size_override=64,
              color_jitter_strength=1.0, seed=5, num_replicas=1, distributed_rank=0, workers_per_replica=2,
              train_transform=[], test_transform=[])
    kw.update(over)
    return kw
