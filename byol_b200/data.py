"""Image-folder input for the reference's ``multi_augment_image_folder`` task: a drop-in for the missing
``datasets.loader.get_loader`` (/root/reference/main.py:414-417) that decodes JPEGs on the GPU and augments them there.

    from byol_b200.data import get_loader
    loader = get_loader(**vars(args), train_transform=..., test_transform=...)   # the transform lists are ignored
    for aug1, aug2, labels in loader.train_loader: ...                          # CUDA fp32 [B, 3, R, R] views in [0, 1]

Layout: ``<data_dir>/train`` and ``<data_dir>/test``, plus ``<data_dir>/valid`` when present.  Each holds one
subdirectory per class; classes are the sorted subdirectory names (index = position), and a class's images are the
files below it, walked recursively in sorted order, whose extension is .jpg, .jpeg, .png or .webp (any case), as in
torchvision's ``ImageFolder``.  The missing submodule's exact conventions are not known; this layout, the per-epoch
shuffle and the sharding below are this module's own choices.

Train: every epoch the whole split is permuted with a generator seeded from ``(seed, epoch)``; rank ``r`` of
``num_replicas`` takes the ``r``-th of ``num_replicas`` equal contiguous parts of that permutation, and the
remainder is dropped, so ``len(train_loader) == num_train_samples // num_replicas // batch_size``.  The two views are
``TwoViewAugment``'s recipe (RandomResizedCrop of the original image, flip, colour jitter, grayscale, blur) with
``image_size_override`` and ``color_jitter_strength``, and ``augmentation`` names the recipe: "reference" (the
default, also when the key is absent) or "byol", the BYOL paper's (bicubic crops, its colour jitter, per-view blur and
solarization; see ``byol_b200.augment``).  A sample's records are keyed by ``(seed, epoch, batch, its position in the
global batch, view)``.  Test / valid: neither sharded nor shuffled, the last batch may be short, and both views are
the same image, transformed by ``eval_transform``: "resize" (the default, also when the key is absent) resizes the whole
image to ``R x R`` (antialiased bilinear, the reference's ``Resize``); "byol" is the BYOL paper's test transform, the
shorter side resized to (8R + 3) // 7 (256 at R = 224) by antialiased bicubic and the centre ``R x R`` crop (see
``byol_b200.augment``); "byol_transfer" is the paper's transfer-evaluation preprocessing, the shorter side resized to
R by antialiased bicubic and the centre ``R x R`` crop.  It is independent of ``augmentation``, and the evaluations
(``knn_accuracy``, ``linear_accuracy``, ``finetune_accuracy``, ``transfer_accuracy``) read their images through it.

Per batch the file bytes are read by a small host thread pool, one batch ahead of the one being decoded.  Images are
decoded and augmented in sub-batches of ``DECODE_BATCH``, each into its slice of the output before the next is
decoded, which bounds the decoded bytes a batch of large images holds.  3-component baseline / progressive JPEGs go
to torchvision's nvJPEG decoder; other files (PNG, WebP, grayscale or CMYK JPEGs, or a sub-batch the GPU decoder
rejects) are decoded on the host by ``torchvision.io.decode_image`` and uploaded.  Everything runs on the current
CUDA stream.  ``num_*_samples`` are global counts, as ``main.py:421-424`` expects.
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .augment import EVAL_TRANSFORMS, RECIPES, TwoViewAugment

TASK = "multi_augment_image_folder"
EXTENSIONS = (".jpg", ".jpeg", ".png", ".webp")
DECODE_BATCH = 64      # images decoded (and augmented) at once


def _scan(root):
    """ImageFolder-style listing: (sorted class names, [(path, class index)])."""
    classes = sorted(e.name for e in os.scandir(root) if e.is_dir())
    samples = []
    for c, name in enumerate(classes):
        for dirpath, dirnames, filenames in sorted(os.walk(os.path.join(root, name), followlinks=True)):
            dirnames.sort()
            for fn in sorted(filenames):
                if fn.lower().endswith(EXTENSIONS):
                    samples.append((os.path.join(dirpath, fn), c))
    return classes, samples


def _read(path):
    with open(path, "rb") as f:
        buf = bytearray(os.fstat(f.fileno()).st_size)
        f.readinto(buf)
    return buf


def _nvjpeg_decodable(data):
    """True for a baseline / extended / progressive Huffman JPEG with three components (SOF0-2, Nf = 3)."""
    if len(data) < 4 or data[0] != 0xFF or data[1] != 0xD8:
        return False
    i = 2
    while i + 3 < len(data):
        if data[i] != 0xFF:
            return False
        m = data[i + 1]
        if m == 0xFF:                                   # fill byte
            i += 1
        elif m == 0x01 or 0xD0 <= m <= 0xD7:            # markers without a length
            i += 2
        elif 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            return m <= 0xC2 and i + 9 < len(data) and data[i + 9] == 3
        elif m in (0xD9, 0xDA):                         # end of image / start of scan before any frame header
            return False
        else:
            i += 2 + ((data[i + 2] << 8) | data[i + 3])
    return False


def decode_batch(datas, device):
    """File bytes -> list of contiguous uint8 [3, H, W] images on ``device`` (RGB)."""
    from torchvision.io import ImageReadMode, decode_image, decode_jpeg
    out = [None] * len(datas)
    gpu = [i for i, d in enumerate(datas) if _nvjpeg_decodable(d)]
    if gpu:
        try:
            dec = decode_jpeg([torch.frombuffer(datas[i], dtype=torch.uint8) for i in gpu], mode=ImageReadMode.RGB,
                              device=device)
            for i, t in zip(gpu, dec):
                out[i] = t.contiguous()
        except RuntimeError:
            pass                                        # the host decodes the whole sub-batch instead
    for i, t in enumerate(out):
        if t is None:
            img = decode_image(torch.frombuffer(datas[i], dtype=torch.uint8), mode=ImageReadMode.RGB)
            out[i] = img.contiguous().to(device)
    return out


class ImageFolderLoader(object):
    """Iterates one split: ``(aug1, aug2, labels)`` CUDA batches (see the module docstring)."""

    def __init__(self, samples, batch_size, augment, train, seed=0, rank=0, replicas=1, workers=2):
        self.samples, self.batch_size, self.augment, self.train = samples, int(batch_size), augment, bool(train)
        self.seed, self.rank, self.replicas, self.workers = int(seed), int(rank), int(replicas), int(workers)
        self.epoch = 0

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def __len__(self):
        if self.train:
            return len(self.samples) // self.replicas // self.batch_size
        return (len(self.samples) + self.batch_size - 1) // self.batch_size

    def indices(self):
        """Sample indices this rank visits this epoch, in order."""
        n = len(self.samples)
        if not self.train:
            return np.arange(n)
        perm = np.random.default_rng([self.seed, self.epoch]).permutation(n)
        per = n // self.replicas
        return perm[self.rank * per:(self.rank + 1) * per][:len(self) * self.batch_size]

    def __iter__(self):
        order = self.indices()
        batches = [order[i:i + self.batch_size] for i in range(0, len(order), self.batch_size)]
        pool = ThreadPoolExecutor(max_workers=self.workers)

        def read(b):
            return [pool.submit(_read, self.samples[i][0]) for i in b]

        try:
            pending = read(batches[0]) if batches else None
            for k, b in enumerate(batches):
                datas = [f.result() for f in pending]
                pending = read(batches[k + 1]) if k + 1 < len(batches) else None    # prefetch during this step
                yield self._batch(datas, [self.samples[i][1] for i in b], self.epoch * len(self) + k)
        finally:
            pool.shutdown(wait=False, cancel_futures=True)

    def _batch(self, datas, labels, step):
        device = torch.device("cuda", torch.cuda.current_device())
        n, R = len(datas), self.augment.R
        out = torch.empty((2, n, 3, R, R), dtype=torch.float32, device=device)
        stream = torch.cuda.current_stream(device)
        for s in range(0, n, DECODE_BATCH):
            images = decode_batch(datas[s:s + DECODE_BATCH], device)
            sizes = [tuple(t.shape[1:]) for t in images]
            if self.train:
                params = self.augment.sample_params_ragged(sizes, device, n0=self.rank * self.batch_size + s,
                                                           total=self.replicas * self.batch_size, step=step)
            else:
                params = self.augment.eval_params(sizes, device)
            v1, v2 = self.augment.apply_ragged(images, params)
            out[0, s:s + len(images)].copy_(v1)
            out[1, s:s + len(images)].copy_(v2)
            for t in images:            # the decoded images are freed only after the kernels queued here have read them
                t.record_stream(stream)
        return out[0], out[1], torch.tensor(labels, dtype=torch.int64).to(device)


class ImageFolderTwoView(object):
    """The object ``main.py`` gets from ``get_loader``."""

    def __init__(self, data_dir, batch_size, image_size=224, color_jitter_strength=1.0, seed=0, rank=0, replicas=1,
                 workers=2, augmentation="reference", eval_transform="resize"):
        if augmentation not in RECIPES:
            raise ValueError("get_loader: unknown augmentation %r (expected one of %s)" % (augmentation, sorted(RECIPES)))
        if eval_transform not in EVAL_TRANSFORMS:
            raise ValueError("get_loader: unknown eval_transform %r (expected one of %s)"
                             % (eval_transform, sorted(EVAL_TRANSFORMS)))
        splits = {}
        for name in ("train", "test", "valid"):
            root = os.path.join(data_dir, name)
            if os.path.isdir(root):
                splits[name] = _scan(root)
            elif name != "valid":
                raise FileNotFoundError("get_loader: %s has no %s/ directory (expected <data_dir>/train and "
                                        "<data_dir>/test, each with one subdirectory per class)" % (data_dir, name))
        classes = splits["train"][0]
        if not classes:
            raise FileNotFoundError("get_loader: %s has no class directories" % os.path.join(data_dir, "train"))
        self.classes = classes
        self.input_shape = [3, int(image_size), int(image_size)]
        self.output_size = len(classes)
        self.num_train_samples = len(splits["train"][1])
        self.num_test_samples = len(splits["test"][1])
        self.num_valid_samples = len(splits["valid"][1]) if "valid" in splits else 0
        if self.num_train_samples // replicas < batch_size:
            raise ValueError("get_loader: %d training images cannot fill one batch of %d on each of %d replicas"
                             % (self.num_train_samples, batch_size, replicas))
        self.augmentation, self.eval_transform = augmentation, eval_transform
        train_aug = TwoViewAugment(image_size=image_size, color_jitter_strength=color_jitter_strength, seed=seed,
                                   recipe=augmentation)
        # eval_transform records only: the recipe is unused
        test_aug = TwoViewAugment(image_size=image_size, seed=seed, eval_transform=eval_transform)
        self.train_loader = ImageFolderLoader(splits["train"][1], batch_size, train_aug, True, seed, rank, replicas,
                                              workers)
        self.test_loader = ImageFolderLoader(splits["test"][1], batch_size, test_aug, False, workers=workers)
        self.valid_loader = ImageFolderLoader(splits["valid"][1], batch_size, test_aug, False, workers=workers) \
            if "valid" in splits else None

    def set_all_epochs(self, epoch):
        for ld in (self.train_loader, self.test_loader, self.valid_loader):
            if ld is not None:
                ld.set_epoch(epoch)


def get_loader(**kwargs):
    """``datasets.loader.get_loader`` for ``--task multi_augment_image_folder``; takes ``vars(args)`` plus the
    transform lists, which are ignored (the training recipe is named by ``augmentation``, the test / validation
    transform by ``eval_transform``; see the module docstring)."""
    task = kwargs.get("task", TASK)
    if "dali" in task:
        raise ValueError("get_loader: DALI tasks are not supported (task %r); use %r" % (task, TASK))
    if task != TASK:
        raise ValueError("get_loader: only the %r task is supported, not %r" % (TASK, task))
    data_dir = kwargs.get("data_dir")
    if not data_dir or not os.path.isdir(data_dir):
        raise FileNotFoundError("get_loader: data directory %r does not exist" % (data_dir,))
    seed = kwargs.get("seed")
    augmentation = kwargs.get("augmentation") or "reference"
    eval_transform = kwargs.get("eval_transform") or "resize"
    return ImageFolderTwoView(data_dir, int(kwargs.get("batch_size", 4096)),
                              image_size=int(kwargs.get("image_size_override") or 224),
                              color_jitter_strength=float(kwargs.get("color_jitter_strength", 1.0)),
                              seed=0 if seed is None else int(seed),
                              rank=int(kwargs.get("distributed_rank") or 0),
                              replicas=max(1, int(kwargs.get("num_replicas") or 1)),
                              workers=max(2, int(kwargs.get("workers_per_replica") or 2)),
                              augmentation=augmentation, eval_transform=eval_transform)
