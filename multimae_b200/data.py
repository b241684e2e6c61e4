"""Input feeds for the unchanged training script (SURVEY.md section 8f n4; utils/datasets.py:66-111, run_pretraining_multimae.py
:338-347, 482-485).  The reference's PIL / albumentations pipeline stays the reference's own code; what this module adds,
opt-in through the overlay launcher:

  * MMAE_DEVICE_FEED=1   every `torch.utils.data.DataLoader` the script builds hands out batches that are ALREADY on the
                         GPU: a background prefetch stage copies batch i+1 host -> device on a copy stream (from pinned
                         memory, double-buffered) while step i runs, so the script's own
                         `tensor.to(device, non_blocking=True)` (:482-485) is a no-op and the H2D never sits on the step's
                         critical path (the same pipeline bench.py's end-to-end leg times).
  * MMAE_SYNTHETIC_DATA=N  `build_multimae_pretraining_dataset` returns N synthetic samples (rgb / depth / semseg tensors of
                         the configured input size) served from a small pool of pre-generated tensors: a data source that
                         keeps up with an H100 (the PIL pipeline delivers a few hundred samples/s per worker), for measuring
                         the unchanged script end to end.
  * MMAE_GPU_AUGMENT=1   `build_multimae_pretraining_dataset` builds the reference's MultiTaskImageFolder with a crop-only
                         transform (CropOnlyTransform): the workers decode, draw the crop and flip exactly as
                         DataAugmentationForMultiMAE draws them, and slice the crop out of the decoded image.  A collate
                         function packs a batch of crops, a descriptor table and the resampling tables into one host
                         buffer (PackedBatch); the DataLoader becomes a DeviceFeed whose copy stream uploads that buffer and
                         runs the resampling kernels (csrc/augment.cu) on it.  The batch it yields is bitwise the
                         reference's `[{'rgb', 'depth', 'semseg'}, target]`, already on the GPU.
                         It also rebinds `build_transform`, so that classification fine-tuning's train and eval datasets
                         get ClsTrainTransform / ClsEvalTransform: the workers make every random draw of the reference's
                         RandomResizedCropAndInterpolation, RandomHorizontalFlip and RandAugment and crop; the GPU
                         (mmae_cls_augment_batch) resizes, flips, applies the RandAugment ops and normalises, bitwise
                         as Pillow does.
"""
import functools
import math
import os
import random
import re

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset


class SyntheticMultiTaskDataset(Dataset):
    """{'rgb': [3,S,S] f32, 'depth': [1,S,S] f32, 'semseg': [S/4,S/4] i64} samples of `domains`, drawn from a pre-generated
    pool (index -> pool[index % pool]); returns `(dict, 0)` like MultiTaskImageFolder (utils/dataset_folder.py)."""

    def __init__(self, length, domains=("rgb", "depth", "semseg"), input_size=224, pool=256, seed=0, num_classes=133):
        g = torch.Generator().manual_seed(seed)
        self.length, self.pool = int(length), min(int(pool), int(length))
        self.data = {}
        for d in domains:
            if d == "semseg":
                self.data[d] = torch.randint(0, num_classes, (self.pool, input_size // 4, input_size // 4), generator=g)
            else:
                self.data[d] = torch.randn(self.pool, 1 if d == "depth" else 3, input_size, input_size, generator=g)

    def __len__(self):
        return self.length

    def __getitem__(self, i):
        j = i % self.pool
        return {d: t[j] for d, t in self.data.items()}, 0


def _to_device(batch, device, pool):
    """Recursively copy the tensors of `batch` to `device` through pinned staging buffers (non-blocking); a PackedBatch is
    uploaded and resampled on the current stream."""
    if isinstance(batch, (PackedBatch, PackedClsBatch)):
        return batch.to_device(device, pool)
    if isinstance(batch, torch.Tensor):
        if batch.is_cuda:
            return batch
        if not batch.is_pinned():
            key = (tuple(batch.shape), batch.dtype, pool["i"])
            stage = pool["bufs"].get(key)
            if stage is None:
                stage = pool["bufs"][key] = torch.empty(batch.shape, dtype=batch.dtype).pin_memory()
            stage.copy_(batch)
            batch = stage
        return batch.to(device, non_blocking=True)
    if isinstance(batch, dict):
        return {k: _to_device(v, device, pool) for k, v in batch.items()}
    if isinstance(batch, (list, tuple)):
        return type(batch)(_to_device(v, device, pool) for v in batch)
    return batch


class DeviceFeed:
    """Iterates `loader`, yielding batches that already live on `device`; the copy of batch i+1 is enqueued on a copy stream
    before batch i is handed out (two pinned staging sets alternate), and the consumer's stream waits for exactly that
    copy.  `len()` and every other attribute are the wrapped loader's."""

    def __init__(self, loader, device=None):
        self.loader = loader
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)

    def __len__(self):
        return len(self.loader)

    def __getattr__(self, name):
        return getattr(self.loader, name)

    def __iter__(self):
        if self.device.type != "cuda":
            yield from self.loader
            return
        copy_stream = torch.cuda.Stream(device=self.device)
        pools = [{"i": 0, "bufs": {}}, {"i": 1, "bufs": {}}]
        reuse = [None, None]                     # event: the consumer is done with the staging set (its copy completed)
        it = iter(self.loader)

        def stage(k):
            try:
                host = next(it)
            except StopIteration:
                return None
            with torch.cuda.stream(copy_stream):
                if reuse[k] is not None:
                    copy_stream.wait_event(reuse[k])
                dev = _to_device(host, self.device, pools[k])
                done = torch.cuda.Event()
                done.record(copy_stream)
            reuse[k] = done
            return dev, done

        k = 0
        nxt = stage(k)
        while nxt is not None:
            dev, done = nxt
            k ^= 1
            nxt = stage(k)                       # the next batch's H2D runs under the step that consumes this one
            torch.cuda.current_stream(self.device).wait_event(done)
            for t in _tensors(dev):
                t.record_stream(torch.cuda.current_stream(self.device))
            yield dev


def _tensors(obj):
    if isinstance(obj, torch.Tensor):
        yield obj
    elif isinstance(obj, dict):
        for v in obj.values():
            yield from _tensors(v)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            yield from _tensors(v)


# ---------------------------------------------------------------------------------------------------------------------
# MMAE_GPU_AUGMENT: DataAugmentationForMultiMAE (utils/datasets.py:66-111) split between the workers (decode, random draws,
# crop) and the GPU (Pillow-exact resize, flip, to_tensor / normalize, semseg nearest maps).
# ---------------------------------------------------------------------------------------------------------------------
from .kernels import AUGMENT_KINDS  # noqa: E402  (task -> kind code of mmae_augment_batch)
_CHANNELS = (3, 1, 1)
_ITEMSIZE = (1, 2, 1)
DESC_FIELDS = 8             # kind, src / 16, crop h, crop w, flip, column table / 16, row table / 16, scratch / 16
TABLE_BICUBIC, TABLE_NEAREST = 1, 2
_PRECISION_BITS = 22        # Pillow's fixed-point coefficients of 8-bit resampling (32 - 8 - 2)


def random_resized_crop_params(height, width, scale=(0.2, 1.0), ratio=(0.75, 1.3333)):
    """torchvision's RandomResizedCrop.get_params for an image of `height` x `width`, with the same torch calls in the same
    order (so the same draws from torch's generator): (i, j, h, w) of the crop, always inside the image."""
    area = height * width
    log_ratio = torch.log(torch.tensor(ratio))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(scale[0], scale[1]).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= width and 0 < h <= height:
            i = torch.randint(0, height - h + 1, size=(1,)).item()
            j = torch.randint(0, width - w + 1, size=(1,)).item()
            return i, j, h, w
    in_ratio = float(width) / float(height)      # fallback: the central crop of the ratio range
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


def _bicubic_filter(x):
    x = np.abs(x)
    a = -0.5
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                    np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))


def _bilinear_filter(x):
    x = np.abs(x)
    return np.where(x < 1.0, 1.0 - x, 0.0)


FILTER_BILINEAR, FILTER_BICUBIC = 2, 3      # PIL.Image.BILINEAR / BICUBIC
_FILTERS = {FILTER_BILINEAR: (_bilinear_filter, 1.0), FILTER_BICUBIC: (_bicubic_filter, 2.0)}


@functools.lru_cache(maxsize=None)
def bicubic_coeffs(n_in, n_out):
    """Pillow's precompute_coeffs for BICUBIC from n_in to n_out samples (the whole axis as the box), in double:
    (bounds int32 [n_out, 2] = (first input sample, number of taps), normalised weights float64 [n_out, ksize])."""
    return resample_coeffs(FILTER_BICUBIC, n_in, n_out)


@functools.lru_cache(maxsize=None)
def resample_coeffs(filt, n_in, n_out):
    """bicubic_coeffs for Pillow's BILINEAR (support 1) or BICUBIC (support 2) filter."""
    fn, filter_support = _FILTERS[filt]
    scale = float(n_in) / n_out
    filterscale = max(scale, 1.0)
    support = filter_support * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(n_out) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)       # C's (int) truncates towards zero
    xmax = np.minimum((center + support + 0.5).astype(np.int64), n_in) - xmin
    x = np.arange(ksize)
    w = fn((x[None, :] + xmin[:, None] - center[:, None] + 0.5) * (1.0 / filterscale))
    w = np.where(x[None, :] < xmax[:, None], w, 0.0)
    ww = np.zeros(n_out)
    for k in range(ksize):                      # Pillow's summation order (zero taps add nothing)
        ww = ww + w[:, k]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    return np.stack([xmin, xmax], 1).astype(np.int32), w


def fixed_point_coeffs(w):
    """Pillow's normalize_coeffs_8bpc: the weights as int32 with 22 fractional bits, rounded half away from zero."""
    scaled = w * float(1 << _PRECISION_BITS)
    return np.where(w < 0, np.trunc(-0.5 + scaled), np.trunc(0.5 + scaled)).astype(np.int32)


@functools.lru_cache(maxsize=None)
def nearest_map(n_in, n_out):
    """Pillow's NEAREST resize along one axis (ImagingScaleAffine): source index of each output sample, taken at the pixel
    centre with the position accumulated step by step in double, as Pillow does."""
    step = float(n_in) / n_out
    pos = step * 0.5
    out = np.empty(n_out, np.int32)
    for k in range(n_out):
        out[k] = -1 if pos < 0 else int(pos)
        pos += step
    return out


def _align16(n):
    return (n + 15) & ~15


@functools.lru_cache(maxsize=None)
def _table_bytes(kind, n_in, n_out):
    """One resampling table as it travels in a PackedBatch: int32 header {n_in, n_out, ksize, kind}, then
    BICUBIC: int32 bounds [n_out, 2], int32 fixed-point weights [n_out, ksize], float64 weights [n_out, ksize] (8-aligned);
    NEAREST: int32 source index [n_out]."""
    if kind == TABLE_NEAREST:
        return np.concatenate([np.array([n_in, n_out, 0, kind], np.int32), nearest_map(n_in, n_out)]).view(np.uint8)
    return _weights_table_bytes(kind, n_in, *bicubic_coeffs(n_in, n_out))


def _weights_table_bytes(kind, n_in, bounds, w):
    n_out, ksize = w.shape
    head = np.concatenate([np.array([n_in, n_out, ksize, kind], np.int32), bounds.reshape(-1),
                           fixed_point_coeffs(w).reshape(-1)]).view(np.uint8)
    pad = np.zeros((-len(head)) % 8, np.uint8)
    return np.concatenate([head, pad, w.reshape(-1).view(np.uint8)])


class Crops:
    """What CropOnlyTransform hands the collate function for one sample: the uint8 / uint16 crop of every task (dict order of
    the dataset), the flip flag and the crop size."""

    def __init__(self, arrays, flip, h, w):
        self.arrays, self.flip, self.h, self.w = arrays, flip, h, w


def _crop(a, i, j, h, w):
    """TF.crop of the decoded image `a`: zero outside the image, as PIL's crop fills it."""
    if i >= 0 and j >= 0 and i + h <= a.shape[0] and j + w <= a.shape[1]:
        return np.ascontiguousarray(a[i:i + h, j:j + w])
    out = np.zeros((h, w) + a.shape[2:], a.dtype)
    y0, x0, y1, x1 = max(i, 0), max(j, 0), min(i + h, a.shape[0]), min(j + w, a.shape[1])
    if y1 > y0 and x1 > x0:
        out[y0 - i:y1 - i, x0 - j:x1 - j] = a[y0:y1, x0:x1]
    return out


class CropOnlyTransform:
    """The worker half of DataAugmentationForMultiMAE: the same draws (random.random() < hflip, then get_params of the first
    task with scale (0.2, 1.0) and ratio (0.75, 1.3333)), then a slice of the decoded image.  `collate` packs a batch."""

    def __init__(self, args):
        default = args.imagenet_default_mean_and_std
        self.mean = (0.485, 0.456, 0.406) if default else (0.5, 0.5, 0.5)      # IMAGENET_DEFAULT / IMAGENET_INCEPTION
        self.std = (0.229, 0.224, 0.225) if default else (0.5, 0.5, 0.5)
        self.input_size = int(args.input_size)
        self.hflip = args.hflip

    def __call__(self, task_dict):
        flip = random.random() < self.hflip
        ijhw = None
        arrays = {}
        for task, img in task_dict.items():
            if task not in AUGMENT_KINDS:
                raise ValueError("MMAE_GPU_AUGMENT: no GPU augmentation for task %r" % task)
            if task == "depth" and img.mode != "I;16":
                raise ValueError("MMAE_GPU_AUGMENT: depth image %s has PIL mode %r; the GPU augmentation resamples 16-bit "
                                 "'I;16' depth only (unset MMAE_GPU_AUGMENT to use the reference transform)"
                                 % (getattr(img, "filename", "") or "<in memory>", img.mode))
            if ijhw is None:
                ijhw = random_resized_crop_params(img.height, img.width)
            arrays[task] = _crop(np.asarray(img), *ijhw)
        return Crops(arrays, flip, ijhw[2], ijhw[3])

    def collate(self, samples):
        return [pack_batch([s[0] for s in samples], self.input_size, self.mean, self.std),
                torch.tensor([s[1] for s in samples])]


class PackedBatch:
    """One batch of crops in one host buffer: int32 descriptors [batch, tasks, DESC_FIELDS] at offset 0, then the
    resampling tables, then the crops, every section 16-byte aligned (offsets in the descriptors count 16-byte units)."""

    def __init__(self, buffer, tasks, batch, size, map4, scratch_bytes, mean, std):
        self.buffer, self.tasks, self.batch, self.size, self.map4 = buffer, tasks, batch, size, map4
        self.scratch_bytes, self.mean, self.std = scratch_bytes, mean, std

    def pin_memory(self):
        self.buffer = self.buffer.pin_memory()
        return self

    def to_device(self, device, pool=None):
        """Upload the buffer and run the resampling kernels on the current stream: {task: tensor} on `device`."""
        from . import kernels
        host = self.buffer
        if not host.is_pinned():
            n = host.numel()
            stage = None if pool is None else pool["bufs"].get("packed")
            if stage is None or stage.numel() < n:
                stage = torch.empty(n + n // 4, dtype=torch.uint8).pin_memory()
                if pool is not None:
                    pool["bufs"]["packed"] = stage
            stage[:n].copy_(host)
            host = stage[:n]
        dev = host.to(device, non_blocking=True)
        return kernels.augment_batch(host, dev, self.tasks, self.batch, self.size, self.map4, self.scratch_bytes, self.mean,
                                     self.std)


def pack_batch(crops, size, mean, std):
    """The collate half: pack `crops` (list of Crops) for output size `size` into a PackedBatch."""
    tasks = list(crops[0].arrays)
    B, T = len(crops), len(tasks)
    size4 = int(size * 0.25)
    desc = np.zeros((B, T, DESC_FIELDS), np.int32)
    pieces, pos, tables = [], _align16(desc.nbytes), {}

    def put(a):
        nonlocal pos
        off = pos
        pieces.append((off, a))
        pos = _align16(pos + a.nbytes)
        return off // 16

    def table(kind, n_in, n_out):
        key = (kind, n_in, n_out)
        if key not in tables:
            tables[key] = put(_table_bytes(kind, n_in, n_out))
        return tables[key]

    map4 = table(TABLE_NEAREST, size, size4)
    scratch = 0
    for b, c in enumerate(crops):
        if list(c.arrays) != tasks:
            raise ValueError("MMAE_GPU_AUGMENT: every sample of a batch must carry the tasks %s" % tasks)
        for t, task in enumerate(tasks):
            kind = AUGMENT_KINDS[task]
            a = c.arrays[task]
            tk = TABLE_NEAREST if kind == 2 else TABLE_BICUBIC
            d = desc[b, t]
            d[0], d[2], d[3], d[4] = kind, c.h, c.w, int(c.flip)
            d[1] = put(a)
            d[5], d[6] = table(tk, c.w, size), table(tk, c.h, size)
            if kind != 2:
                d[7] = scratch // 16
                scratch = _align16(scratch + c.h * size * _CHANNELS[kind] * _ITEMSIZE[kind])
    buf = torch.empty(pos, dtype=torch.uint8)
    flat = buf.numpy()
    flat[:desc.nbytes] = desc.reshape(-1).view(np.uint8)
    for off, a in pieces:
        flat[off:off + a.nbytes] = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    return PackedBatch(buf, tasks, B, size, map4, scratch, mean, std)


def build_gpu_augment_dataset(args, stock):
    """MMAE_GPU_AUGMENT's build_multimae_pretraining_dataset: the reference's MultiTaskImageFolder with a CropOnlyTransform,
    or `stock(args)` (the reference's builder), with one printed line, when a domain has no GPU augmentation or there is
    no CUDA device."""
    import utils.datasets as ud  # type: ignore  (the reference's module)
    other = [d for d in args.all_domains if d not in AUGMENT_KINDS]
    if other:
        print("MMAE_GPU_AUGMENT: no GPU augmentation for domain(s) %s; keeping the reference transform" % ", ".join(other))
        return stock(args)
    if not torch.cuda.is_available():
        print("MMAE_GPU_AUGMENT: CUDA is not available; keeping the reference transform")
        return stock(args)
    return ud.MultiTaskImageFolder(args.data_path, args.all_domains, transform=CropOnlyTransform(args))


# ---------------------------------------------------------------------------------------------------------------------
# MMAE_GPU_AUGMENT for classification fine-tuning: utils/datasets.py:build_transform (transforms_imagenet_train with
# RandAugment, or Resize + CenterCrop) split between the workers (decode, every random draw, the op arguments, crop) and
# the GPU (Pillow-exact resize, flip, RandAugment ops, to_tensor / normalize: mmae_cls_augment_batch).
# ---------------------------------------------------------------------------------------------------------------------
TABLE_BILINEAR = 3          # same layout as TABLE_BICUBIC
_TABLE_OF = {FILTER_BILINEAR: TABLE_BILINEAR, FILTER_BICUBIC: TABLE_BICUBIC}
(OP_IDENTITY, OP_INVERT, OP_POSTERIZE, OP_SOLARIZE, OP_SOLARIZE_ADD, OP_AUTOCONTRAST, OP_EQUALIZE, OP_COLOR, OP_CONTRAST,
 OP_BRIGHTNESS, OP_SHARPNESS, OP_AFFINE, OP_TRANSPOSE) = range(13)
OP_DTYPE = np.dtype([("kind", "<i4"), ("filter", "<i4"), ("iarg", "<i4"), ("pad", "<i4"), ("factor", "<f8"),
                     ("m", "<f8", (6,))])                       # 72 bytes, the C side's ClsOp
_RAND_TRANSFORMS = ("AutoContrast", "Equalize", "Invert", "Rotate", "Posterize", "Solarize", "SolarizeAdd", "Color",
                    "Contrast", "Brightness", "Sharpness", "ShearX", "ShearY", "TranslateXRel", "TranslateYRel")
_RAND_INCREASING = {"Posterize": "PosterizeIncreasing", "Solarize": "SolarizeIncreasing", "Color": "ColorIncreasing",
                    "Contrast": "ContrastIncreasing", "Brightness": "BrightnessIncreasing",
                    "Sharpness": "SharpnessIncreasing"}
_RAND_CHOICE_WEIGHTS_0 = {"Rotate": 0.3, "ShearX": 0.2, "ShearY": 0.2, "TranslateXRel": 0.1, "TranslateYRel": 0.1,
                          "Color": .025, "Sharpness": 0.025, "AutoContrast": 0.025, "Solarize": .005, "SolarizeAdd": .005,
                          "Contrast": .005, "Brightness": .005, "Equalize": .005, "Posterize": 0, "Invert": 0}
_LEVEL_DENOM = 10.


class ClsOp:
    """One RandAugment op as the kernels apply it: kind (OP_*), resample filter, integer argument (bits, threshold,
    addend, rotation of a transpose), blend factor, inverse affine matrix."""

    def __init__(self, kind, iarg=0, factor=0.0, matrix=(0.0,) * 6, filt=0):
        self.kind, self.iarg, self.factor, self.matrix, self.filter = kind, int(iarg), float(factor), tuple(matrix), filt

    def __repr__(self):
        return "ClsOp(%d, %d, %r, %r, %d)" % (self.kind, self.iarg, self.factor, self.matrix, self.filter)


class ClsSample:
    """What a classification worker hands the collate function: the uint8 [h, w, 3] crop, its resize filter, the flip,
    the op records; for eval, (input extent, resized extent, first output) of the rows and columns instead."""

    def __init__(self, crop, filt, flip, ops, rows=None, cols=None):
        self.crop, self.filter, self.flip, self.ops, self.rows, self.cols = crop, filt, flip, ops, rows, cols


def _negate(v):
    return -v if random.random() > 0.5 else v


def _rotate_matrix(angle, w, h):
    """Image.rotate's inverse matrix (no expand, no centre / translate)."""
    center = (w / 2, h / 2)
    angle = -math.radians(angle)
    m = [round(math.cos(angle), 15), round(math.sin(angle), 15), 0.0, round(-math.sin(angle), 15),
         round(math.cos(angle), 15), 0.0]
    a, b, c, d, e, f = m
    x, y = -center[0] - 0, -center[1] - 0
    m[2], m[5] = a * x + b * y + c, d * x + e * y + f
    m[2] += center[0]
    m[5] += center[1]
    return m


class RandAugmentDraws:
    """utils/auto_augment.py:rand_augment_transform(config, hparams) as the draws it makes and the ops it applies:
    np.random.choice of the layers' ops, then per op random.random() > 0.5 (skip), random.gauss / uniform of the
    magnitude, the level function (with _randomly_negate) and, for the geometric ops when the filter is random,
    random.choice of the filter; every argument computed as the reference and Pillow's Python code compute it."""

    def __init__(self, config, img_mean, filt):
        self.magnitude, self.num_layers, weight_idx, names = _LEVEL_DENOM, 2, None, list(_RAND_TRANSFORMS)
        self.mstd, self.mmax = 0, None
        parts = config.split("-")
        if parts[0] != "rand":
            raise ValueError("not a RandAugment config: %r" % config)
        for c in parts[1:]:
            cs = re.split(r"(\d.*)", c)
            if len(cs) < 2:
                continue
            key, val = cs[:2]
            if key == "mstd":
                self.mstd = float("inf") if float(val) > 100 else float(val)
            elif key == "mmax":
                self.mmax = int(val)
            elif key == "inc":
                if bool(val):
                    names = [_RAND_INCREASING.get(n, n) for n in names]
            elif key == "m":
                self.magnitude = int(val)
            elif key == "n":
                self.num_layers = int(val)
            elif key == "w":
                weight_idx = int(val)
            else:
                raise ValueError("unknown RandAugment config section %r" % c)
        self.names = names
        self.weights = None
        if weight_idx is not None:
            if weight_idx != 0:
                raise ValueError("RandAugment weight index %d" % weight_idx)
            p = [_RAND_CHOICE_WEIGHTS_0[k] for k in _RAND_TRANSFORMS]
            self.weights = p / np.sum(p)
        self.fill, self.filter = tuple(int(v) for v in img_mean), filt     # filt None: random.choice per op

    def __call__(self, size):
        chosen = np.random.choice(len(self.names), self.num_layers, replace=self.weights is None, p=self.weights)
        return [self._op(self.names[k], size) for k in chosen]

    def _op(self, name, size):
        if random.random() > 0.5:
            return ClsOp(OP_IDENTITY)
        m = self.magnitude
        if self.mstd > 0:
            m = random.uniform(0, m) if self.mstd == float("inf") else random.gauss(m, self.mstd)
        return self.level_op(name, max(0., min(m, self.mmax or _LEVEL_DENOM)), size)

    def level_op(self, name, m, size):
        """The op `name` at magnitude `m`: the level function (with its _randomly_negate draw), then, for the geometric
        ops, the filter's draw.  Above magnitude 10 (`mmax`) the LUT ops' arguments leave the range where they still
        change the table; they are clamped to the in-range value that gives the same table."""
        if name in ("AutoContrast", "Equalize", "Invert"):
            return ClsOp({"AutoContrast": OP_AUTOCONTRAST, "Equalize": OP_EQUALIZE, "Invert": OP_INVERT}[name])
        if name.startswith("Posterize"):
            bits = int((m / _LEVEL_DENOM) * 4)
            bits = 4 - bits if name == "PosterizeIncreasing" else bits
            # bits < 0: ~(2 ** (8 - bits) - 1) clears every bit of a byte, as bits = 0 does
            return ClsOp(OP_IDENTITY) if bits >= 8 else ClsOp(OP_POSTERIZE, max(bits, 0))
        if name.startswith("Solarize") and name != "SolarizeAdd":
            t = int((m / _LEVEL_DENOM) * 256)
            t = 256 - t if name == "SolarizeIncreasing" else t
            return ClsOp(OP_SOLARIZE, min(max(t, 0), 256))     # below 0 every level inverts, above 256 none does
        if name == "SolarizeAdd":
            return ClsOp(OP_SOLARIZE_ADD, min(int((m / _LEVEL_DENOM) * 110), 255))   # min(255, i + add) saturates
        for base, kind in (("Color", OP_COLOR), ("Contrast", OP_CONTRAST), ("Brightness", OP_BRIGHTNESS),
                           ("Sharpness", OP_SHARPNESS)):
            if name.startswith(base):
                if name.endswith("Increasing"):
                    f = max(0.1, 1.0 + _negate((m / _LEVEL_DENOM) * .9))
                else:
                    f = (m / _LEVEL_DENOM) * 1.8 + 0.1
                return ClsOp(kind, factor=f)
        # geometric: the level function's draw, then the filter's
        if name == "Rotate":
            arg = _negate((m / _LEVEL_DENOM) * 30.)
        elif name in ("ShearX", "ShearY"):
            arg = _negate((m / _LEVEL_DENOM) * 0.3)
        else:
            arg = _negate((m / _LEVEL_DENOM) * 0.45)
        filt = random.choice((FILTER_BILINEAR, FILTER_BICUBIC)) if self.filter is None else self.filter
        if name == "Rotate":
            angle = arg % 360.0
            if angle == 0:
                return ClsOp(OP_IDENTITY)
            if angle in (90, 180, 270):          # Image.rotate's transpose shortcuts (the image is square)
                return ClsOp(OP_TRANSPOSE, int(angle))
            return ClsOp(OP_AFFINE, matrix=_rotate_matrix(angle, size, size), filt=filt)
        if name == "ShearX":
            mat = (1, arg, 0, 0, 1, 0)
        elif name == "ShearY":
            mat = (1, 0, 0, arg, 1, 0)
        elif name == "TranslateXRel":
            mat = (1, 0, arg * size, 0, 1, 0)
        else:
            mat = (1, 0, 0, 0, 1, arg * size)
        return ClsOp(OP_AFFINE, matrix=[float(v) for v in mat], filt=filt)


def autocontrast_lut(h):
    """ImageOps.autocontrast's table of one channel (cutoff 0, no ignore) from its 256-bin histogram."""
    nz = np.nonzero(np.asarray(h))[0]
    lo, hi = (int(nz[0]), int(nz[-1])) if len(nz) else (255, 0)
    if hi <= lo:
        return list(range(256))
    scale = 255.0 / (hi - lo)
    offset = -lo * scale
    return [min(max(int(ix * scale + offset), 0), 255) for ix in range(256)]


def equalize_lut(h):
    """ImageOps.equalize's table of one channel from its 256-bin histogram, clipped to 255 as Image.point clips it."""
    h = [int(v) for v in h]
    histo = [v for v in h if v]
    if len(histo) <= 1:
        return list(range(256))
    step = (sum(histo) - histo[-1]) // 255
    if not step:
        return list(range(256))
    n, out = step // 2, []
    for i in range(256):
        out.append(min(n // step, 255))
        n = n + h[i]
    return out


def contrast_mean(h):
    """ImageEnhance.Contrast's grey level: int(ImageStat mean of the L image + 0.5)."""
    s = 0.0
    for j in range(256):
        s += j * int(h[j])
    return int(s / sum(int(v) for v in h) + 0.5)


def rrc_params(height, width, scale=(0.08, 1.0), ratio=(3. / 4., 4. / 3.)):
    """utils/transforms.py:RandomResizedCropAndInterpolation.get_params, drawing from Python's random."""
    area = width * height
    for _ in range(10):
        target_area = random.uniform(*scale) * area
        log_ratio = (math.log(ratio[0]), math.log(ratio[1]))
        aspect_ratio = math.exp(random.uniform(*log_ratio))
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if w <= width and h <= height:
            return random.randint(0, height - h), random.randint(0, width - w), h, w
    in_ratio = width / height
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


def _norm(args):
    if args.imagenet_default_mean_and_std:
        return (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    return (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)


def _rgb_array(img):
    return np.asarray(img.convert("RGB") if img.mode != "RGB" else img)


class _ClsTransform:
    def __init__(self, args):
        self.input_size = int(args.input_size)
        self.mean, self.std = _norm(args)
        self.fill = tuple(min(255, round(255 * x)) for x in self.mean)     # aa_params['img_mean']
        self.transforms = [self]                                            # build_dataset prints transform.transforms

    def collate(self, samples):
        return [pack_cls_batch([s[0] for s in samples], self.input_size, self.mean, self.std, self.fill),
                torch.tensor([s[1] for s in samples])]


class ClsTrainTransform(_ClsTransform):
    """The worker half of transforms_imagenet_train(RandAugment): RandomResizedCropAndInterpolation.get_params and, for
    'random', random.choice of the filter (Python's random), RandomHorizontalFlip's torch.rand(1) < 0.5, then the
    RandAugment draws; returns the crop and the op records (ClsSample)."""

    def __init__(self, args):
        super().__init__(args)
        interp = args.train_interpolation
        self.filter = None if interp == "random" else (FILTER_BICUBIC if interp == "bicubic" else FILTER_BILINEAR)
        self.ra = RandAugmentDraws(args.aa, self.fill, self.filter)

    def __call__(self, img):
        a = _rgb_array(img)
        i, j, h, w = rrc_params(a.shape[0], a.shape[1])
        filt = random.choice((FILTER_BILINEAR, FILTER_BICUBIC)) if self.filter is None else self.filter
        flip = bool(torch.rand(1) < 0.5)
        ops = self.ra(self.input_size)
        return ClsSample(_crop(a, i, j, h, w), filt, flip, ops)

    def __repr__(self):
        return "ClsTrainTransform(size=%d, RandAugment %d layers of %s; resampled on the GPU)" % (
            self.input_size, self.ra.num_layers, ", ".join(self.ra.names))


def eval_geometry(n_in, n_resized, start, size, filt=FILTER_BICUBIC):
    """The input samples [first, first + extent) that outputs [start, start + size) of a resize n_in -> n_resized
    depend on."""
    bounds, _ = resample_coeffs(filt, n_in, n_resized)
    sl = bounds[start:start + size]
    first = int(sl[:, 0].min())
    return first, int((sl[:, 0] + sl[:, 1]).max()) - first


@functools.lru_cache(maxsize=None)
def sliced_table(filt, n_in, n_resized, start, size):
    """(bounds shifted to the first input sample used, fixed-point weights, double weights, first, extent) of outputs
    [start, start + size) of the resize n_in -> n_resized."""
    bounds, w = resample_coeffs(filt, n_in, n_resized)
    first, extent = eval_geometry(n_in, n_resized, start, size, filt)
    b = bounds[start:start + size].copy()
    b[:, 0] -= first
    ws = w[start:start + size]
    return b, fixed_point_coeffs(ws), ws, first, extent


class ClsEvalTransform(_ClsTransform):
    """The worker half of Resize(int(input_size / crop_pct), bicubic) + CenterCrop(input_size): the region of the
    decoded image the centre crop depends on, with the rows' and columns' (input extent, resized extent, first output)."""

    def __init__(self, args):
        super().__init__(args)
        self.resize = int(args.input_size / args.crop_pct)

    def __call__(self, img):
        a = _rgb_array(img)
        H, W = a.shape[:2]
        short, long = (W, H) if W <= H else (H, W)
        new_long = int(self.resize * long / short)
        new_w, new_h = (self.resize, new_long) if W <= H else (new_long, self.resize)
        S = self.input_size
        top, left = int(round((new_h - S) / 2.0)), int(round((new_w - S) / 2.0))
        r0, rh = eval_geometry(H, new_h, top, S)
        c0, cw = eval_geometry(W, new_w, left, S)
        return ClsSample(np.ascontiguousarray(a[r0:r0 + rh, c0:c0 + cw]), FILTER_BICUBIC, False, [],
                         rows=(H, new_h, top), cols=(W, new_w, left))

    def __repr__(self):
        return "ClsEvalTransform(resize=%d, center crop %d; resampled on the GPU)" % (self.resize, self.input_size)


class PackedClsBatch:
    """One classification batch in one host buffer: int32 descriptors [batch, DESC_FIELDS] (pack_batch's layout with one
    task), then the op records OP_DTYPE [batch, layers], then the tables, then the crops, every section 16-byte
    aligned."""

    def __init__(self, buffer, batch, size, layers, ops_offset, inter_bytes, mean, std, fill):
        self.buffer, self.batch, self.size, self.layers, self.ops_offset = buffer, batch, size, layers, ops_offset
        self.inter_bytes, self.mean, self.std, self.fill = inter_bytes, mean, std, fill

    def pin_memory(self):
        self.buffer = self.buffer.pin_memory()
        return self

    def to_device(self, device, pool=None):
        """Upload the buffer and run the kernels on the current stream: fp32 [B, 3, S, S] on `device`."""
        from . import kernels
        host = self.buffer
        if not host.is_pinned():
            n = host.numel()
            stage = None if pool is None else pool["bufs"].get("packed")
            if stage is None or stage.numel() < n:
                stage = torch.empty(n + n // 4, dtype=torch.uint8).pin_memory()
                if pool is not None:
                    pool["bufs"]["packed"] = stage
            stage[:n].copy_(host)
            host = stage[:n]
        dev = host.to(device, non_blocking=True)
        return kernels.cls_augment_batch(host, dev, self.batch, self.size, self.layers, self.ops_offset,
                                         self.inter_bytes, self.mean, self.std, self.fill)


def pack_cls_batch(samples, size, mean, std, fill):
    """The collate half: pack `samples` (list of ClsSample, all train or all eval) into a PackedClsBatch."""
    B = len(samples)
    layers = len(samples[0].ops)
    desc = np.zeros((B, DESC_FIELDS), np.int32)
    ops = np.zeros((B, layers), OP_DTYPE)
    ops_offset = _align16(desc.nbytes)
    pieces, pos, tables = [], _align16(ops_offset + ops.nbytes), {}

    def put(a):
        nonlocal pos
        off = pos
        pieces.append((off, a))
        pos = _align16(pos + a.nbytes)
        return off // 16

    def table(key, make):
        if key not in tables:
            tables[key] = put(make())
        return tables[key]

    inter = 0
    for b, s in enumerate(samples):
        if len(s.ops) != layers or (s.rows is None) != (samples[0].rows is None):
            raise ValueError("MMAE_GPU_AUGMENT: every sample of a batch must have the same transform")
        h, w = s.crop.shape[:2]
        d = desc[b]
        d[0], d[2], d[3], d[4] = 0, h, w, int(s.flip)
        d[1] = put(s.crop)
        kind = _TABLE_OF[s.filter]
        if s.rows is None:
            d[5] = table((kind, w, size), lambda: _weights_table_bytes(kind, w, *resample_coeffs(s.filter, w, size)))
            d[6] = table((kind, h, size), lambda: _weights_table_bytes(kind, h, *resample_coeffs(s.filter, h, size)))
        else:
            for field, (n_in, n_res, start), extent in ((5, s.cols, w), (6, s.rows, h)):
                def make(n_in=n_in, n_res=n_res, start=start, extent=extent):
                    b_, _, ws, _, e = sliced_table(s.filter, n_in, n_res, start, size)
                    assert e == extent
                    return _weights_table_bytes(kind, extent, b_, ws)
                d[field] = table((kind, n_in, n_res, start), make)
        d[7] = inter // 16
        inter = _align16(inter + h * size * 3)
        for l, op in enumerate(s.ops):
            ops[b, l] = (op.kind, op.filter, op.iarg, 0, op.factor, op.matrix)
    buf = torch.empty(pos, dtype=torch.uint8)
    flat = buf.numpy()
    flat[:desc.nbytes] = desc.reshape(-1).view(np.uint8)
    flat[ops_offset:ops_offset + ops.nbytes] = ops.reshape(-1).view(np.uint8)
    for off, a in pieces:
        flat[off:off + a.nbytes] = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    return PackedClsBatch(buf, B, size, layers, ops_offset // 16, inter, mean, std, fill)


def cls_fallback_reason(is_train, args):
    """Why build_transform(is_train, args) keeps the reference transform under MMAE_GPU_AUGMENT, or None."""
    if args.input_size <= 32:
        return "input_size %d <= 32 (RandomCrop with padding)" % args.input_size
    if is_train:
        if getattr(args, "reprob", 0) > 0:
            return "--reprob %g > 0 (RandomErasing)" % args.reprob
        aa = getattr(args, "aa", None)
        if not aa:
            return "--aa is empty (ColorJitter)"
        if not aa.startswith("rand"):
            return "--aa %s is not RandAugment" % aa
        if args.train_interpolation in ("lanczos", "hamming"):      # no affine transform filter in Pillow
            return "--train_interpolation %s" % args.train_interpolation
    elif args.crop_pct is not None and int(args.input_size / args.crop_pct) < args.input_size:
        return "crop_pct %g > 1 (CenterCrop pads)" % args.crop_pct
    if not torch.cuda.is_available():
        return "CUDA is not available"
    return None


def build_gpu_cls_transform(is_train, args, stock):
    """MMAE_GPU_AUGMENT's build_transform: a ClsTrainTransform / ClsEvalTransform, or `stock(is_train, args)` (the
    reference's) with one printed line."""
    reason = cls_fallback_reason(is_train, args)
    if reason is not None:
        print("MMAE_GPU_AUGMENT: %s; keeping the reference %s transform" % (reason, "train" if is_train else "eval"))
        return stock(is_train, args)
    if is_train:
        return ClsTrainTransform(args)
    if args.crop_pct is None:                    # build_transform's default
        args.crop_pct = 224 / 256 if args.input_size < 384 else 1.0
    return ClsEvalTransform(args)


_GPU_TRANSFORMS = (CropOnlyTransform, ClsTrainTransform, ClsEvalTransform)


def _crop_only(dataset):
    return isinstance(getattr(dataset, "transform", None), _GPU_TRANSFORMS)


class _FeedingDataLoader(DataLoader):
    """torch.utils.data.DataLoader whose iterator is a DeviceFeed (MMAE_DEVICE_FEED=1, overlay launcher only).  Over a
    dataset with a CropOnlyTransform (MMAE_GPU_AUGMENT=1) it also collates with that transform's packer."""

    feed_all = True         # False: only loaders over a CropOnlyTransform dataset feed the device

    def __init__(self, dataset, *args, **kwargs):
        if _crop_only(dataset) and kwargs.get("collate_fn") is None and len(args) < 6:
            kwargs["collate_fn"] = dataset.transform.collate
        super().__init__(dataset, *args, **kwargs)

    def __iter__(self):
        base = super().__iter__()
        if not torch.cuda.is_available() or not (self.feed_all or _crop_only(self.dataset)):
            return base

        class _Once:
            def __init__(self, it, n):
                self.it, self.n = it, n

            def __iter__(self):
                return self.it

            def __len__(self):
                return self.n
        return iter(DeviceFeed(_Once(base, len(self))))


class _AugmentingDataLoader(_FeedingDataLoader):
    """MMAE_GPU_AUGMENT=1 without MMAE_DEVICE_FEED: only loaders over a CropOnlyTransform dataset feed the device."""

    feed_all = False


def install():
    """Called by overlay.install(): apply the three environment switches (all off by default)."""
    did = []
    n = int(os.environ.get("MMAE_SYNTHETIC_DATA", "0") or 0)
    if n > 0:
        try:
            import utils.datasets as ud  # type: ignore  (the reference's module)

            def build(args):
                doms = list(dict.fromkeys(list(args.in_domains) + list(args.out_domains)))
                return SyntheticMultiTaskDataset(n, doms, getattr(args, "input_size", 224))
            ud.build_multimae_pretraining_dataset = build
            did.append("synthetic")
        except Exception:  # noqa: BLE001
            pass
    if os.environ.get("MMAE_GPU_AUGMENT", "0") == "1":
        if n > 0:
            print("MMAE_GPU_AUGMENT: MMAE_SYNTHETIC_DATA is set; the synthetic dataset has nothing to augment")
        else:
            try:
                import torch.utils.data as tud
                import utils.datasets as ud  # type: ignore  (the reference's module)
                stock = ud.build_multimae_pretraining_dataset
                ud.build_multimae_pretraining_dataset = functools.partial(build_gpu_augment_dataset, stock=stock)
                if hasattr(ud, "build_transform"):      # build_dataset (classification) looks it up at call time
                    ud.build_transform = functools.partial(build_gpu_cls_transform, stock=ud.build_transform)
                tud.DataLoader = _AugmentingDataLoader
                did.append("gpu_augment")
            except ImportError:
                pass
    if os.environ.get("MMAE_DEVICE_FEED", "0") == "1":
        import torch.utils.data as tud
        tud.DataLoader = _FeedingDataLoader
        did.append("device_feed")
    return did
