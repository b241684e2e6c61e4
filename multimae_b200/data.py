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
"""
import functools
import math
import os
import random

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
    if isinstance(batch, PackedBatch):
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


@functools.lru_cache(maxsize=None)
def bicubic_coeffs(n_in, n_out):
    """Pillow's precompute_coeffs for BICUBIC from n_in to n_out samples (the whole axis as the box), in double:
    (bounds int32 [n_out, 2] = (first input sample, number of taps), normalised weights float64 [n_out, ksize])."""
    scale = float(n_in) / n_out
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(n_out) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)       # C's (int) truncates towards zero
    xmax = np.minimum((center + support + 0.5).astype(np.int64), n_in) - xmin
    x = np.arange(ksize)
    w = _bicubic_filter((x[None, :] + xmin[:, None] - center[:, None] + 0.5) * (1.0 / filterscale))
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
    bounds, w = bicubic_coeffs(n_in, n_out)
    ksize = w.shape[1]
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


def _crop_only(dataset):
    return isinstance(getattr(dataset, "transform", None), CropOnlyTransform)


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
                tud.DataLoader = _AugmentingDataLoader
                did.append("gpu_augment")
            except ImportError:
                pass
    if os.environ.get("MMAE_DEVICE_FEED", "0") == "1":
        import torch.utils.data as tud
        tud.DataLoader = _FeedingDataLoader
        did.append("device_feed")
    return did
