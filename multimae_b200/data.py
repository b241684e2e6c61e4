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
"""
import os

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
    """Recursively copy the tensors of `batch` to `device` through pinned staging buffers (non-blocking)."""
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


class _FeedingDataLoader(DataLoader):
    """torch.utils.data.DataLoader whose iterator is a DeviceFeed (MMAE_DEVICE_FEED=1, overlay launcher only)."""

    def __iter__(self):
        base = super().__iter__()
        if not torch.cuda.is_available():
            return base

        class _Once:
            def __init__(self, it, n):
                self.it, self.n = it, n

            def __iter__(self):
                return self.it

            def __len__(self):
                return self.n
        return iter(DeviceFeed(_Once(base, len(self))))


def install():
    """Called by overlay.install(): apply the two environment switches (both off by default)."""
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
    if os.environ.get("MMAE_DEVICE_FEED", "0") == "1":
        import torch.utils.data as tud
        tud.DataLoader = _FeedingDataLoader
        did.append("device_feed")
    return did
