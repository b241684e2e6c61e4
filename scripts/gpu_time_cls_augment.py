"""Time the GPU classification fine-tuning augmentation (MMAE_GPU_AUGMENT, mmae_cls_augment_batch) against the
reference's CPU transform on one GPU.

    python scripts/gpu_time_cls_augment.py [--images 512] [--iters 50] [--loader-batches 24]

Writes a seeded image folder of JPEG files (quality 90, sizes drawn from 300 to 600 per side, ImageNet-like) to a
temporary directory.  The reference's transform is played by the stand-in `utils.datasets` of
tests/cls_augment_standin: the reference's draws, then the same Pillow calls as the reference (bitwise its output).
The transform is run_finetuning_cls.py's default: input 224, --aa rand-m9-mstd0.5-inc1, bicubic, eval crop_pct 0.875.

Prints one JSON line per figure:
  - the GPU name, power limit, current and maximum SM clock, read in the same run (first and last line);
  - mmae_cls_augment_batch per batch of 128 at S = 224, train and eval: each kernel's device time from torch.profiler
    over --iters calls, and CUDA events around the whole call (output and scratch allocation and the host's argument
    checks of 128 samples included), after a warm-up;
  - worker CPU time per sample (process time, one process with one torch thread as in a DataLoader worker, after a
    warm-up pass): the stand-in reference transform (decode + the reference's draws + the reference's Pillow calls)
    against the switch's worker transform (decode + draws + crop), and the packing of a batch of 128 per sample;
  - DataLoader samples/s at batch 128 with 10 workers, both ending with the batch on the GPU: off is the stand-in's
    loader wrapped in DeviceFeed, on is the switch's loader.  One iterator over one epoch of (2 x workers +
    --loader-batches) batches read round-robin from the images; the first 2 x workers batches (worker start-up and
    prefetch) are not timed, the next --loader-batches are."""
import argparse
import functools
import json
import os
import random
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "cls_augment_standin"))

import cls_augment_oracle as O  # noqa: E402
from multimae_b200 import data as D  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power, clock, max_clock = [s.strip() for s in out.strip().splitlines()[0].split(",")]
    except Exception:  # noqa: BLE001
        name, power, clock, max_clock = torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"
    return dict(gpu=name, power_limit=power, sm_clock=clock, max_sm_clock=max_clock)


def write_tree(root, n, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    for k in range(n):
        d = os.path.join(root, "class_%d" % (k % 4))
        os.makedirs(d, exist_ok=True)
        h, w = int(rng.integers(300, 601)), int(rng.integers(300, 601))
        Image.fromarray(O.make_image(int(rng.integers(1 << 30)), h, w)).save(os.path.join(d, "%05d.jpg" % k),
                                                                              quality=90)


class Cycle(torch.utils.data.Dataset):
    """`length` samples read round-robin from `ds`; keeps the wrapped dataset's transform visible."""

    def __init__(self, ds, length):
        self.ds, self.length, self.transform = ds, length, ds.transform

    def __len__(self):
        return self.length

    def __getitem__(self, k):
        return self.ds[k % len(self.ds)]


def args_for(root):
    return SimpleNamespace(input_size=224, imagenet_default_mean_and_std=True, aa="rand-m9-mstd0.5-inc1",
                           train_interpolation="bicubic", reprob=0.0, crop_pct=None, data_path=root,
                           eval_data_path=root, nb_classes=4, color_jitter=0.4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--loader-batches", type=int, default=24)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this script measures on a CUDA device"
    dev = torch.device("cuda:0")
    emit(**gpu_info())
    import utils.datasets as ud
    stock = ud.build_transform
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, a.images)
        # kernel time per batch of 128
        for is_train in (True, False):
            ud.build_transform = functools.partial(D.build_gpu_cls_transform, stock=stock)
            ds, _ = ud.build_dataset(is_train, args_for(root))
            random.seed(0)
            np.random.seed(0)
            torch.manual_seed(0)
            packed, _ = ds.transform.collate([ds[k] for k in range(128)])
            host = packed.buffer.pin_memory()
            devbuf = host.to(dev)
            from multimae_b200 import kernels

            def call():
                return kernels.cls_augment_batch(host, devbuf, packed.batch, packed.size, packed.layers,
                                                 packed.ops_offset, packed.inter_bytes, packed.mean, packed.std,
                                                 packed.fill)
            for _ in range(5):
                call()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.iters):
                call()
            t1.record()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    call()
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA and ("augment_" in ev.name or "cls_" in ev.name):
                    name = next(k for k in ("horizontal", "vertical_u8", "vertical", "prepare", "apply") if k in ev.name)
                    kern[name] = kern.get(name, 0.0) + ev.device_time / 1e3 / a.iters
            emit(figure="per_batch", transform="train" if is_train else "eval", batch=128, size=224,
                 layers=packed.layers, kernels_ms={k: round(v, 4) for k, v in kern.items()},
                 kernels_total_ms=round(sum(kern.values()), 4), call_event_ms=round(t0.elapsed_time(t1) / a.iters, 4),
                 iters=a.iters)
        # worker CPU time per sample
        torch.set_num_threads(1)
        for is_train in (True, False):
            ud.build_transform = stock
            ref_ds, _ = ud.build_dataset(is_train, args_for(root))
            ud.build_transform = functools.partial(D.build_gpu_cls_transform, stock=stock)
            gpu_ds, _ = ud.build_dataset(is_train, args_for(root))
            n = min(len(ref_ds), 256)
            res = {}
            for name, ds in (("standin_reference", ref_ds), ("gpu_augment_worker", gpu_ds)):
                for k in range(16):
                    ds[k]
                c0 = time.process_time()
                items = [ds[k] for k in range(n)]
                res[name] = (time.process_time() - c0) / n * 1e3
            c0 = time.process_time()
            for b in range(0, n - 127, 128):
                gpu_ds.transform.collate(items[b:b + 128])
            res["pack"] = (time.process_time() - c0) / (n // 128 * 128) * 1e3
            emit(figure="worker_cpu_ms_per_sample", transform="train" if is_train else "eval", samples=n, **res)
        torch.set_num_threads(min(16, os.cpu_count() or 1))
        # DataLoader throughput: one iterator over one epoch long enough for the warm-up and the timed batches
        from torch.utils.data import DataLoader
        workers = 10
        need = 2 * workers + a.loader_batches
        for name in ("off", "on"):
            ud.build_transform = stock if name == "off" else functools.partial(D.build_gpu_cls_transform, stock=stock)
            ds, _ = ud.build_dataset(True, args_for(root))
            ds = Cycle(ds, need * 128)
            cls = DataLoader if name == "off" else D._AugmentingDataLoader
            loader = cls(ds, batch_size=128, shuffle=True, num_workers=workers, drop_last=True, pin_memory=True)
            if name == "off":
                loader = D.DeviceFeed(loader, dev)
            got, t0 = 0, None
            for x, y in loader:
                got += 1
                if got == 2 * workers:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
            torch.cuda.synchronize()
            assert got == need
            dt = time.perf_counter() - t0
            emit(figure="dataloader_samples_per_s", switch=name, workers=workers, batch=128, cpus=os.cpu_count(),
                 samples_per_s=round(a.loader_batches * 128 / dt, 1), timed_batches=a.loader_batches)
    emit(**gpu_info())


if __name__ == "__main__":
    main()
