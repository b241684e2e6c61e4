"""Time the GPU pre-training augmentation (MMAE_GPU_AUGMENT) against the reference's CPU transform on one GPU.

    python scripts/gpu_time_augment.py [--images 1024] [--iters 50] [--loader-batches 16]

Writes a seeded image folder in MultiTaskImageFolder layout (rgb JPEG quality 90, 16-bit depth PNG, P-mode semseg PNG,
sizes drawn around 500 x 375) to a temporary directory.  The reference's transform is played by the stand-in
`utils.datasets` of tests/augment_standin (tests/augment_oracle.py, bitwise the reference's outputs).

Prints one JSON line per figure:
  - the GPU name, power limit and maximum SM clock, read in the same run (first and last line);
  - mmae_augment_batch per batch at B = 128 and 256, S = 224: the two kernels' device time from torch.profiler over
    --iters calls, and CUDA events / the host clock around the whole call (output allocation and the host's argument
    checks included);
  - worker CPU time per sample (process time, one process with one torch thread as in a DataLoader worker, after a
    warm-up pass over the images): decoding alone, the reference transform with the switch off (decode +
    DataAugmentationForMultiMAE), the crop-only transform with it on (decode + draws + crop), and the packing of a batch
    of 128 per sample;
  - DataLoader samples/s at batch 128 with 4 and 10 workers, both ending with the batch on the GPU: off is the stock
    loader wrapped in DeviceFeed (MMAE_DEVICE_FEED), on is the switch's loader.  The images are read round-robin; the
    first 2 x workers batches (what the workers prefetch) are not timed, the next --loader-batches are."""
import argparse
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
sys.path.insert(0, os.path.join(ROOT, "tests", "augment_standin"))

import augment_oracle as AO  # noqa: E402
from multimae_b200 import data as D  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def write_tree(root, n, seed=0):
    rng = np.random.default_rng(seed)
    for k in range(n):
        c = "class_%d" % (k % 4)
        h, w = int(rng.integers(330, 420)), int(rng.integers(440, 560))
        if k % 2:
            h, w = w, h
        imgs = AO.make_images(int(rng.integers(1 << 30)), h, w)
        for task, img in imgs.items():
            os.makedirs(os.path.join(root, task, c), exist_ok=True)
            if task == "rgb":
                img.save(os.path.join(root, task, c, "%05d.jpg" % k), quality=90)
            else:
                img.save(os.path.join(root, task, c, "%05d.png" % k))


class Cycle(torch.utils.data.Dataset):
    """`length` samples read round-robin from `ds`; keeps the wrapped dataset's transform visible."""

    def __init__(self, ds, length):
        self.ds, self.length, self.transform = ds, length, ds.transform

    def __len__(self):
        return self.length

    def __getitem__(self, k):
        return self.ds[k % len(self.ds)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--loader-batches", type=int, default=16)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    emit(**gpu_info())
    import utils.datasets as ud  # the stand-in
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, a.images)
        args = SimpleNamespace(input_size=224, hflip=0.5, imagenet_default_mean_and_std=True, data_path=root,
                               all_domains=["rgb", "depth", "semseg"])
        ref_ds = ud.build_multimae_pretraining_dataset(args)
        gpu_ds = D.build_gpu_augment_dataset(args, ud.build_multimae_pretraining_dataset)
        decode_ds = ud.MultiTaskImageFolder(root, args.all_domains, transform=None)
        crop = gpu_ds.transform

        # ---- kernel time per batch
        random.seed(0)
        torch.manual_seed(0)
        for B in (128, 256):
            packed = crop.collate([gpu_ds[k % len(gpu_ds)] for k in range(B)])[0]
            host = packed.buffer.pin_memory()
            devbuf = host.to(dev)

            def call():                      # the resampling kernels alone, on the uploaded buffer
                return packed.resample(host, devbuf)
            for _ in range(5):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            for _ in range(a.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) / a.iters
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    call()
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.events():
                if "augment_" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                    name = "horizontal" if "horizontal" in ev.name else "vertical"
                    kern[name] = kern.get(name, 0.0) + ev.device_time / 1e3 / a.iters
            emit(figure="kernel_per_batch", batch=B, size=224, kernels_ms={k: round(v, 4) for k, v in kern.items()},
                 call_event_ms=round(e0.elapsed_time(e1) / a.iters, 4), call_host_ms=round(wall * 1e3, 4),
                 packed_mb=round(host.numel() / 1e6, 2))

        # ---- worker CPU time per sample
        threads = torch.get_num_threads()
        torch.set_num_threads(1)                   # as in a DataLoader worker
        n = min(len(ref_ds), 256)

        def cpu_per_sample(fn):
            for k in range(min(n, 16)):
                fn(k)
            t0 = time.process_time()
            for k in range(n):
                fn(k)
            return (time.process_time() - t0) / n * 1e3
        decode = cpu_per_sample(lambda k: decode_ds[k])
        off = cpu_per_sample(lambda k: ref_ds[k])
        on = cpu_per_sample(lambda k: gpu_ds[k])
        samples = [gpu_ds[k] for k in range(128)]
        t0 = time.process_time()
        for _ in range(4):
            crop.collate(samples)
        pack = (time.process_time() - t0) / (4 * 128) * 1e3
        emit(figure="worker_cpu_ms_per_sample", decode=round(decode, 3), switch_off=round(off, 3),
             switch_on=round(on, 3), switch_on_collate=round(pack, 3),
             saving=round(off - on - pack, 3), augment_off=round(off - decode, 3), augment_on=round(on - decode + pack, 3))
        torch.set_num_threads(threads)

        # ---- DataLoader throughput
        from torch.utils.data import DataLoader
        for workers in (4, 10):
            warm = 2 * workers
            length = (warm + a.loader_batches + 1) * 128
            for name in ("off", "on"):
                ds = Cycle(ref_ds if name == "off" else gpu_ds, length)
                if name == "off":
                    loader = D.DeviceFeed(DataLoader(ds, batch_size=128, shuffle=True, num_workers=workers,
                                                     pin_memory=True, drop_last=True), dev)
                else:
                    loader = D._AugmentingDataLoader(ds, batch_size=128, shuffle=True, num_workers=workers,
                                                     pin_memory=True, drop_last=True,
                                                     collate_fn=gpu_ds.transform.collate)
                it = iter(loader)
                for _ in range(warm):               # the batches the workers prefetch
                    next(it)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                got = 0
                for _ in range(a.loader_batches):
                    x, _ = next(it)
                    got += x["rgb"].shape[0]
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                del it
                emit(figure="dataloader", workers=workers, switch=name, samples_per_s=round(got / dt, 1), batches=got // 128)
    emit(**gpu_info())


if __name__ == "__main__":
    main()
