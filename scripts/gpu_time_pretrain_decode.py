"""Time the GPU decode of pre-training images (MMAE_GPU_JPEG with MMAE_GPU_AUGMENT, mmae_png_decode_batch and
mmae_jpeg_decode_batch) on one GPU.

    python scripts/gpu_time_pretrain_decode.py [--images 256] [--iters 20] [--loader-batches 12] [--steps 20] [--rounds 3]

A seeded folder tree of ImageNet-like sizes (400 to 500 x 300 to 400): rgb as quality-90 JPEGs, depth as 16-bit
PNGs, semseg as 8-bit palette PNGs, written with Pillow's defaults; input size 224.  "before" is MMAE_GPU_AUGMENT
alone (the workers decode with Pillow), "after" adds the GPU decode (CompressedMultiTaskImages).

Prints one JSON line per figure:
  - the GPU name, power limit and SM clocks, read in the same run;
  - per batch of 128 and per domain, each decode kernel's device time from torch.profiler over --iters calls;
  - per PNG domain: how many streams took the parallel inflate, the decode call's time, and with --baseline-lib the
    same call of an earlier build of the library on the same packed batch, alternating, with both outputs compared;
  - worker CPU time per sample (process time, one torch thread, in this process), before and after;
  - DataLoader samples/s at batch 128 with 10 workers, before and after, batches ending on the GPU: the first
    20 batches (what the workers prefetch) are not timed, the next --loader-batches are;
  - the benchmark's pre-training step (bench.py's model and TrainStep, batch 128, eager) alone, and with a batch's
    upload + decode + resampling running back to back on a second stream beside it, as the loader's copy stream runs
    it: CUDA events on each stream; --rounds rounds of --steps steps, alone and beside alternating."""
import argparse
import json
import os
import random
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "augment_standin")]

import augment_oracle as AO  # noqa: E402
from multimae_b200 import data as D  # noqa: E402
from multimae_b200 import kernels  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def write_tree(root, n, seed=0):
    rng = np.random.default_rng(seed)
    for k in range(n):
        h, w = int(rng.integers(300, 401)), int(rng.integers(400, 501))
        imgs = AO.make_images(int(rng.integers(1 << 30)), h, w)
        imgs["semseg"].putpalette(list(range(256)) * 3)
        for task, img, ext in (("rgb", imgs["rgb"], ".jpg"), ("depth", imgs["depth"], ".png"),
                               ("semseg", imgs["semseg"], ".png")):
            os.makedirs(os.path.join(root, task, "c%d" % (k % 4)), exist_ok=True)
            path = os.path.join(root, task, "c%d" % (k % 4), "img%04d%s" % (k, ext))
            img.save(path, quality=90) if ext == ".jpg" else img.save(path)


class Args:
    def __init__(self, data_path):
        self.input_size, self.hflip, self.imagenet_default_mean_and_std = 224, 0.5, True
        self.data_path, self.all_domains = data_path, ["rgb", "depth", "semseg"]


def per_sample_cpu(ds, n):
    torch.set_num_threads(1)
    t0 = time.process_time()
    for i in range(n):
        ds[i % len(ds)]
    return (time.process_time() - t0) / n * 1e3


class Cycle(torch.utils.data.Dataset):
    """`n` samples of `ds`, index modulo its length (the timed window outlasts the folder)."""

    def __init__(self, ds, n):
        self.ds, self.n, self.transform = ds, n, ds.transform

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return self.ds[i % len(self.ds)]


def loader_rate(ds, batches, workers=10):
    """Steady-state samples/s: the first 2 x workers batches (what the workers prefetch, built before the clock could
    start) are not timed, the next `batches` are."""
    skip = 2 * workers
    loader = D._AugmentingDataLoader(Cycle(ds, (batches + skip) * 128), batch_size=128, shuffle=True,
                                     num_workers=workers, drop_last=True, pin_memory=True, persistent_workers=False)
    it = iter(loader)
    for _ in range(skip):
        next(it)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(batches):
        next(it)
    torch.cuda.synchronize()
    return batches * 128 / (time.perf_counter() - t0)


def baseline_png_call(path):
    """mmae_png_decode_batch of the library at `path` (an earlier commit's), on this batch's packing and scratch size."""
    import ctypes
    from multimae_b200 import _lib as L
    f = ctypes.CDLL(path).mmae_png_decode_batch
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int64,
                  ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]

    def call(host, dev, desc_offset, num_images, raw_bytes):
        scratch = torch.empty(max(raw_bytes, 16), dtype=torch.uint8, device=dev.device)
        status = torch.empty(num_images, dtype=torch.int32, device=dev.device)
        assert f(host.data_ptr(), dev.data_ptr(), host.numel(), dev.numel(), num_images, desc_offset,
                 scratch.data_ptr(), max(raw_bytes, 16), status.data_ptr(), L.current_stream()) == 0
        return status
    return call


def png_paths(host, png_args, scratch):
    """{path: streams} of one decode: 'one warp' (under the size threshold), or the parallel inflate's stream state."""
    from multimae_b200 import png as P
    off, n, _ = png_args
    pd = host.numpy()[off * 16:].view(np.int32)[:n * D.PNG_FIELDS].reshape(n, D.PNG_FIELDS)
    sc = scratch.cpu().numpy()
    names = {P.PATH_PARALLEL: "parallel", P.PATH_WALK: "fallback_walk", P.PATH_BOUND: "fallback_bound",
             P.PATH_EXPAND: "fallback_expand", P.PATH_RESOLVE: "fallback_resolve"}
    out = {}
    for d in pd:
        k = "one_warp" if not d[14] else names.get(int(sc[d[14] * 16:d[14] * 16 + 4].view(np.int32)[0]), "unknown")
        out[k] = out.get(k, 0) + 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--loader-batches", type=int, default=12)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--baseline-lib", default=None,
                    help="also time mmae_jpeg_decode_batch and mmae_png_decode_batch of this build of the "
                         "library (an earlier commit's)")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    emit(gpu=torch.cuda.get_device_name(0), nvidia_smi=q)
    import utils.datasets as ud
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, a.images)
        args = Args(root)
        before = D.build_gpu_augment_dataset(args, ud.build_multimae_pretraining_dataset)
        after = D.build_gpu_augment_dataset(args, ud.build_multimae_pretraining_dataset, compressed=True)
        random.seed(0)
        torch.manual_seed(0)
        packed = after.transform.collate([after[i] for i in range(128)])[0]
        host = packed.buffer.pin_memory()
        tail = torch.empty(packed.device_bytes, dtype=torch.uint8, device=dev)
        tail[:host.numel()].copy_(host)

        def decode():
            kernels.jpeg_decode_batch(host, tail, *packed.jpeg)
            return kernels.png_decode_batch(host, tail, *packed.png)
        assert int(decode().abs().sum()) == 0
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.iters):
                decode()
            torch.cuda.synchronize()
        kt = {}
        for e in prof.key_averages():
            m = re.search(r"(png|jpeg)_\w+_kernel", e.key)
            if m:
                kt[m.group(0)] = kt.get(m.group(0), 0.0) + e.device_time_total / 1e3 / a.iters
        emit(figure="decode kernels per batch of 128 (ms)", batch=128, png_images=packed.png[1],
             jpeg_images=packed.jpeg[1], kernels=kt)
        if a.baseline_lib:
            import gpu_time_jpeg_decode as G
            base = G.baseline_call(a.baseline_lib)
            tail[host.numel():].zero_()
            decode()
            ours = tail.clone()
            tail[host.numel():].zero_()
            base(host, tail, *packed.jpeg)
            kernels.png_decode_batch(host, tail, *packed.png)
            torch.cuda.synchronize()
            times = {"this": [], "baseline": []}
            for _ in range(3):
                times["this"].append(round(G.time_calls(lambda: kernels.jpeg_decode_batch(host, tail, *packed.jpeg),
                                                        a.iters), 4))
                times["baseline"].append(round(G.time_calls(lambda: base(host, tail, *packed.jpeg), a.iters), 4))
            emit(figure="jpeg decode call per batch of 128 (ms) vs baseline", call_event_ms=times,
                 bitwise_equal=bool(torch.equal(ours, tail)))
        for task in ("depth", "semseg"):
            rects = [after[i][0].arrays[task] for i in range(128)]
            sub = [D.Crops({task: r}, False, *r[1][2:]) for r in rects]
            pb = D.pack_batch(sub, 224, (0.5,) * 3, (0.5,) * 3)
            h2 = pb.buffer.pin_memory()
            t2 = torch.empty(pb.device_bytes, dtype=torch.uint8, device=dev)
            t2[:h2.numel()].copy_(h2)
            scratch = torch.empty(max(pb.png[2], 16), dtype=torch.uint8, device=dev)
            status = kernels.png_decode_batch(h2, t2, *pb.png, scratch=scratch).cpu()
            emit(figure="png streams per batch of 128 by path", task=task, **png_paths(h2, pb.png, scratch),
                 nonzero_status=int(status.ne(0).sum()))
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.iters):
                kernels.png_decode_batch(h2, t2, *pb.png)
            e.record()
            torch.cuda.synchronize()
            emit(figure="png decode per batch of 128, CUDA events (ms)", task=task, ms=s.elapsed_time(e) / a.iters)
            if a.baseline_lib:
                base = baseline_png_call(a.baseline_lib)
                t2[h2.numel():].zero_()
                kernels.png_decode_batch(h2, t2, *pb.png)
                ours = t2.clone()
                t2[h2.numel():].zero_()
                base(h2, t2, *pb.png)
                torch.cuda.synchronize()
                import gpu_time_jpeg_decode as G
                times = {"this": [], "baseline": []}
                for _ in range(3):
                    times["this"].append(round(G.time_calls(lambda: kernels.png_decode_batch(h2, t2, *pb.png),
                                                            a.iters), 3))
                    times["baseline"].append(round(G.time_calls(lambda: base(h2, t2, *pb.png), a.iters), 3))
                emit(figure="png decode call per batch of 128 (ms) vs baseline", task=task, call_event_ms=times,
                     bitwise_equal=bool(torch.equal(ours, t2)))
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(a.iters):
                        kernels.png_decode_batch(h2, t2, *pb.png)
                    torch.cuda.synchronize()
                kt = {}
                for ev_ in prof.key_averages():
                    m = re.search(r"png_\w+_kernel", ev_.key)
                    if m:
                        kt[m.group(0)] = round(kt.get(m.group(0), 0.0) + ev_.device_time_total / 1e3 / a.iters, 3)
                emit(figure="png kernels per batch of 128 (ms)", task=task, kernels=kt)
        emit(figure="worker CPU per sample (ms)", before=per_sample_cpu(before, 64), after=per_sample_cpu(after, 64))
        torch.set_num_threads(min(16, os.cpu_count() or 1))
        emit(figure="DataLoader samples/s, batch 128, 10 workers", before=loader_rate(before, a.loader_batches),
             after=loader_rate(after, a.loader_batches))

        import bench
        from multimae_b200.native_scaler import NativeScalerWithGradNormCount
        from multimae_b200.optim import FlatAdamW
        from multimae_b200.train_step import TrainStep
        torch.manual_seed(0)
        model, losses = bench.build_model_and_losses(dev)
        opt = FlatAdamW(model, lr=1e-4 * 128 / 256, betas=(0.9, 0.95), weight_decay=0.05)
        scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
        stepper = TrainStep(model, losses, opt, scaler, num_encoded_tokens=98, alphas=1.0,
                            loss_sources={"norm_rgb": "rgb"})
        x = {k: v.to(dev) for k, v in bench.synthetic_batch(128, 0).items()}
        side = torch.cuda.Stream(dev)

        def feed():                          # what DeviceFeed runs on its copy stream for one batch
            packed.to_device(dev)
        ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
        for _ in range(3):
            stepper(x)
            with torch.cuda.stream(side):
                feed()
        torch.cuda.synchronize()
        for r in range(a.rounds):
            row = {}
            for beside in (False, True):
                s0, s1 = ev(), ev()
                s0.record()
                for _ in range(a.steps):
                    stepper(x)
                    if beside:
                        with torch.cuda.stream(side):
                            feed()
                s1.record()
                torch.cuda.synchronize()
                row["step_ms_beside" if beside else "step_ms_alone"] = s0.elapsed_time(s1) / a.steps
            emit(figure="pre-training step, batch 128 (ms)", round=r, **row)
    emit(gpu=torch.cuda.get_device_name(0), nvidia_smi=subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
        capture_output=True, text=True).stdout.strip())


if __name__ == "__main__":
    main()
