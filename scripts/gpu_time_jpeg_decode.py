"""Time the GPU JPEG decode of classification fine-tuning (MMAE_GPU_AUGMENT, mmae_jpeg_decode_batch) on one GPU.

    python scripts/gpu_time_jpeg_decode.py [--images 512] [--iters 50] [--loader-batches 24] [--steps 20] [--rounds 3]
                                           [--restart-rows N] [--baseline-lib PATH]

Same images and config as scripts/gpu_time_cls_augment.py: a seeded folder of quality-90 4:2:0 JPEGs of 300 to 600
pixels per side, input 224, --aa rand-m9-mstd0.5-inc1, bicubic, eval crop_pct 0.875.  "before" is the switch as it
was (the workers decode with Pillow, the GPU resamples), "after" adds the GPU decode (jpeg_loader).

Prints one JSON line per figure:
  - the GPU name, power limit, current and maximum SM clock, read in the same run (first and last line);
  - mmae_jpeg_decode_batch per batch of 128, train and eval: each kernel's device time from torch.profiler over --iters
    calls, and CUDA events around the whole call (scratch allocation and the host's checks included), after a warm-up;
  - worker CPU time per sample (process time, one torch thread), before and after, and the packing per sample;
  - DataLoader samples/s at batch 128 with 10 workers, before and after, batches ending on the GPU (as in
    scripts/gpu_time_cls_augment.py);
  - the classification training step of scripts/gpu_time_finetune_cls.py (multivit_base + LinearOutputAdapter, batch
    128, 224 x 224, drop_path 0.1, bf16 autocast, AdamW) alone, and with the train batch's decode running back to back
    on a second stream beside it, as a loader's copy stream would: CUDA events on each stream give the step's time and
    the decode's time per call; --rounds rounds of --steps steps, alone and beside alternating.  The decode is kept
    busy for the whole window (its calls are queued ahead of the steps).

--restart-rows N writes the JPEGs with a restart marker every N MCU rows.  --baseline-lib runs mmae_jpeg_decode_batch
of another build of the library (an earlier commit's) on the same packed batches, alternating with this one, and
reports both calls' CUDA-event times and whether their decoded rectangles are bitwise equal."""
import argparse
import functools
import os
import random
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import gpu_time_cls_augment as C  # noqa: E402  (puts the repository, tests/ and the stand-in on sys.path)
import gpu_time_finetune_cls as F  # noqa: E402
from multimae_b200 import data as D  # noqa: E402
from multimae_b200 import kernels  # noqa: E402


def datasets(ud, stock, root, is_train):
    """(before, after): the switch's dataset with Pillow's loader, and with jpeg_loader."""
    ud.build_transform = functools.partial(D.build_gpu_cls_transform, stock=stock)
    before, _ = ud.build_dataset(is_train, C.args_for(root))
    after, _ = D.build_gpu_cls_dataset(is_train, C.args_for(root), ud.build_dataset)
    return before, after


def step_beside_decode(decode, steps, rounds, dev):
    """(step ms alone, step ms beside the decode, decode ms per call beside the step) per round."""
    from cls_head_oracle import soft_target_ce
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import LinearOutputAdapter
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16,
                                                         image_size=224)},
                             {"cls": LinearOutputAdapter(1000)}, drop_path_rate=0.1).to(dev)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount()
    x = torch.randn(128, 3, 224, 224, device=dev)
    target = F.soft_targets(128, 1000, dev)

    def step():
        model.train()
        with torch.cuda.amp.autocast():
            loss = soft_target_ce(model(x)["cls"], target)
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())
        opt.zero_grad()
    side = torch.cuda.Stream(dev)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    for _ in range(5):
        step()
        with torch.cuda.stream(side):
            decode()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        row = []
        for beside in (False, True):
            calls = 0
            if beside:                                   # enough decodes queued to outlast the steps
                d0 = ev()
                with torch.cuda.stream(side):
                    d0.record()
                    while calls * 40 < steps * 100:      # decode >= 40 ms a call against a step <= 100 ms
                        decode()
                        calls += 1
                    d1 = ev()
                    d1.record()
            s0, s1 = ev(), ev()
            s0.record()
            for _ in range(steps):
                step()
            s1.record()
            torch.cuda.synchronize()
            row.append(s0.elapsed_time(s1) / steps)
            if beside:
                row.append(d0.elapsed_time(d1) / calls)
        out.append(row)
    return out


def write_tree(root, n, restart_rows, seed=0):
    """C.write_tree's images, optionally with restart markers."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    for k in range(n):
        d = os.path.join(root, "class_%d" % (k % 4))
        os.makedirs(d, exist_ok=True)
        h, w = int(rng.integers(300, 601)), int(rng.integers(300, 601))
        Image.fromarray(C.O.make_image(int(rng.integers(1 << 30)), h, w)).save(
            os.path.join(d, "%05d.jpg" % k), quality=90, **({"restart_marker_rows": restart_rows} if restart_rows else {}))


def baseline_call(path):
    """mmae_jpeg_decode_batch of the library at `path`, as kernels.jpeg_decode_batch calls it (same scratch size)."""
    import ctypes
    from multimae_b200 import _lib as L
    lib = ctypes.CDLL(path)
    f = lib.mmae_jpeg_decode_batch
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int64,
                  ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]

    def call(host, dev, desc_offset, num_images, coef_blocks, plane_bytes):
        n = kernels.jpeg_scratch_bytes(coef_blocks, plane_bytes,
                                       kernels.jpeg_subsequence_slots(host, desc_offset, num_images))
        scratch = torch.empty(n, dtype=torch.uint8, device=dev.device)
        assert f(host.data_ptr(), dev.data_ptr(), host.numel(), dev.numel(), num_images, desc_offset,
                 scratch.data_ptr(), n, L.current_stream()) == 0
    return call


def time_calls(call, iters):
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        call()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--restart-rows", type=int, default=0)
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--loader-batches", type=int, default=24)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this script measures on a CUDA device"
    dev = torch.device("cuda:0")
    C.emit(**C.gpu_info())
    import utils.datasets as ud
    stock = ud.build_transform
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, a.images, a.restart_rows)
        base = baseline_call(a.baseline_lib) if a.baseline_lib else None
        for is_train in (True, False):
            _, ds = datasets(ud, stock, root, is_train)
            random.seed(0)
            np.random.seed(0)
            torch.manual_seed(0)
            packed, _ = ds.transform.collate([ds[k] for k in range(128)])
            assert packed.jpeg is not None and packed.jpeg[1] == 128
            host = packed.buffer.pin_memory()
            devbuf = torch.empty(packed.device_bytes, dtype=torch.uint8, device=dev)
            devbuf[:host.numel()].copy_(host)

            def call():
                kernels.jpeg_decode_batch(host, devbuf, *packed.jpeg)
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
                if ev.device_type == torch.autograd.DeviceType.CUDA and "jpeg_" in ev.name:
                    name = next(k for k in ("parallel", "entropy", "idct", "color") if k in ev.name)
                    kern[name] = kern.get(name, 0.0) + ev.device_time / 1e3 / a.iters
            if base is not None:
                devbuf[host.numel():].zero_()
                call()
                ours = devbuf.clone()
                devbuf[host.numel():].zero_()
                base(host, devbuf, *packed.jpeg)
                torch.cuda.synchronize()
                same = bool(torch.equal(ours[host.numel():], devbuf[host.numel():]))
                times = {"this": [], "baseline": []}
                for _ in range(3):
                    times["this"].append(round(time_calls(call, a.iters), 4))
                    times["baseline"].append(round(time_calls(lambda: base(host, devbuf, *packed.jpeg), a.iters), 4))
                C.emit(figure="decode_call_ms_vs_baseline", transform="train" if is_train else "eval", batch=128,
                       restart_rows=a.restart_rows, call_event_ms=times, bitwise_equal=same)
            if is_train:
                rounds = step_beside_decode(call, a.steps, a.rounds, dev)
                C.emit(figure="step_beside_decode", batch=128, steps=a.steps,
                       step_ms_alone=[round(r[0], 3) for r in rounds], step_ms_beside=[round(r[1], 3) for r in rounds],
                       decode_ms_per_call_beside=[round(r[2], 3) for r in rounds])
            C.emit(figure="decode_per_batch", transform="train" if is_train else "eval", batch=128,
                   restart_rows=a.restart_rows,
                   kernels_ms={k: round(v, 4) for k, v in kern.items()}, kernels_total_ms=round(sum(kern.values()), 4),
                   call_event_ms=round(t0.elapsed_time(t1) / a.iters, 4), iters=a.iters,
                   compressed_bytes=int(sum(int(x) for x in host.numpy()[packed.jpeg[0] * 16:].view(np.int32)[
                       7:packed.jpeg[1] * D.JPEG_FIELDS:D.JPEG_FIELDS])),
                   decoded_bytes=int(packed.device_bytes - host.numel()))
        torch.set_num_threads(1)
        for is_train in (True, False):
            before, after = datasets(ud, stock, root, is_train)
            n = min(len(before), 256)
            res = {}
            for name, ds in (("before", before), ("after", after)):
                for k in range(16):
                    ds[k]
                c0 = time.process_time()
                items = [ds[k] for k in range(n)]
                res[name] = (time.process_time() - c0) / n * 1e3
                c0 = time.process_time()
                for b in range(0, n - 127, 128):
                    ds.transform.collate(items[b:b + 128])
                res["pack_" + name] = (time.process_time() - c0) / (n // 128 * 128) * 1e3
            C.emit(figure="worker_cpu_ms_per_sample", transform="train" if is_train else "eval", samples=n,
                   **{k: round(v, 4) for k, v in res.items()})
        torch.set_num_threads(min(16, os.cpu_count() or 1))
        workers = 10
        need = 2 * workers + a.loader_batches
        for name, k in (("before", 0), ("after", 1)):
            ds = C.Cycle(datasets(ud, stock, root, True)[k], need * 128)
            loader = D._AugmentingDataLoader(ds, batch_size=128, shuffle=True, num_workers=workers, drop_last=True,
                                             pin_memory=True)
            got, t0 = 0, None
            for x, y in loader:
                got += 1
                if got == 2 * workers:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
            torch.cuda.synchronize()
            assert got == need
            C.emit(figure="dataloader_samples_per_s", decode=name, workers=workers, batch=128, cpus=os.cpu_count(),
                   samples_per_s=round(a.loader_batches * 128 / (time.perf_counter() - t0), 1),
                   timed_batches=a.loader_batches)
    C.emit(**C.gpu_info())


if __name__ == "__main__":
    main()
