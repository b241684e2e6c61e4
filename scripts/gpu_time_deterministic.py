"""Cost of deterministic mode (torch.use_deterministic_algorithms) on one GPU.

    python scripts/gpu_time_deterministic.py [--batch 128] [--cls-batch 128] [--steps 20] [--warmup 5] [--rounds 3]

Two workloads, each timed with the mode off and on, alternating in one process for --rounds rounds:
  - the bench's pre-training step (bench.py cfg2: MultiMAE-B, rgb + depth + semseg in, four decoders, FlatAdamW),
    replayed as one CUDA graph; the graph of each mode is captured with that mode set, after eager warm-up steps;
  - the classification fine-tuning step (MultiViT-B/16 on rgb at 224 x 224, 1000 classes, stock torch.optim.AdamW and
    NativeScalerWithGradNormCount under bf16 autocast), run eagerly as the fine-tuning script does.
torch's own ops run with warn_only=True: the point is the library's ordered forms, not torch's.

Prints one JSON line per figure: ms per step for each mode and round, the on / off ratio of the medians, and the GPU
name, power limit and maximum SM clock, read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def set_mode(on):
    from multimae_b200 import functional as Fn
    torch.use_deterministic_algorithms(on, warn_only=True)
    Fn.sync_deterministic()


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def pretrain_steps(batch):
    """{mode: callable replaying that mode's captured graph}"""
    import bench
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model, loss_fns = bench.build_model_and_losses(dev, "base", 224)
    opt = FlatAdamW(model, lr=1e-4 * batch / 256, betas=(0.9, 0.95), weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
    x = {k: v.to(dev) for k, v in bench.synthetic_batch(batch, 0).items()}
    steps = {}
    for on in (False, True):
        set_mode(on)
        st = TrainStep(model, loss_fns, opt, scaler, num_encoded_tokens=98, alphas=1.0, loss_sources={"norm_rgb": "rgb"})
        st.capture(x)
        steps[on] = (lambda s: lambda: s(x))(st)
    return steps


def cls_step(batch):
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import LinearOutputAdapter
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=224)},
                             {"cls": LinearOutputAdapter(1000)}, drop_path_rate=0.1).to(dev)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount()
    x = torch.randn(batch, 3, 224, 224, device=dev)
    y = torch.randint(0, 1000, (batch,), device=dev)

    def step():
        model.train()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(model({"rgb": x})["cls"].float(), y)
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())
        opt.zero_grad()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128, help="pre-training batch (the bench's)")
    ap.add_argument("--cls-batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this script measures on the GPU"
    emit(**gpu_info())
    work = {"pretrain_graph": pretrain_steps(args.batch)}
    cls = cls_step(args.cls_batch)
    work["cls_finetune"] = {False: cls, True: cls}     # eager: the mode is whatever is set when it runs
    times = {(w, on): [] for w in work for on in (False, True)}
    for r in range(args.rounds):
        for w, fns in work.items():
            for on in (False, True):
                set_mode(on)
                ms = timed(fns[on], args.steps, args.warmup)
                times[(w, on)].append(ms)
                emit(workload=w, deterministic=on, round=r, ms_per_step=round(ms, 3))
    set_mode(False)
    for w in work:
        off, on = statistics.median(times[(w, False)]), statistics.median(times[(w, True)])
        emit(workload=w, median_ms_off=round(off, 3), median_ms_on=round(on, 3), on_over_off=round(on / off, 4))


if __name__ == "__main__":
    main()
