"""Cost of stochastic depth on the MultiMAE-B pre-training step: batch 128, graph-captured TrainStep, drop_path_rate 0
against 0.1 (encoder and decoders), the two settings alternating in one process after warm-up.

    python scripts/gpu_time_drop_path.py [--rounds 5] [--steps 20]

Both graphs are captured from one model (the rate only changes the scale arguments of the recorded block calls).  Each timed
window is bracketed by device synchronisations; prints ms/step per setting (median over rounds), GPU name and power limit."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    from bench import build_model_and_losses, synthetic_batch
    from multimae_b200.multimae_utils import DropPath
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model, loss_fns = build_model_and_losses(dev)
    opt = FlatAdamW(model, lr=1e-4 * args.batch / 256, betas=(0.9, 0.95), weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
    x = {k: v.to(dev) for k, v in synthetic_batch(args.batch, 0).items()}
    stacks = [model.encoder] + [ad.decoder_transformer for ad in model.output_adapters.values()]

    def set_rate(rate):
        for blocks in stacks:
            dpr = [v.item() for v in torch.linspace(0, rate, len(blocks))]
            for b, p in zip(blocks, dpr):
                b.drop_path = DropPath(p) if p > 0 else torch.nn.Identity()

    steps = {}
    for rate in (0.0, 0.1):
        set_rate(rate)
        steps[rate] = TrainStep(model, loss_fns, opt, scaler, num_encoded_tokens=98, alphas=1.0,
                                loss_sources={"norm_rgb": "rgb"}).capture(x, warmup=3)
    for rate, st in steps.items():                       # warm-up replays of both graphs
        for _ in range(5):
            st(x)
    times = {r: [] for r in steps}
    for _ in range(args.rounds):
        for rate, st in steps.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                loss, _ = st(x)
            torch.cuda.synchronize()
            times[rate].append((time.perf_counter() - t0) * 1e3 / args.steps)
    assert all(bool(torch.isfinite(st.static_out[0])) for st in steps.values())
    print("# %s, batch %d, %d rounds x %d graph replays per setting" % (gpu, args.batch, args.rounds, args.steps))
    base = statistics.median(times[0.0])
    for rate in steps:
        med = statistics.median(times[rate])
        print("drop_path_rate %.1f: %.2f ms/step (median; rounds %s)  %+.2f %%" %
              (rate, med, " ".join("%.2f" % t for t in times[rate]), 100.0 * (med - base) / base))


if __name__ == "__main__":
    main()
