"""Time the model EMA of classification fine-tuning (run_finetuning_cls.py --model_ema) on one GPU.

    python scripts/gpu_time_model_ema.py [--batch 128] [--steps 20] [--warmup 5] [--rounds 3] [--updates 200]

Workload: multivit_base on rgb at 224 x 224 with a 1000-class LinearOutputAdapter - 152 state_dict entries, 86,566,888
fp32 values.  One update has to read the EMA and the model and write the EMA: 12 bytes per value, 1.039 GB.

Prints one JSON line per figure:
  - the GPU name, power limit and maximum SM clock, read in the same run (first and last line);
  - one EMA update, CUDA events over --updates updates after a warm-up: the mmae_ema_update call alone (the kernel),
    multimae_b200.model_ema.ModelEma.update (the same launch plus its host work) and the reference's per-tensor torch
    loop (utils/model_ema.py:72-84, restated below: four kernels per entry), with achieved GB/s against the 1.039 GB
    minimum; and whether the ModelEma and loop EMAs are bitwise equal after the same updates;
  - the training step of gpu_time_finetune_cls.py (batch --batch, drop_path 0.1, soft-target cross-entropy, stock
    torch.optim.AdamW, NativeScalerWithGradNormCount with loss scaling) without EMA, with EMA through ModelEma and with
    EMA through the restated loop; the three alternate in one process, --rounds times, and the spread across rounds is
    reported."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from gpu_time_finetune_cls import HBM_BYTES_PER_S, gpu_info, soft_targets, timed  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def loop_update(ema_model, model, decay):
    """The reference's ModelEma.update body on one GPU (no '.module' prefix, no device move)."""
    with torch.no_grad():
        msd = model.state_dict()
        for k, ema_v in ema_model.state_dict().items():
            model_v = msd[k].detach()
            ema_v.copy_(ema_v * decay + (1. - decay) * model_v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--decay", type=float, default=0.9999)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    from cls_head_oracle import soft_target_ce
    from multimae_b200 import _lib as L
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.model_ema import ModelEma
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import LinearOutputAdapter

    dev = torch.device("cuda:0")
    emit(**gpu_info())
    B, C, decay = args.batch, args.classes, args.decay
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=224)},
                             {"cls": LinearOutputAdapter(C)}, drop_path_rate=0.1).to(dev)
    ema = ModelEma(model, decay=decay)
    ema_loop = ModelEma(model, decay=decay)               # a second copy for the restated loop
    sd = model.state_dict()
    values = sum(v.numel() for v in sd.values())
    min_bytes = 12 * values

    # ---- one update, both ways, on the same tensors' shapes; an equal number of updates keeps the two copies equal
    lib = L.lib()
    n0 = lib.mmae_launch_count()
    ema.update(model)
    launches = lib.mmae_launch_count() - n0
    loop_update(ema_loop.ema, model, decay)
    warm = max(20, args.updates // 10)
    t_update = timed(lambda: ema.update(model), args.updates, warm)
    t_loop = timed(lambda: loop_update(ema_loop.ema, model, decay), args.updates, warm)
    # the launch alone, with the pointer arrays ModelEma built: the kernel's own time (the host work of update() aside)
    ema_only = ModelEma(model, decay=decay)                # a third copy, so that the first two see equal update counts
    ema_only.update(model)
    _, dst, src, sizes = ema_only._args

    def kernel_only():
        L.check(lib.mmae_ema_update(dst, src, sizes, len(sd), float(decay), float(1.0 - decay), L.current_stream()))
    t_kernel = timed(kernel_only, args.updates, warm)
    for name, t, n in (("mmae_ema_update_call", t_kernel, launches), ("ModelEma.update", t_update, launches),
                       ("torch_loop", t_loop, 4 * len(sd))):
        emit(figure="ema_update", impl=name, entries=len(sd), values=values, launches_per_update=n, updates=args.updates,
             us=round(t * 1e3, 1), gbps_of_min_bytes=round(min_bytes / (t * 1e-3) / 1e9, 1), min_bytes=min_bytes,
             share_of_3_35_tbps=round(min_bytes / (t * 1e-3) / HBM_BYTES_PER_S, 3))
    e, r = ema.ema.state_dict(), ema_loop.ema.state_dict()
    emit(figure="ema_update_speedup", update_over_loop=round(t_loop / t_update, 2),
         bitwise_equal=all(torch.equal(e[k], r[k]) for k in e))
    del ema_only
    torch.cuda.empty_cache()

    # ---- the training step without EMA, with ModelEma, with the restated loop
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount()
    x = torch.randn(B, 3, 224, 224, device=dev)
    target = soft_targets(B, C, dev)

    def step(variant):
        model.train()
        with torch.cuda.amp.autocast():
            loss = soft_target_ce(model(x)["cls"], target)
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())
        opt.zero_grad()
        if variant == "ema_model_ema_kernel":
            ema.update(model)
        elif variant == "ema_torch_loop":
            loop_update(ema_loop.ema, model, decay)

    variants = ("no_ema", "ema_model_ema_kernel", "ema_torch_loop")
    res = {v: [] for v in variants}
    for _ in range(args.rounds):
        for v in variants:
            res[v].append(timed(lambda v=v: step(v), args.steps, args.warmup))
    med = {}
    for v, ts in res.items():
        med[v] = sorted(ts)[len(ts) // 2]
        emit(figure="train_step", variant=v, batch=B, ms_per_step=[round(t, 3) for t in ts], median_ms=round(med[v], 3),
             spread_ms=round(max(ts) - min(ts), 3))
    for v in variants[1:]:
        emit(figure="train_step_ema_cost", variant=v, median_ms_over_no_ema=round(med[v] - med["no_ema"], 3),
             share_of_step=round((med[v] - med["no_ema"]) / med["no_ema"], 4))
    emit(**gpu_info())


if __name__ == "__main__":
    main()
