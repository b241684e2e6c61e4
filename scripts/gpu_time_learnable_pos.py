"""Cost of trainable position tables (learnable_pos_emb=True) against frozen ones, on one GPU.

    python scripts/gpu_time_learnable_pos.py [--steps 20] [--warmup 5] [--rounds 3] [--skip-pretrain]

Two workloads, each built twice (frozen tables / trainable tables, same seed) and timed alternately in one process,
--rounds times, with CUDA events:
  - semseg: run_finetuning_semseg.py's train_one_epoch body on the ADE config: MultiViT-B/16 on rgb at 512 x 512, batch 4,
    drop_path 0.1, ConvNeXtAdapter(151 classes, embed_dim 6144, preds_per_patch 16, depth 4), fp16 autocast, the stock
    torch.optim.AdamW and NativeScalerWithGradNormCount (the table is 32 x 32 x 768, resized by the identity);
  - pretrain: bench.py's workload (MultiMAE-B, rgb + depth + semseg at 224 x 224, batch 128, 98 visible tokens, four
    decoders, FlatAdamW), each step replayed as one CUDA graph (TrainStep.capture) like bench.py does; three 14 x 14 tables.
Prints one JSON line per figure, and the GPU name and power limit read in the same run."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from gpu_time_finetune_semseg import emit, gpu_info, timed  # noqa: E402


def semseg_pair(dev, B=4, S=512, K=151):
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import ConvNeXtAdapter
    mm.AUTO_OWN_GRADIENTS = True
    crit = torch.nn.CrossEntropyLoss(ignore_index=255)
    x = torch.randn(B, 3, S, S, device=dev)
    target = torch.randint(0, K, (B, S, S), device=dev)
    target[torch.rand(target.shape, device=dev) < 0.1] = 255
    steps = {}
    for learnable in (False, True):
        torch.manual_seed(0)
        model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=S,
                                                             learnable_pos_emb=learnable)},
                                 {"semseg": ConvNeXtAdapter(K, embed_dim=6144, preds_per_patch=16, depth=4)},
                                 drop_path_rate=0.1).to(dev)
        opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
        scaler = NativeScalerWithGradNormCount()

        def step(model=model, opt=opt, scaler=scaler):
            model.train()
            with torch.cuda.amp.autocast():
                loss = crit(model(x)["semseg"], target)
            scaler(loss, opt, clip_grad=None, parameters=model.parameters())
            opt.zero_grad()
        steps["trainable" if learnable else "frozen"] = step
    return steps


def pretrain_pair(dev, B=128):
    import bench
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep
    x = {k: v.to(dev) for k, v in bench.synthetic_batch(B, 0).items()}
    steps = {}
    for learnable in (False, True):
        torch.manual_seed(0)
        model, loss_fns = bench.build_model_and_losses(dev)
        if learnable:
            for ad in model.input_adapters.values():
                ad.pos_emb.requires_grad_(True)
        opt = FlatAdamW(model, lr=1e-4 * B / 256, betas=(0.9, 0.95), weight_decay=0.05)
        scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
        stepper = TrainStep(model, loss_fns, opt, scaler, num_encoded_tokens=98, alphas=1.0, loss_sources={"norm_rgb": "rgb"})
        stepper.capture(x, warmup=3)
        steps["trainable" if learnable else "frozen"] = lambda stepper=stepper: stepper(x)
    return steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-pretrain", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    dev = torch.device("cuda:0")
    emit(**gpu_info())
    workloads = [("semseg_ade_b4_512", semseg_pair)] + ([] if args.skip_pretrain else [("pretrain_bench_b128", pretrain_pair)])
    for name, make in workloads:
        steps = make(dev)
        res = {k: [] for k in steps}
        for _ in range(args.rounds):
            for k, fn in steps.items():
                res[k].append(timed(fn, args.steps, args.warmup))
        med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
        for k, v in res.items():
            emit(workload=name, tables=k, ms_per_step=[round(t, 3) for t in v], median_ms=round(med[k], 3))
        emit(workload=name, overhead_pct=round(100.0 * (med["trainable"] / med["frozen"] - 1.0), 2))
        del steps
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
