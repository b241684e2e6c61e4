"""Time the grouped flat AdamW (multimae_b200.optim.GroupedFlatAdamW, MMAE_FLAT_ADAMW=1) against torch.optim.AdamW on
one GPU.

    python scripts/gpu_time_flat_adamw.py [--opt-steps 200] [--steps 20] [--warmup 5] [--rounds 3]

Prints one JSON line per figure:
  - the optimizer step alone over multivit_base + a 1000-class head (86.4 M trainable fp32 parameters) with the layer-decay
    groups of run_finetuning_cls.py (layer_decay 0.65, weight decay 0.05, 28 groups, lr / wd written into param_groups
    before every step as the script does): torch's default (foreach) AdamW, torch's fused=True AdamW (for context) and
    GroupedFlatAdamW, CUDA events over --opt-steps steps after warm-up, with GB/s against the 30 bytes per parameter a
    single pass must move (read p, g, m, v; write p, m, v and the bf16 twin);
  - the classification fine-tuning step at the shapes of gpu_time_finetune_cls.py (B = 128, 224 x 224, drop_path 0.1,
    soft-target cross-entropy, loss scaling) and the ConvNeXt semantic-segmentation step at the ADE20K shapes of
    gpu_time_finetune_semseg.py (B = 4, 512 x 512, 151 classes), each with the stock AdamW and with GroupedFlatAdamW over
    the script's groups; the two alternate in one process, --rounds times, and no step reads a value back to the host
    besides what the scaler does;
  - the GPU name, power limit and SM clocks, read in the same run."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet
BYTES_PER_PARAM = 30                # read p, g, m, v (16); write p, m, v (12) and the bf16 twin (2)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock, max_clock = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, power, clock, max_clock = torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"
    return dict(gpu=name, power_limit=power, sm_clock=clock, max_sm_clock=max_clock)


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


def factory():
    """The layer-decay groups of utils/optim_factory.py (the tests' stand-in restatement)."""
    spec = importlib.util.spec_from_file_location("_optim_factory",
                                                  os.path.join(ROOT, "tests", "adamw_standin", "utils", "optim_factory.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def script_groups(model, layer_decay=0.65, weight_decay=0.05):
    f = factory()
    lda = f.layer_decay_assigner(model, layer_decay)
    return f.get_parameter_groups(model, weight_decay, model.no_weight_decay(), lda.get_layer_id, lda.get_scale)


def schedule(opt, it):
    """run_finetuning_cls.py:503-508: lr and weight decay written into every group before each step."""
    for g in opt.param_groups:
        g["lr"] = 1e-4 * (0.999 ** it) * g["lr_scale"]
        if g["weight_decay"] > 0:
            g["weight_decay"] = 0.05


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--opt-steps", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    from cls_head_oracle import soft_target_ce
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import GroupedFlatAdamW
    from multimae_b200.output_adapters import ConvNeXtAdapter, LinearOutputAdapter

    dev = torch.device("cuda:0")
    emit(**gpu_info())
    mm.AUTO_OWN_GRADIENTS = True

    def cls_model(seed=0, drop_path_rate=0.0):
        torch.manual_seed(seed)
        return mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16,
                                                            image_size=224)},
                                {"cls": LinearOutputAdapter(1000)}, drop_path_rate=drop_path_rate).to(dev)

    # ---- 1. the optimizer step alone
    for kind in ("torch_foreach", "torch_fused", "flat"):
        model = cls_model()
        groups = script_groups(model)
        if kind == "flat":
            opt = GroupedFlatAdamW(groups, lr=1e-4, weight_decay=0.0)
        else:
            opt = torch.optim.AdamW(groups, lr=1e-4, weight_decay=0.0, fused=(kind == "torch_fused"))
        gen = torch.Generator(device=dev).manual_seed(1)
        for p in model.parameters():
            if p.requires_grad:
                g = torch.randn(p.shape, generator=gen, device=dev) * 1e-2
                if p.grad is None:
                    p.grad = g
                else:
                    p.grad.copy_(g)
        n = sum(p.numel() for p in model.parameters() if p.requires_grad)
        state = {"it": 0}

        def step():
            schedule(opt, state["it"])
            state["it"] += 1
            opt.step()
        ms = timed(step, args.opt_steps, 20)
        emit(figure="optimizer_step", optimizer=kind, params=n, groups=len(opt.param_groups), steps=args.opt_steps,
             us=round(ms * 1e3, 1), gbps_at_30_bytes_per_param=round(BYTES_PER_PARAM * n / (ms * 1e-3) / 1e9, 1),
             share_of_3_35_tbps=round(BYTES_PER_PARAM * n / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
        del opt, model, groups
        torch.cuda.empty_cache()

    # ---- 2. and 3. fine-tuning steps, stock and flat alternating
    def workload(name):
        if name == "cls":
            B = 128
            x = torch.randn(B, 3, 224, 224, device=dev)
            y = torch.randint(0, 1000, (B,), device=dev)
            t = torch.full((B, 1000), 0.1 / 1000, device=dev).scatter_(1, y[:, None], 0.9 + 0.1 / 1000)
            target = t * 0.7 + t.flip(0) * 0.3

            def build(seed):
                return cls_model(seed, drop_path_rate=0.1)

            def loss_of(model):
                return soft_target_ce(model(x)["cls"], target)
            return dict(batch=B, size=224), build, loss_of
        B, S, K = 4, 512, 151
        x = torch.randn(B, 3, S, S, device=dev)
        target = torch.randint(0, K, (B, S, S), device=dev)
        target[torch.rand(target.shape, device=dev) < 0.1] = 255
        crit = torch.nn.CrossEntropyLoss(ignore_index=255)

        def build(seed):
            torch.manual_seed(seed)
            return mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16,
                                                                image_size=S)},
                                    {"semseg": ConvNeXtAdapter(K, embed_dim=6144, preds_per_patch=16, depth=4)},
                                    drop_path_rate=0.1).to(dev)

        def loss_of(model):
            return crit(model(x)["semseg"], target)
        return dict(batch=B, size=S, classes=K), build, loss_of

    for name in ("cls", "semseg"):
        shape, build, loss_of = workload(name)
        runs = {}
        for kind in ("stock", "flat"):
            model = build(0)
            groups = script_groups(model)
            opt = (GroupedFlatAdamW if kind == "flat" else torch.optim.AdamW)(groups, lr=1e-4, weight_decay=0.0)
            scaler = NativeScalerWithGradNormCount()
            state = {"it": 0}

            def step(model=model, opt=opt, scaler=scaler, state=state):
                schedule(opt, state["it"])
                state["it"] += 1
                model.train()
                with torch.cuda.amp.autocast():
                    loss = loss_of(model)
                scaler(loss, opt, clip_grad=None, parameters=model.parameters())
                opt.zero_grad()
            runs[kind] = step
        res = {"stock": [], "flat": []}
        for _ in range(args.rounds):
            for kind in ("stock", "flat"):
                res[kind].append(timed(runs[kind], args.steps, args.warmup))
        med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
        for kind, v in res.items():
            emit(figure="%s_train_step" % name, optimizer=kind, ms_per_step=[round(t, 3) for t in v],
                 median_ms=round(med[kind], 3), spread_ms=round(max(v) - min(v), 3), **shape)
        emit(figure="%s_train_step_saving" % name, ms=round(med["stock"] - med["flat"], 3),
             ratio=round(med["stock"] / med["flat"], 3))
        del runs
        torch.cuda.empty_cache()
    emit(**gpu_info())


if __name__ == "__main__":
    main()
