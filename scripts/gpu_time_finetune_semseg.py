"""Time semantic-segmentation fine-tuning (run_finetuning_semseg.py, ADE20K config) on one GPU.

    python scripts/gpu_time_finetune_semseg.py [--batch 4] [--classes 150] [--steps 10] [--warmup 3] [--rounds 3]

Workload: MultiViT-B/16 on rgb at 512 x 512 (1025 encoder tokens), drop_path 0.1, ConvNeXtAdapter(150 + 1 void classes,
embed_dim 6144, preds_per_patch 16, depth 4), CrossEntropyLoss(ignore_index=255), the stock torch.optim.AdamW and
NativeScalerWithGradNormCount with loss scaling - the script's train_one_epoch body under the overlay.

Prints one JSON line per figure:
  - train step time and eval forward time (torch.no_grad, model.eval()) of this package;
  - the same for torch eager under bf16 autocast: the oracle's encoder (no stochastic depth) plus the adapter restated in
    torch (tests/convnext_head_oracle.py, channels-first cuDNN depthwise conv), on the same parameter values; the two
    alternate in one process, --rounds times;
  - per kernel (torch.profiler, a separate pass over the head alone): depthwise conv forward / backward and upsample
    forward / backward with the bytes each must move and the achieved GB/s against the H100 SXM's 3.35 TB/s; the head's
    GEMMs (forward + backward) as TFLOP/s from mmae_profile_gemm;
  - the GPU name, power limit and maximum SM clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--classes", type=int, default=150)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    from cls_head_oracle import vit_config
    from convnext_head_oracle import convnext_head
    from multimae_b200 import _lib as L
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import ConvNeXtAdapter
    from oracle import multimae_oracle as O

    dev = torch.device("cuda:0")
    emit(**gpu_info())
    B, S, K = args.batch, args.size, args.classes + 1
    n = (S // 16) ** 2
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=S)},
                             {"semseg": ConvNeXtAdapter(K, embed_dim=6144, preds_per_patch=16, depth=4)},
                             drop_path_rate=0.1).to(dev)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount()
    crit = torch.nn.CrossEntropyLoss(ignore_index=255)
    x = torch.randn(B, 3, S, S, device=dev)
    target = torch.randint(0, K, (B, S, S), device=dev)
    target[torch.rand(target.shape, device=dev) < 0.1] = 255

    def ours_step():
        model.train()
        with torch.cuda.amp.autocast():
            loss = crit(model(x)["semseg"], target)
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())
        opt.zero_grad()

    def ours_eval():
        model.eval()
        with torch.no_grad(), torch.cuda.amp.autocast():
            model(x)["semseg"]

    # torch eager: oracle encoder + restated adapter, the same parameter values, bf16 autocast
    cfg = vit_config(("rgb",), 768, 12, 12, S)
    p = {k: v.detach().clone().requires_grad_(not k.endswith("pos_emb")) for k, v in model.state_dict().items()}
    opt_e = torch.optim.AdamW([v for v in p.values() if v.requires_grad], lr=1e-4, weight_decay=0.05)
    gscaler = torch.amp.GradScaler("cuda")
    ids = torch.arange(n, device=dev).unsqueeze(0).expand(B, -1)

    def eager_out():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, enc = O.forward(p, {"rgb": x}, cfg, ids, ids)
            return convnext_head(enc, p, [0], n, S, S, 16, 4, prefix="output_adapters.semseg.")

    def eager_step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = crit(eager_out(), target)
        gscaler.scale(loss).backward()
        gscaler.step(opt_e)
        gscaler.update()
        opt_e.zero_grad()

    def eager_eval():
        with torch.no_grad():
            eager_out()

    res = {"ours_train": [], "eager_train": [], "ours_eval": [], "eager_eval": []}
    for _ in range(args.rounds):
        res["ours_train"].append(timed(ours_step, args.steps, args.warmup))
        res["eager_train"].append(timed(eager_step, args.steps, args.warmup))
        res["ours_eval"].append(timed(ours_eval, args.steps, args.warmup))
        res["eager_eval"].append(timed(eager_eval, args.steps, args.warmup))
    for k, v in res.items():
        emit(figure=k, batch=B, size=S, classes=K, ms_per_step=[round(t, 3) for t in v], median_ms=sorted(v)[len(v) // 2])
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    emit(figure="speedup_vs_eager", train=round(med["eager_train"] / med["ours_train"], 3),
         eval=round(med["eager_eval"] / med["ours_eval"], 3))

    # ---- the head alone: GEMM rate through mmae_profile_gemm, kernels through torch.profiler
    del opt_e, p
    torch.cuda.empty_cache()
    head = model.output_adapters["semseg"].train()
    info = {"image_size": (S, S), "tasks": {"rgb": {"num_tokens": n, "start_idx": 0, "end_idx": n}}}
    enc = torch.randn(B, n + 1, 768, device=dev, requires_grad=True)
    dout = torch.randn(B, K, S, S, device=dev)

    def head_step():
        head(enc, info).backward(dout)
    timed(head_step, 2, 2)
    lib = L.lib()
    lib.mmae_profile_gemm(1)
    head_step()
    import ctypes
    flops, ms, launches = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
    L.check(lib.mmae_profile_gemm_read(ctypes.byref(flops), ctypes.byref(ms), ctypes.byref(launches)))
    lib.mmae_profile_gemm(0)
    emit(figure="head_gemms", launches=launches.value, tflop=round(flops.value / 1e12, 3), ms=round(ms.value, 3),
         tflops=round(flops.value / (ms.value * 1e-3) / 1e12, 1))
    emit(figure="head_step", ms=round(timed(head_step, 5, 2), 3))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            head_step()
        torch.cuda.synchronize()
    P, C, Kp = B * n * 16, 384, (K + 7) // 8 * 8
    nbytes = {"dwconv_kernel<false>": 2 * P * C * 4, "dwconv_kernel<true>": 3 * P * C * 4, "dwconv_wgrad_kernel": 2 * P * C * 4,
              "upsample_fwd_kernel": B * K * S * S * 4 + P * Kp * 4, "upsample_bwd_kernel": B * K * S * S * 4 + P * Kp * 4}
    kern = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            for key in nbytes:
                if key in ev.name:                   # demangled names: "void mmae::(anonymous namespace)::dwconv_kernel<true>(..."
                    kern.setdefault(key, []).append(ev.time_range.elapsed_us())
    for key, ts in kern.items():
        us = sorted(ts)[len(ts) // 2]
        emit(figure="kernel", name=key, launches=len(ts), median_us=round(us, 2), bytes=nbytes[key],
             gbps=round(nbytes[key] / (us * 1e-6) / 1e9, 1),
             share_of_3_35_tbps=round(nbytes[key] / (us * 1e-6) / HBM_BYTES_PER_S, 3))
    if not kern:
        emit(figure="kernel", error="no ConvNeXt head kernels found in the profiler trace")
    emit(**gpu_info())


if __name__ == "__main__":
    main()
