"""Time ImageNet-style classification fine-tuning (run_finetuning_cls.py) on one GPU.

    python scripts/gpu_time_finetune_cls.py [--batch 128] [--eval-batch 192] [--steps 20] [--warmup 5] [--rounds 3]

Workload: MultiViT-B/16 on rgb at 224 x 224 (N = 197 tokens), 1000 classes, drop_path 0.1, mixup-style soft targets with
soft-target cross-entropy, the stock torch.optim.AdamW and NativeScalerWithGradNormCount with loss scaling - the script's
train_one_epoch body under the overlay (AUTO_OWN_GRADIENTS: p.grad aliases the flat gradient arena).

Prints one JSON line per figure:
  - train step time and eval forward time (B = --eval-batch, torch.no_grad, model.eval()) of this package;
  - the same for torch eager under bf16 autocast: the oracle's encoder (oracle/multimae_oracle.py, no stochastic depth)
    plus the head restated in torch, on the same parameter values; the two alternate in one process, --rounds times;
  - the classification-head kernels alone (torch.profiler, a separate pass): the pool kernel (reads B*N*D*4 bytes) and
    the head backward kernel (writes B*N*D*4 bytes), with achieved GB/s against the H100 SXM's 3.35 TB/s, and the whole
    mmae_clshead_forward / _backward calls timed with CUDA events;
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def soft_targets(B, C, dev, lam=0.7, smoothing=0.1):
    y = torch.randint(0, C, (B,), device=dev)
    off, on = smoothing / C, 1.0 - smoothing + smoothing / C
    t = torch.full((B, C), off, device=dev).scatter_(1, y[:, None], on)
    return t * lam + t.flip(0) * (1 - lam)


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
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--eval-batch", type=int, default=192)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    from cls_head_oracle import cls_head, soft_target_ce, vit_config
    from multimae_b200 import _lib as L
    from multimae_b200 import functional as Fn
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import LinearOutputAdapter
    from oracle import multimae_oracle as O

    dev = torch.device("cuda:0")
    emit(**gpu_info())
    B, Be, C = args.batch, args.eval_batch, args.classes
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=224)},
                             {"cls": LinearOutputAdapter(C)}, drop_path_rate=0.1).to(dev)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount()
    x = torch.randn(B, 3, 224, 224, device=dev)
    xe = torch.randn(Be, 3, 224, 224, device=dev)
    target = soft_targets(B, C, dev)

    def ours_step():
        model.train()
        with torch.cuda.amp.autocast():
            loss = soft_target_ce(model(x)["cls"], target)
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())
        opt.zero_grad()

    def ours_eval():
        model.eval()
        with torch.no_grad(), torch.cuda.amp.autocast():
            model(xe)["cls"]

    # torch eager: oracle encoder + head, the same parameter values, bf16 autocast
    cfg = vit_config(("rgb",), 768, 12, 12, 224)
    p = {k: v.detach().clone().requires_grad_(not k.endswith("pos_emb")) for k, v in model.state_dict().items()}
    opt_e = torch.optim.AdamW([v for v in p.values() if v.requires_grad], lr=1e-4, weight_decay=0.05)
    gscaler = torch.amp.GradScaler("cuda")

    def eager_logits(inp):
        ids = torch.arange(196, device=dev).unsqueeze(0).expand(inp.shape[0], -1)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, enc = O.forward(p, {"rgb": inp}, cfg, ids, ids)
            return cls_head(enc.float(), p)

    def eager_step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = soft_target_ce(eager_logits(x), target)
        gscaler.scale(loss).backward()
        gscaler.step(opt_e)
        gscaler.update()
        opt_e.zero_grad()

    def eager_eval():
        with torch.no_grad():
            eager_logits(xe)

    res = {"ours_train": [], "eager_train": [], "ours_eval": [], "eager_eval": []}
    for r in range(args.rounds):
        res["ours_train"].append(timed(ours_step, args.steps, args.warmup))
        res["eager_train"].append(timed(eager_step, args.steps, args.warmup))
        res["ours_eval"].append(timed(ours_eval, args.steps, args.warmup))
        res["eager_eval"].append(timed(eager_eval, args.steps, args.warmup))
    for k, v in res.items():
        emit(figure=k, batch=Be if k.endswith("eval") else B, ms_per_step=[round(t, 3) for t in v], median_ms=sorted(v)[len(v) // 2])
    mo, me = sorted(res["ours_train"])[args.rounds // 2], sorted(res["eager_train"])[args.rounds // 2]
    emit(figure="train_speedup_vs_eager", ratio=round(me / mo, 3), samples_per_s=round(B * 1000 / mo, 1))

    # ---- the head alone: entry points with CUDA events, kernels with torch.profiler
    del opt_e, p
    torch.cuda.empty_cache()
    head = model.output_adapters["cls"].train()
    N, D = 197, 768
    enc = torch.randn(B, N, D, device=dev, requires_grad=True)
    dlog = torch.randn(B, C, device=dev)
    lib = L.lib()
    saved = torch.empty(lib.mmae_clshead_saved_bytes(B, N, D, C), dtype=torch.uint8, device=dev)
    ws = Fn.Workspace.get(lib.mmae_clshead_workspace_bytes(B, N, D, C), dev)
    out = torch.empty(B, C, device=dev)
    dx = torch.empty(B, N, D, device=dev)
    arena = model.grad_arena()
    gp = [arena.views["output_adapters.cls." + n].data_ptr() for n in Fn.CLS_PARAM_NAMES]

    def fwd():
        L.check(lib.mmae_clshead_forward(enc.data_ptr(), B, N, D, C, 1, 1e-6, head.norm.weight.data_ptr(),
                                         head.norm.bias.data_ptr(), head.head.weight.data_ptr(), head.head.bias.data_ptr(),
                                         out.data_ptr(), saved.data_ptr(), ws.data_ptr(), L.current_stream()))

    def bwd():
        L.check(lib.mmae_clshead_backward(dlog.data_ptr(), B, N, D, C, 1, head.norm.weight.data_ptr(),
                                          head.head.weight.data_ptr(), *gp, dx.data_ptr(), saved.data_ptr(), ws.data_ptr(),
                                          L.current_stream()))
    nbytes = B * N * D * 4
    t_f = timed(fwd, 200, 20)
    t_b = timed(bwd, 200, 20)
    emit(figure="clshead_forward_call", B=B, N=N, D=D, C=C, us=round(t_f * 1e3, 2),
         gbps_pool_bytes=round(nbytes / (t_f * 1e-3) / 1e9, 1))
    emit(figure="clshead_backward_call", B=B, N=N, D=D, C=C, us=round(t_b * 1e3, 2),
         gbps_token_grad_bytes=round(nbytes / (t_b * 1e-3) / 1e9, 1))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            fwd()
            bwd()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            for key in ("cls_pool_kernel", "cls_pool_ln_kernel", "cls_head_bwd_kernel"):
                if key + "(" in ev.name or ev.name.endswith(key):
                    kern.setdefault(key, []).append(ev.time_range.elapsed_us())
    for key, ts in kern.items():
        us = sorted(ts)[len(ts) // 2]
        row = dict(figure="kernel", name=key, launches=len(ts), median_us=round(us, 2))
        if key in ("cls_pool_kernel", "cls_head_bwd_kernel"):
            row["bytes"] = nbytes
            row["gbps"] = round(nbytes / (us * 1e-6) / 1e9, 1)
            row["share_of_3_35_tbps"] = round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)
        emit(**row)
    if not kern:
        emit(figure="kernel", error="no cls_* kernels found in the profiler trace")
    emit(**gpu_info())


if __name__ == "__main__":
    main()
