"""Time depth fine-tuning with the ConvNeXt head (run_finetuning_depth.py --output_adapter convnext) on one GPU.

    python scripts/gpu_time_finetune_depth.py [--batch 64] [--eval_batch 96] [--steps 5] [--warmup 2] [--rounds 3]

Workload: the script's defaults - MultiViT-B/16 on rgb at 256 x 256 (257 encoder tokens), ConvNeXtAdapter(1,
preds_per_patch=64) with the adapter's default embed_dim 6144 and depth 4 (96 channels per pixel on a 128 x 128 map, x2
upsample), the masked berhu loss against a mask_valid with invalid pixels, the stock torch.optim.AdamW over the layer-decay
groups (0.75), NativeScalerWithGradNormCount(enabled=False) and autocast(enabled=False) - the train_one_epoch body under
the overlay.

Prints one JSON line per figure:
  - train step time (batch --batch) and eval forward time (torch.no_grad, model.eval(), batch --eval_batch = 1.5 x the
    script's default) of this package;
  - the same for torch eager in fp32, as the script asks: the oracle's encoder plus the adapter restated in torch
    (tests/convnext_head_oracle.py, channels-first cuDNN depthwise conv), on the same parameter values; the two alternate in
    one process, --rounds times;
  - the head alone: a forward + backward with depth 4 and with depth 0 (proj_dec + final_layer + upsample only: an upper
    bound on the share of the padded 8-column final_layer GEMM);
  - per call: the narrow LayerNorm forward / backward at P = 64 x 128 x 128 pixels, C = 96, with the least bytes each must
    move and the achieved GB/s against the H100 SXM's 3.35 TB/s;
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


def layer_decay_groups(model, weight_decay, layer_decay):
    """utils/optim_factory.py get_parameter_groups with LayerDecayValueAssigner, as the script builds them."""
    num_layers = model.get_num_layers()
    values = [layer_decay ** (num_layers + 1 - i) for i in range(num_layers + 2)]
    skip, groups = model.no_weight_decay(), {}
    for name, p in model.named_parameters():
        if not p.requires_grad:
            continue
        no_decay = p.ndim == 1 or name.endswith(".bias") or name in skip
        if name in ("global_tokens",) or name.startswith("input_adapters"):
            lid = 0
        elif name.startswith("encoder"):
            lid = int(name.split(".")[1]) + 1
        else:
            lid = len(values) - 1
        key = (lid, no_decay)
        groups.setdefault(key, {"weight_decay": 0.0 if no_decay else weight_decay, "params": [], "lr_scale": values[lid]})
        groups[key]["params"].append(p)
    return list(groups.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--eval_batch", type=int, default=96)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    from cls_head_oracle import vit_config
    from convnext_depth_oracle import masked_berhu_loss
    from convnext_head_oracle import convnext_head
    from multimae_b200 import kernels as Kn
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import ConvNeXtAdapter
    from oracle import multimae_oracle as O

    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True                   # run_finetuning_depth.py:324
    emit(**gpu_info())
    B, EB, S = args.batch, args.eval_batch, args.size
    n = (S // 16) ** 2
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=S)},
                             {"depth": ConvNeXtAdapter(1, preds_per_patch=64, main_tasks=["rgb"])}).to(dev)
    opt = torch.optim.AdamW(layer_decay_groups(model, 1e-4, 0.75), lr=1e-4)
    scaler = NativeScalerWithGradNormCount(enabled=False)
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, 3, S, S, device=dev, generator=g)
    xe = torch.randn(EB, 3, S, S, device=dev, generator=g)
    target = 0.5 + 4.0 * torch.rand(B, 1, S, S, device=dev, generator=g)
    mask_valid = torch.rand(B, 1, S, S, device=dev, generator=g) >= 0.15

    def ours_step():
        model.train()
        with torch.cuda.amp.autocast(enabled=False):
            loss = masked_berhu_loss(model({"rgb": x})["depth"].float(), target, mask_valid)
        opt.zero_grad()
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())

    def ours_eval():
        model.eval()
        with torch.no_grad(), torch.cuda.amp.autocast(enabled=False):
            model({"rgb": xe})["depth"]

    # torch eager in fp32: oracle encoder + restated adapter on the same parameter values
    cfg = vit_config(("rgb",), 768, 12, 12, S)
    p = {k: v.detach().clone().requires_grad_(not k.endswith("pos_emb")) for k, v in model.state_dict().items()}
    pg = {id(v): k for k, v in model.named_parameters()}
    groups = [dict(gr, params=[p[pg[id(q)]] for q in gr["params"]]) for gr in layer_decay_groups(model, 1e-4, 0.75)]
    opt_e = torch.optim.AdamW(groups, lr=1e-4)

    def eager_out(inp):
        ids = torch.arange(n, device=dev).unsqueeze(0).expand(inp.shape[0], -1)
        _, enc = O.forward(p, {"rgb": inp}, cfg, ids, ids)
        return convnext_head(enc, p, [0], n, S, S, 64, 4, prefix="output_adapters.depth.")

    def eager_step():
        loss = masked_berhu_loss(eager_out(x), target, mask_valid)
        opt_e.zero_grad()
        loss.backward()
        opt_e.step()

    def eager_eval():
        with torch.no_grad():
            eager_out(xe)

    res = {"ours_train": [], "eager_train": [], "ours_eval": [], "eager_eval": []}
    for _ in range(args.rounds):
        res["ours_train"].append(timed(ours_step, args.steps, args.warmup))
        res["eager_train"].append(timed(eager_step, args.steps, args.warmup))
        res["ours_eval"].append(timed(ours_eval, args.steps, args.warmup))
        res["eager_eval"].append(timed(eager_eval, args.steps, args.warmup))
    for k, v in res.items():
        emit(figure=k, batch=EB if k.endswith("eval") else B, size=S, ms_per_step=[round(t, 3) for t in v],
             median_ms=sorted(v)[len(v) // 2])
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    emit(figure="speedup_vs_eager_fp32", train=round(med["eager_train"] / med["ours_train"], 3),
         eval=round(med["eager_eval"] / med["ours_eval"], 3))

    # ---- the head alone, with its blocks and without them (proj_dec + final_layer GEMM + upsample)
    del opt_e, p, groups
    torch.cuda.empty_cache()
    info = {"image_size": (S, S), "tasks": {"rgb": {"num_tokens": n, "start_idx": 0, "end_idx": n}}}
    enc = torch.randn(B, n + 1, 768, device=dev, requires_grad=True)
    dout = torch.randn(B, 1, S, S, device=dev)
    for depth in (4, 0):
        head = ConvNeXtAdapter(1, preds_per_patch=64, depth=depth)
        head.init(768)
        head = head.to(dev).train()

        def head_step():
            head(enc, info).backward(dout)
        t = timed(head_step, 5, 2)
        emit(figure="head_step", depth=depth, batch=B, ms=round(t, 3), share_of_train_step=round(t / med["ours_train"], 4))
        del head
    torch.cuda.empty_cache()

    # ---- the narrow LayerNorm at the head's shape: P = B x 128 x 128 pixels of C = 96 channels
    P, C = B * (S // 2) ** 2, 96
    xs = torch.randn(P, C, device=dev)
    gamma, beta = 1.0 + 0.1 * torch.randn(C, device=dev), 0.1 * torch.randn(C, device=dev)
    yb, _, mean, rstd = Kn.layernorm_fwd(xs, gamma, beta)
    dy = torch.randn(P, C, device=dev).to(torch.bfloat16)
    dgamma, dbeta, dx = torch.zeros(C, device=dev), torch.zeros(C, device=dev), torch.empty(P, C, device=dev)
    fwd_ms = timed(lambda: Kn.layernorm_fwd(xs, gamma, beta), 50, 5)
    bwd_ms = timed(lambda: Kn.layernorm_bwd(dy, xs, mean, rstd, gamma, dgamma, dbeta, dx=dx), 50, 5)
    # least traffic: forward reads x (fp32) and writes y (bf16) + mean / rstd; backward reads dy (bf16), x, mean / rstd and
    # writes dx (fp32).  gamma / beta and the [blocks, 3C] partial rows are a few hundred KB and are not counted.
    for name, ms, nbytes in (("layernorm_forward", fwd_ms, P * C * (4 + 2) + P * 8),
                             ("layernorm_backward", bwd_ms, P * C * (2 + 4 + 4) + P * 8)):
        emit(figure="narrow_layernorm", name=name, rows=P, D=C, us_per_call=round(ms * 1e3, 2), min_bytes=nbytes,
             gbps=round(nbytes / (ms * 1e-3) / 1e9, 1), share_of_3_35_tbps=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
    emit(**gpu_info())


if __name__ == "__main__":
    main()
