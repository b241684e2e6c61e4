"""Time semantic-segmentation fine-tuning with the Segmenter head (run_finetuning_semseg.py --output_adapter segmenter
--decoder_dim 768, ADE20K shapes) on one GPU.

    python scripts/gpu_time_finetune_segmenter.py [--batch 4] [--classes 150] [--steps 10] [--warmup 3] [--rounds 3]

Workload: MultiViT-B/16 on rgb at 512 x 512 (1025 encoder tokens), drop_path 0.1, SegmenterMaskTransformerAdapter(150 + 1
void classes, embed_dim 768, 12 heads, depth 2, drop_path 0.1), CrossEntropyLoss(ignore_index=255), the stock
torch.optim.AdamW and NativeScalerWithGradNormCount with loss scaling - the script's train_one_epoch body under the
overlay.  Seeded synthetic data.  It needs a CUDA device and fails without one.

Prints one JSON line per figure:
  - train step time and eval forward time (torch.no_grad, model.eval()) of this package;
  - the same for torch eager under bf16 autocast: the oracle's encoder plus the head restated in torch
    (tests/segmenter_head_oracle.py, no stochastic depth), on the same parameter values; the two alternate in one process,
    --rounds times, and every round is printed (the spread);
  - the fused mask kernels alone (mmae_segmenter_mask_forward / _backward), CUDA events over many launches, with the FLOPs
    and bytes computed here from the shapes;
  - the GPU name, power limit and SM clocks, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


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
    from multimae_b200 import _lib as L
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import SegmenterMaskTransformerAdapter
    from oracle import multimae_oracle as O
    from segmenter_head_oracle import segmenter_head

    dev = torch.device("cuda:0")
    emit(**gpu_info())
    B, S, K, E = args.batch, args.size, args.classes + 1, 768
    n = (S // 16) ** 2
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=S)},
                             {"semseg": SegmenterMaskTransformerAdapter(K, embed_dim=E, depth=2, drop_path_rate=0.1)},
                             drop_path_rate=0.1).to(dev)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount()
    crit = torch.nn.CrossEntropyLoss(ignore_index=255)
    x = torch.randn(B, 3, S, S, device=dev)
    target = torch.randint(0, K, (B, S, S), device=dev)
    target[torch.rand(target.shape, device=dev) < 0.1] = 255

    def ours_step():
        model.train()
        with torch.autocast("cuda", dtype=torch.float16):
            loss = crit(model(x)["semseg"], target)
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())
        opt.zero_grad()

    def ours_eval():
        model.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            model(x)["semseg"]

    cfg = vit_config(("rgb",), 768, 12, 12, S)
    p = {k: v.detach().clone().requires_grad_(not k.endswith("pos_emb")) for k, v in model.state_dict().items()}
    opt_e = torch.optim.AdamW([v for v in p.values() if v.requires_grad], lr=1e-4, weight_decay=0.05)
    gscaler = torch.amp.GradScaler("cuda")
    ids = torch.arange(n, device=dev).unsqueeze(0).expand(B, -1)

    def eager_out():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, enc = O.forward(p, {"rgb": x}, cfg, ids, ids)
            return segmenter_head(enc, p, [0], n, S, S, 2, 12, prefix="output_adapters.semseg.")

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

    # ---- the head alone, then the fused mask kernels alone
    del opt_e, p
    torch.cuda.empty_cache()
    head = model.output_adapters["semseg"].train()
    info = {"image_size": (S, S), "tasks": {"rgb": {"num_tokens": n, "start_idx": 0, "end_idx": n}}}
    enc = torch.randn(B, n + 1, 768, device=dev, requires_grad=True)
    dout = torch.randn(B, K, S, S, device=dev)
    emit(figure="head_step", ms=round(timed(lambda: head(enc, info).backward(dout), 10, 3), 3))
    lib, st = L.lib(), torch.cuda.current_stream().cuda_stream
    Kp = (K + 7) // 8 * 8
    P = torch.randn(B * n, E, device=dev).bfloat16()
    C = torch.randn(B * K, E, device=dev).bfloat16()
    rp, rc = 1 / P.float().norm(dim=1), 1 / C.float().norm(dim=1)
    gamma, beta = torch.ones(K, device=dev), torch.zeros(K, device=dev)
    cmap, dcm = torch.empty(B * n, Kp, device=dev), torch.randn(B * n, Kp, device=dev)
    mean, rstd = torch.empty(B * n, device=dev), torch.empty(B * n, device=dev)
    dP, dC = torch.empty_like(P), torch.empty_like(C)
    dg, db = torch.zeros(K, device=dev), torch.zeros(K, device=dev)
    ws = torch.empty(lib.mmae_segmenter_mask_workspace_bytes(B, n, K), dtype=torch.uint8, device=dev)

    def mask_fwd():
        L.check(lib.mmae_segmenter_mask_forward(P.data_ptr(), C.data_ptr(), rp.data_ptr(), rc.data_ptr(), gamma.data_ptr(),
                                                beta.data_ptr(), 1e-6, B, n, K, E, cmap.data_ptr(), mean.data_ptr(),
                                                rstd.data_ptr(), st))

    def mask_bwd():
        L.check(lib.mmae_segmenter_mask_backward(P.data_ptr(), C.data_ptr(), rp.data_ptr(), rc.data_ptr(), gamma.data_ptr(),
                                                 mean.data_ptr(), rstd.data_ptr(), dcm.data_ptr(), B, n, K, E, dP.data_ptr(),
                                                 dC.data_ptr(), dg.data_ptr(), db.data_ptr(), ws.data_ptr(), st))
    prod = 2.0 * B * n * K * E
    for name, fn, flop, nbytes in (
            ("mask_forward (1 kernel)", mask_fwd, prod, (B * n + B * K) * E * 2 + B * n * Kp * 4),
            ("mask_backward (3 kernels + 2 reductions)", mask_bwd, 3 * prod,
             2 * (B * n + B * K) * E * 2 + B * n * Kp * (4 + 2))):
        ms = timed(fn, 200, 20)
        emit(figure="kernel", name=name, us=round(ms * 1e3, 2), gflop=round(flop / 1e9, 3), mbytes=round(nbytes / 1e6, 2),
             tflops=round(flop / (ms * 1e-3) / 1e12, 2), gbps=round(nbytes / (ms * 1e-3) / 1e9, 1))
    emit(**gpu_info())


if __name__ == "__main__":
    main()
