"""Cost of dropout on classification fine-tuning and on the attention kernels.

    python scripts/gpu_time_dropout.py [--rounds 3] [--steps 20]

1. The fine-tuning step of run_finetuning_cls.py: multivit_base + LinearOutputAdapter(1000), rgb 224 x 224, batch 128,
   drop_path_rate 0.1, autocast, loss scaling, torch.optim.AdamW.  drop = attn_drop = 0 against 0.1 (the rates are set on
   the same model's nn.Dropout modules), alternating in one process after warm-up; ms/step from CUDA events.
2. Per call, the attention forward and backward at 197 x 197 and 577 x 577 keys, dh 64, 12 heads, batch 128, without and
   with dropout 0.1 (the dropout_p argument of mmae_attention_forward / _backward).

Prints one JSON line per figure with the GPU name and power limit."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    from gpu_time_finetune_cls import emit, gpu_info, soft_targets, timed
    from cls_head_oracle import soft_target_ce
    from multimae_b200 import _lib as L
    from multimae_b200 import multimae as mm
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import LinearOutputAdapter

    dev = torch.device("cuda:0")
    info = gpu_info()
    B, C = args.batch, args.classes
    torch.manual_seed(0)
    mm.AUTO_OWN_GRADIENTS = True
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=224)},
                             {"cls": LinearOutputAdapter(C)}, drop_path_rate=0.1).to(dev)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount()
    x = torch.randn(B, 3, 224, 224, device=dev)
    target = soft_targets(B, C, dev)

    def set_rate(rate):
        for blk in model.encoder:
            blk.attn.attn_drop.p = blk.attn.proj_drop.p = blk.mlp.drop.p = rate

    def step():
        model.train()
        with torch.cuda.amp.autocast():
            loss = soft_target_ce(model(x)["cls"], target)
        scaler(loss, opt, clip_grad=None, parameters=model.parameters())
        opt.zero_grad()

    rates = (0.0, 0.1)
    for r in rates:
        set_rate(r)
        timed(step, 2, args.warmup)
    times = {r: [] for r in rates}
    for _ in range(args.rounds):
        for r in rates:
            set_rate(r)
            times[r].append(timed(step, args.steps, 2))
    base = statistics.median(times[0.0])
    for r in rates:
        med = statistics.median(times[r])
        emit(figure="finetune_cls_step", drop=r, attn_drop=r, batch=B, ms_per_step=round(med, 3),
             rounds=[round(t, 3) for t in times[r]], overhead_pct=round(100.0 * (med - base) / base, 2), **info)

    lib = L.lib()
    H, dh = 12, 64
    D = H * dh
    seed = torch.tensor(12345, dtype=torch.int64, device=dev)
    for N in (197, 577):
        qkv = torch.randn(B * N, 3 * D, device=dev).bfloat16()
        d_o = torch.randn(B * N, D, device=dev).bfloat16()
        o = torch.empty(B * N, D, dtype=torch.bfloat16, device=dev)
        lse = torch.empty(B, H, N, device=dev)
        delta = torch.empty(B, H, N, device=dev)
        dqkv = torch.empty_like(qkv)
        q, k, v = qkv.data_ptr(), qkv[:, D:].data_ptr(), qkv[:, 2 * D:].data_ptr()
        st = L.current_stream()

        def fwd(p):
            return lambda: L.check(lib.mmae_attention_forward(q, 3 * D, k, 3 * D, v, 3 * D, o.data_ptr(), D, lse.data_ptr(),
                                                              B, H, N, N, dh, dh ** -0.5, p, seed.data_ptr(), st))

        def bwd(p):
            return lambda: L.check(lib.mmae_attention_backward(
                q, 3 * D, k, 3 * D, v, 3 * D, o.data_ptr(), D, d_o.data_ptr(), D, lse.data_ptr(), delta.data_ptr(),
                dqkv.data_ptr(), 3 * D, dqkv[:, D:].data_ptr(), 3 * D, dqkv[:, 2 * D:].data_ptr(), 3 * D, B, H, N, N, dh,
                dh ** -0.5, p, seed.data_ptr(), st))
        res = {}
        for p in (0.0, 0.1):
            fwd(p)()
            res[("fwd", p)] = statistics.median(timed(fwd(p), 50, 5) for _ in range(args.rounds))
            res[("bwd", p)] = statistics.median(timed(bwd(p), 50, 5) for _ in range(args.rounds))
        for kind in ("fwd", "bwd"):
            emit(figure="attention_" + kind, N=N, head_dim=dh, heads=H, batch=B,
                 us_no_dropout=round(1e3 * res[(kind, 0.0)], 1), us_dropout_0_1=round(1e3 * res[(kind, 0.1)], 1), **info)
    print(json.dumps({"done": True}))


if __name__ == "__main__":
    main()
