"""Per-shape timings of the wgmma GEMM at the MultiMAE-B bs 128 step's shapes, and its fixed cost per output tile.

    python scripts/gpu_time_gemm.py               # every distinct GEMM shape / operand-major combination of the step
    python scripts/gpu_time_gemm.py --fixed-cost  # per-tile fixed cost: intercept of time over k-blocks
    python scripts/gpu_time_gemm.py --variant 8   # the step's shapes on one tile variant (mmae_gemm_set_variant)
    python scripts/gpu_time_gemm.py --variant 3 9 # ... on several, side by side (wgrad shapes included)

Shapes: encoder M = 128 x 99 tokens (D 768, MLP 3072), decoders M = 128 x 196 query tokens and 128 x 99 context tokens
(D 256, MLP 1024), with the epilogue each call has in the step: forward = bf16 out + bias, dgrad = bf16 out with an
MN-major weight, wgrad = fp32 accumulate with both operands MN-major and the automatic split-K.  CUDA events around 50
back-to-back calls after 5 warm-up calls; prints microseconds per call, TFLOP/s and the share of the H100 SXM data-sheet
dense BF16 rate (989 TFLOP/s).

--fixed-cost times one 128 x 256 output tile per SM over 96 k-blocks (fp32 reduce-add output), cut into 1, 2, 4, 8 and
12 split-K work items per SM.  The MMA work stays the same, so the time added per extra item is the fixed cost of one
item: its epilogue, its reduce-add traffic and the hand-over between items.  (One tile per SM at K = 64 against K = 768
does not isolate it: at K = 64 a tile's output write takes longer than its one k-block of MMAs.)  It then times
bf16-output items with a bias, as the forward GEMMs run them, at K = 256 and 768 for each tile of VARIANT_BN, and
fp32-output items without one for the 128-column tiles of the cooperative and asynchronous-epilogue kernels
(fixed_cost_bf16)."""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multimae_b200 import _lib as L  # noqa: E402
from multimae_b200 import kernels as KN  # noqa: E402

ENC, DQ, DC = 128 * 99, 128 * 196, 128 * 99
# (class, name, M, N, K, kind)
SHAPES = [
    ("enc K=768", "qkv fwd", ENC, 2304, 768, "fwd"), ("enc K=768", "proj fwd", ENC, 768, 768, "fwd"),
    ("enc K=768", "fc1 fwd", ENC, 3072, 768, "fwd"), ("enc K=768", "fc2 dgrad", ENC, 3072, 768, "dgrad"),
    ("enc K=768", "proj dgrad", ENC, 768, 768, "dgrad"),
    ("enc K=2304/3072", "fc2 fwd", ENC, 768, 3072, "fwd"), ("enc K=2304/3072", "fc1 dgrad", ENC, 768, 3072, "dgrad"),
    ("enc K=2304/3072", "qkv dgrad", ENC, 768, 2304, "dgrad"),
    ("enc wgrad", "qkv wgrad", 2304, 768, ENC, "wgrad"), ("enc wgrad", "proj wgrad", 768, 768, ENC, "wgrad"),
    ("enc wgrad", "fc1 wgrad", 3072, 768, ENC, "wgrad"), ("enc wgrad", "fc2 wgrad", 768, 3072, ENC, "wgrad"),
    ("dec", "q / proj / depth-out fwd", DQ, 256, 256, "fwd"), ("dec", "kv fwd", DC, 512, 256, "fwd"),
    ("dec", "fc1 fwd", DQ, 1024, 256, "fwd"), ("dec", "fc2 fwd", DQ, 256, 1024, "fwd"),
    ("dec", "rgb-out fwd", DQ, 768, 256, "fwd"), ("dec", "semseg-out fwd", DQ, 2128, 256, "fwd"),
    ("dec", "context proj fwd", DC, 1024, 768, "fwd"),
    ("dec", "q / proj dgrad", DQ, 256, 256, "dgrad"), ("dec", "kv dgrad", DC, 256, 512, "dgrad"),
    ("dec", "fc2 dgrad", DQ, 1024, 256, "dgrad"), ("dec", "fc1 dgrad", DQ, 256, 1024, "dgrad"),
    ("dec", "q / proj wgrad", 256, 256, DQ, "wgrad"), ("dec", "kv wgrad", 512, 256, DC, "wgrad"),
    ("dec", "fc1 wgrad", 1024, 256, DQ, "wgrad"), ("dec", "fc2 wgrad", 256, 1024, DQ, "wgrad"),
    ("dec", "rgb-out wgrad", 768, 256, DQ, "wgrad"), ("dec", "semseg-out wgrad", 2128, 256, DQ, "wgrad"),
    ("dec", "context proj wgrad", 1024, 768, DC, "wgrad"),
]
PEAK_TFLOPS = 989.0
# variants timed by --fixed-cost (8 / 9 / 10: asynchronous epilogue): their output tile width
VARIANT_BN = {1: 128, 3: 192, 2: 256, 8: 128, 9: 192, 10: 256}
F32_VARIANTS = (1, 8)


def timed(fn, n=50):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3


def gpu_state():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def rnd(dev, *shape):
    return (torch.randn(*shape, device=dev) * 0.5).to(torch.bfloat16)


def gemm_call(dev, M, N, K, kind):
    """The call as the step makes it: operands laid out as in the step, outputs allocated once."""
    if kind == "fwd":
        A, B, bias = rnd(dev, M, K), rnd(dev, N, K), torch.randn(N, device=dev)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        return lambda: KN.gemm(A, B, bias=bias, out_bf16=out)
    if kind == "dgrad":
        A, B = rnd(dev, M, K), rnd(dev, K, N)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        return lambda: KN.gemm(A, B, b_mn=True, out_bf16=out)
    A, B = rnd(dev, K, M), rnd(dev, K, N)
    out = torch.zeros(M, N, device=dev)
    return lambda: KN.gemm(A, B, a_mn=True, b_mn=True, out_f32=out, accumulate=True, split_k=0)


def shapes(variants):
    """Microseconds per call of every shape under each variant in turn (TF/s and share of peak for the first)."""
    dev = torch.device("cuda:0")
    print("%-16s %-26s %6s %5s %6s %-5s" % ("class", "gemm", "M", "N", "K", "kind") +
          "".join(" %9s" % ("us v%d" % v) for v in variants) + " %7s %6s" % ("TF/s", "%989"))
    try:
        for cls, name, M, N, K, kind in SHAPES:
            call = gemm_call(dev, M, N, K, kind)
            us = []
            for v in variants:
                L.lib().mmae_gemm_set_variant(v)
                us.append(timed(call))
            tf = 2.0 * M * N * K / (us[0] * 1e-6) / 1e12
            print("%-16s %-26s %6d %5d %6d %-5s" % (cls, name, M, N, K, kind) + "".join(" %9.1f" % u for u in us) +
                  " %7.1f %6.1f" % (tf, 100 * tf / PEAK_TFLOPS))
    finally:
        L.lib().mmae_gemm_set_variant(-1)


def fixed_cost():
    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    M, N, K = 128 * sms, 256, 96 * 64   # one 128 x 256 output tile per SM, 96 k-blocks
    A, B = rnd(dev, K, M), rnd(dev, K, N)
    out = torch.zeros(M, N, device=dev)
    L.lib().mmae_gemm_set_variant(2)    # 128 x 256 tiles, one CTA
    try:
        t = {s: timed(lambda: KN.gemm(A, B, a_mn=True, b_mn=True, out_f32=out, accumulate=True, split_k=s), n=200)
             for s in (1, 2, 4, 8, 12, 1)}
    finally:
        L.lib().mmae_gemm_set_variant(-1)
    kb = t[1] / 96
    print("%-8s %10s %12s %10s %16s" % ("splits", "items/SM", "k-blk/item", "us", "us per extra item"))
    for s in (1, 2, 4, 8, 12):
        extra = (t[s] - t[1]) / (s - 1) if s > 1 else 0.0
        print("%-8d %10d %12d %10.2f %16.3f" % (s, s, 96 // s, t[s], extra))
    per_item = (t[12] - t[1]) / 11
    print("fixed cost of one work item (128 x 256, fp32 reduce-add epilogue): %.2f us = %.1f k-block times (%.3f us per "
          "k-block)" % (per_item, per_item / kb, kb))
    fixed_cost_bf16(dev, sms)


def fixed_cost_bf16(dev, sms):
    """bf16-output items (bias, TMA tile store) at N = 768, the encoder's width, so that the n-tiles of one A row block
    run side by side and read it from L2 as in the step.  Per-item time = slope of the call time over items per SM
    (3 -> 12); k-block time = slope of the per-item time over K (768 -> 3072); fixed cost = per-item time minus the item's
    k-blocks at that rate: the epilogue and the hand-over that the tensor cores do not overlap."""
    N = 768
    print("%-8s %-7s %-5s %5s %10s %12s %12s %12s" % ("variant", "tile", "out", "K", "us/item", "us/k-block", "fixed us",
                                                     "fixed k-blk"))
    for variant, f32 in [(v, False) for v in sorted(VARIANT_BN)] + [(v, True) for v in F32_VARIANTS]:
        bn = VARIANT_BN[variant]
        tiles_n = N // bn
        bias = torch.randn(N, device=dev)
        L.lib().mmae_gemm_set_variant(variant)
        try:
            per_item = {}
            for K in (256, 768, 3072):
                B = rnd(dev, N, K)
                t = {}
                for n in (3, 12):   # items per SM
                    assert sms * n % tiles_n == 0
                    M = 128 * sms * n // tiles_n
                    A = rnd(dev, M, K)
                    if f32:
                        out = torch.empty(M, N, device=dev)
                        t[n] = timed(lambda: KN.gemm(A, B, out_f32=out), n=100)
                    else:
                        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
                        t[n] = timed(lambda: KN.gemm(A, B, bias=bias, out_bf16=out), n=100)
                    del A, out
                per_item[K] = (t[12] - t[3]) / 9
        finally:
            L.lib().mmae_gemm_set_variant(-1)
        kb = (per_item[3072] - per_item[768]) / ((3072 - 768) // 64)
        for K in (256, 768):
            fixed = per_item[K] - K // 64 * kb
            print("%-8d %-7s %-5s %5d %10.3f %12.3f %12.3f %12.2f" % (variant, "128x%d" % bn, "fp32" if f32 else "bf16", K,
                                                                     per_item[K], kb, fixed, fixed / kb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fixed-cost", action="store_true", help="time the per-tile fixed cost instead of the step's shapes")
    ap.add_argument("--variant", type=int, nargs="+", default=[-1],
                    help="tile variant(s) of every call (-1: the heuristic's choice), timed side by side")
    a = ap.parse_args()
    torch.manual_seed(0)
    print("# %s (name, power limit, SM clock, max SM clock; before)" % gpu_state())
    fixed_cost() if a.fixed_cost else shapes(a.variant)
    print("# %s (after)" % gpu_state())


if __name__ == "__main__":
    main()
