"""Per-kernel attention timings at the MultiMAE-B bs 128 shapes, mma.sync kernels against the wgmma kernels.

    python scripts/gpu_time_attention.py

CUDA events around 50 back-to-back calls after 5 warm-up calls, per shape and direction; prints microseconds per call."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multimae_b200 import _lib as L  # noqa: E402
from multimae_b200 import kernels as KN  # noqa: E402

SHAPES = [("encoder self 99x99 dh64", 128, 12, 99, 99, 64), ("decoder cross 196x99 dh32", 128, 8, 196, 99, 32),
          ("decoder self 196x196 dh32", 128, 8, 196, 196, 32)]


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


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("# %s" % gpu)
    print("%-28s %12s %12s %12s %12s" % ("shape", "fwd mma.sync", "fwd wgmma", "bwd mma.sync", "bwd wgmma"))
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    for name, B, H, Nq, Nk, dh in SHAPES:
        D = H * dh
        q = (torch.randn(B * Nq, D, device=dev) * 0.5).to(torch.bfloat16)
        kv = (torch.randn(B * Nk, 2 * D, device=dev) * 0.5).to(torch.bfloat16)
        k, v = kv[:, :D], kv[:, D:]
        do = (torch.randn(B * Nq, D, device=dev) * 0.5).to(torch.bfloat16)
        dq = torch.empty(B * Nq, D, device=dev, dtype=torch.bfloat16)
        dkv = torch.empty(B * Nk, 2 * D, device=dev, dtype=torch.bfloat16)
        row = []
        for tc in (0, 1 | 128):
            L.lib().mmae_attention_set_tc(tc)
            row.append(timed(lambda: KN.attention_fwd(q, k, v, B, H, Nq, Nk, dh, dh ** -0.5)))
        o, lse = KN.attention_fwd(q, k, v, B, H, Nq, Nk, dh, dh ** -0.5)
        for tc in (0, 64):
            L.lib().mmae_attention_set_tc(tc)
            row.append(timed(lambda: KN.attention_bwd(q, k, v, o, do, lse, dq, dkv[:, :D], dkv[:, D:], B, H, Nq, Nk, dh,
                                                      dh ** -0.5)))
        L.lib().mmae_attention_set_tc(-1)
        print("%-28s %12.1f %12.1f %12.1f %12.1f" % ((name,) + tuple(row)))


if __name__ == "__main__":
    main()
