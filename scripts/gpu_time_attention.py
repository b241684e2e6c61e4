"""Per-kernel attention timings at the MultiMAE-B bs 128 shapes, mma.sync kernels against the wgmma kernels.

    python scripts/gpu_time_attention.py

CUDA events around 50 back-to-back calls after 5 warm-up calls, per shape and direction; prints microseconds per call,
the HBM bytes one call must move (computed from the shapes: every operand read once, every result written once), the
achieved rate and its share of the H100 SXM data-sheet bandwidth (3.35 TB/s).  Self-attention operands are column
slices of one [B*N, 3D] qkv buffer, and their gradients of one dqkv buffer, as in the transformer block."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from multimae_b200 import _lib as L  # noqa: E402
from multimae_b200 import kernels as KN  # noqa: E402

SHAPES = [("encoder self 99x99 dh64", 128, 12, 99, 99, 64, True), ("decoder cross 196x99 dh32", 128, 8, 196, 99, 32, False),
          ("decoder self 196x196 dh32", 128, 8, 196, 196, 32, True)]
HBM_BYTES_PER_S = 3.35e12


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


def hbm_bytes(B, H, Nq, Nk, dh):
    """(forward, backward) bytes: bf16 Q, K, V -> O + fp32 lse; Q, K, V, O, dO, lse -> dQ, dK, dV."""
    q, kv, lse = 2 * B * Nq * H * dh, 2 * B * Nk * H * dh, 4 * B * H * Nq
    return 2 * q + 2 * kv + lse, 4 * q + 4 * kv + lse


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("# %s" % gpu)
    print("%-28s %-4s %8s | %-26s | %-26s" % ("shape", "dir", "MB", "mma.sync us  GB/s  %HBM", "wgmma us  GB/s  %HBM"))
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    for name, B, H, Nq, Nk, dh, self_attn in SHAPES:
        D = H * dh

        def rnd(*shape):
            return (torch.randn(*shape, device=dev) * 0.5).to(torch.bfloat16)
        if self_attn:
            qkv = rnd(B * Nq, 3 * D)
            q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
            dqkv = torch.empty(B * Nq, 3 * D, device=dev, dtype=torch.bfloat16)
            dq, dk, dv = dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:]
        else:
            q, kv = rnd(B * Nq, D), rnd(B * Nk, 2 * D)
            k, v = kv[:, :D], kv[:, D:]
            dq = torch.empty(B * Nq, D, device=dev, dtype=torch.bfloat16)
            dkv = torch.empty(B * Nk, 2 * D, device=dev, dtype=torch.bfloat16)
            dk, dv = dkv[:, :D], dkv[:, D:]
        do = rnd(B * Nq, D)
        fwd, bwd = [], []
        for tc in (0, 1 | 128):
            L.lib().mmae_attention_set_tc(tc)
            fwd.append(timed(lambda: KN.attention_fwd(q, k, v, B, H, Nq, Nk, dh, dh ** -0.5)))
        L.lib().mmae_attention_set_tc(0)
        o, lse = KN.attention_fwd(q, k, v, B, H, Nq, Nk, dh, dh ** -0.5)
        for tc in (0, 64):
            L.lib().mmae_attention_set_tc(tc)
            bwd.append(timed(lambda: KN.attention_bwd(q, k, v, o, do, lse, dq, dk, dv, B, H, Nq, Nk, dh, dh ** -0.5)))
        L.lib().mmae_attention_set_tc(-1)
        for direction, nbytes, us in zip(("fwd", "bwd"), hbm_bytes(B, H, Nq, Nk, dh), (fwd, bwd)):
            cols = ["%8.1f %6.0f %5.1f" % (t, nbytes / t * 1e-3, 100 * nbytes / (t * 1e-6) / HBM_BYTES_PER_S) for t in us]
            print("%-28s %-4s %8.1f | %-26s | %-26s" % (name, direction, nbytes / 1e6, cols[0], cols[1]))


if __name__ == "__main__":
    main()
