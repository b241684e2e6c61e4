"""GPU: the fused attention backward (one CTA per (batch, head), Nk <= 256) against a torch fp32 reference.

Covers the MultiMAE-B bs 128 shapes in the layouts the blocks use, both sides of the 256-key dispatch boundary, fewer
than 16 keys, and run-to-run bitwise equality (every dQ / dK / dV element is written by exactly one thread, no atomics).
Tolerance: 1e-2 relative L2, as for the other attention tests (bf16 P / dS operands)."""
import pytest
import torch

from helpers import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture()
def KN():
    from multimae_b200 import _lib as L
    from multimae_b200 import kernels
    L.lib().mmae_attention_set_tc(0)          # mma.sync kernels: the fused backward serves every Nk <= 256
    yield kernels
    L.lib().mmae_attention_set_tc(-1)


def _inputs(B, H, Nq, Nk, dh, self_attn, seed=0):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(seed)
    D = H * dh

    def r(*shape):
        return (torch.randn(*shape, device=dev, generator=gen) * 0.5).to(torch.bfloat16)
    if self_attn:                             # q, k, v (and dq, dk, dv) are column slices of one [B*N, 3D] buffer
        qkv = r(B * Nq, 3 * D)
        q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        dqkv = torch.empty(B * Nq, 3 * D, device=dev, dtype=torch.bfloat16)
        grads = dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:]
    else:
        q, kv = r(B * Nq, D), r(B * Nk, 2 * D)
        k, v = kv[:, :D], kv[:, D:]
        dkv = torch.empty(B * Nk, 2 * D, device=dev, dtype=torch.bfloat16)
        grads = torch.empty(B * Nq, D, device=dev, dtype=torch.bfloat16), dkv[:, :D], dkv[:, D:]
    return q, k, v, r(B * Nq, D), grads


def _check(KN, B, H, Nq, Nk, dh, self_attn):
    D, scale = H * dh, dh ** -0.5
    q, k, v, do, (dq, dk, dv) = _inputs(B, H, Nq, Nk, dh, self_attn)
    o, lse = KN.attention_fwd(q, k, v, B, H, Nq, Nk, dh, scale)
    KN.attention_bwd(q, k, v, o, do, lse, dq, dk, dv, B, H, Nq, Nk, dh, scale)

    def heads(x, n):
        return x.float().reshape(B, n, H, dh).transpose(1, 2).detach().requires_grad_(True)
    qf, kf, vf = heads(q, Nq), heads(k, Nk), heads(v, Nk)
    ref = (torch.softmax((qf @ kf.transpose(-2, -1)) * scale, -1) @ vf).transpose(1, 2).reshape(B * Nq, D)
    ref.backward(do.float())
    for got, want in ((dq, qf.grad), (dk, kf.grad), (dv, vf.grad)):
        err = rel_l2(got, want.transpose(1, 2).reshape(got.shape))
        assert err < 1e-2, (B, H, Nq, Nk, dh, err)


@pytest.mark.parametrize("case", [(128, 12, 99, 99, 64, True), (128, 8, 196, 99, 32, False), (128, 8, 196, 196, 32, True)],
                         ids=["encoder", "decoder_cross", "decoder_self"])
def test_fused_backward_bench_shapes(KN, case):
    _check(KN, *case)


@pytest.mark.parametrize("case", [(2, 2, 200, 255, 32, False), (2, 3, 256, 256, 64, True), (2, 2, 150, 257, 64, False),
                                  (1, 2, 257, 257, 32, True)])
def test_fused_backward_dispatch_boundary(KN, case):
    _check(KN, *case)


# (Nk = 1 is left out: its exact dQ and dK are zero, so a relative error has no scale)
@pytest.mark.parametrize("case", [(2, 3, 40, 7, 64, False), (3, 2, 5, 2, 32, False), (2, 4, 15, 15, 32, True),
                                  (1, 2, 70, 16, 64, False)])
def test_fused_backward_few_keys(KN, case):
    _check(KN, *case)


@pytest.mark.parametrize("case", [(16, 12, 99, 99, 64, True), (16, 8, 196, 196, 32, True)])
def test_fused_backward_bitwise_repeatable(KN, case):
    B, H, Nq, Nk, dh, self_attn = case
    scale = dh ** -0.5
    q, k, v, do, grads = _inputs(B, H, Nq, Nk, dh, self_attn)
    o, lse = KN.attention_fwd(q, k, v, B, H, Nq, Nk, dh, scale)
    runs = []
    for _ in range(2):
        for g in grads:
            g.fill_(float("nan"))
        KN.attention_bwd(q, k, v, o, do, lse, *grads, B, H, Nq, Nk, dh, scale)
        runs.append([g.clone() for g in grads])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
