"""Thin tensor-level wrappers over the C ABI primitives (pointer extraction + shape checks only).

All compute happens in libmultimae_b200.so; tensors must be CUDA tensors.
"""
import ctypes

import torch

from . import _lib as L


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise L.MmaeError("multimae_b200 kernels need CUDA tensors (no CPU fallback)")


def gemm(A, B, *, a_mn=False, b_mn=False, bias=None, act=0, residual=None, dgelu_z=None, preact=None,
         out_f32=None, out_bf16=None, accumulate=False, split_k=1, alpha=1.0):
    """C[M,N] = epilogue(alpha * A @ B^T).  A: [M,K] (or [K,M] if a_mn), B: [N,K] (or [K,N] if b_mn); bf16."""
    _need_cuda(A, B)
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    assert A.dim() == 2 and B.dim() == 2 and A.stride(1) == 1 and B.stride(1) == 1
    if a_mn:
        K, M = A.shape
    else:
        M, K = A.shape
    if b_mn:
        Kb, N = B.shape
    else:
        N, Kb = B.shape
    assert K == Kb, "contraction mismatch %d vs %d" % (K, Kb)
    ep = L.GemmEpilogue()
    ep.alpha = alpha
    ep.act = act
    ep.accumulate = 1 if accumulate else 0
    for name, ldname, t, dt in (("residual", "ld_residual", residual, torch.float32),
                                ("dgelu_z", "ld_dgelu_z", dgelu_z, torch.bfloat16),
                                ("preact_bf16", "ld_preact", preact, torch.bfloat16),
                                ("out_f32", "ld_out_f32", out_f32, torch.float32),
                                ("out_bf16", "ld_out_bf16", out_bf16, torch.bfloat16)):
        if t is not None:
            assert t.dtype == dt and t.shape[0] == M and t.shape[1] == N and t.stride(1) == 1, name
            setattr(ep, name, t.data_ptr())
            setattr(ep, ldname, t.stride(0))
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == N
        ep.bias = bias.data_ptr()
    L.check(L.lib().mmae_gemm_bf16(A.data_ptr(), A.stride(0), int(a_mn), B.data_ptr(), B.stride(0), int(b_mn),
                                   M, N, K, split_k, ctypes.byref(ep), L.current_stream()), "mmae_gemm_bf16")


def cast_bf16(src, dst=None):
    _need_cuda(src)
    assert src.dtype == torch.float32 and src.is_contiguous()
    if dst is None:
        dst = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    L.check(L.lib().mmae_cast_f32_to_bf16(src.data_ptr(), dst.data_ptr(), src.numel(), L.current_stream()),
            "mmae_cast_f32_to_bf16")
    return dst


def cast_colsum(src, dst=None, colsum=None):
    _need_cuda(src)
    M, N = src.shape
    L.check(L.lib().mmae_cast_colsum_f32(src.data_ptr(), src.stride(0), L.ptr(dst), dst.stride(0) if dst is not None else 0,
                                         L.ptr(colsum), M, N, L.current_stream()), "mmae_cast_colsum_f32")


def colsum_bf16(src, colsum):
    M, N = src.shape
    L.check(L.lib().mmae_colsum_bf16(src.data_ptr(), src.stride(0), colsum.data_ptr(), M, N, L.current_stream()),
            "mmae_colsum_bf16")


def transpose_bf16(src, dst=None):
    M, N = src.shape
    if dst is None:
        dst = torch.empty((N, M), dtype=torch.bfloat16, device=src.device)
    L.check(L.lib().mmae_transpose_bf16(src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0), M, N,
                                        L.current_stream()), "mmae_transpose_bf16")
    return dst


def layernorm_fwd(x, gamma, beta, eps=1e-6, out_bf16=True, out_f32=False):
    """x [M,D] fp32 -> (y_bf16|None, y_f32|None, mean[M], rstd[M])."""
    _need_cuda(x)
    M, D = x.shape
    yb = torch.empty((M, D), dtype=torch.bfloat16, device=x.device) if out_bf16 else None
    yf = torch.empty((M, D), dtype=torch.float32, device=x.device) if out_f32 else None
    mean = torch.empty(M, dtype=torch.float32, device=x.device)
    rstd = torch.empty(M, dtype=torch.float32, device=x.device)
    L.check(L.lib().mmae_layernorm_forward(x.data_ptr(), x.stride(0), gamma.data_ptr(), beta.data_ptr(), L.ptr(yb),
                                           D, L.ptr(yf), D, mean.data_ptr(), rstd.data_ptr(), M, D, eps,
                                           L.current_stream()), "mmae_layernorm_forward")
    return yb, yf, mean, rstd


def layernorm_bwd(dy, x, mean, rstd, gamma, dgamma, dbeta, dx_resid=None, dx=None):
    M, D = x.shape
    if dx is None:
        dx = torch.empty((M, D), dtype=torch.float32, device=x.device)
    L.check(L.lib().mmae_layernorm_backward(dy.data_ptr(), int(dy.dtype == torch.bfloat16), dy.stride(0), x.data_ptr(),
                                            x.stride(0), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(),
                                            L.ptr(dx_resid), dx_resid.stride(0) if dx_resid is not None else 0,
                                            dx.data_ptr(), dx.stride(0), L.ptr(dgamma), L.ptr(dbeta), M, D,
                                            L.current_stream()), "mmae_layernorm_backward")
    return dx


def attention_fwd(q, k, v, B, H, Nq, Nk, dh, scale, out=None):
    """q: [B*Nq, >=H*dh] view, k/v: [B*Nk, ...] views (bf16, unit inner stride). Returns (o [B*Nq, H*dh], lse)."""
    _need_cuda(q, k, v)
    if out is None:
        out = torch.empty((B * Nq, H * dh), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((B, H, Nq), dtype=torch.float32, device=q.device)
    L.check(L.lib().mmae_attention_forward(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(),
                                           v.stride(0), out.data_ptr(), out.stride(0), lse.data_ptr(), B, H, Nq, Nk,
                                           dh, scale, 0.0, None, L.current_stream()), "mmae_attention_forward")
    return out, lse


def attention_bwd(q, k, v, o, do, lse, dq, dk, dv, B, H, Nq, Nk, dh, scale):
    delta = torch.empty((B, H, Nq), dtype=torch.float32, device=q.device)
    L.check(L.lib().mmae_attention_backward(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(),
                                            v.stride(0), o.data_ptr(), o.stride(0), do.data_ptr(), do.stride(0),
                                            lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), dq.stride(0),
                                            dk.data_ptr(), dk.stride(0), dv.data_ptr(), dv.stride(0), B, H, Nq, Nk, dh,
                                            scale, 0.0, None, L.current_stream()), "mmae_attention_backward")



AUGMENT_KINDS = {"rgb": 0, "depth": 1, "semseg": 2, "semseg_coco": 2}     # task -> kind code of mmae_augment_batch


def augment_batch(host, dev, tasks, batch, size, map4, scratch_bytes, mean, std):
    """Resample one packed batch (multimae_b200.data.pack_batch: `host` its uint8 host buffer, `dev` the device copy) on
    the current stream: {task: fp32 [B,3,S,S] (rgb) | fp32 [B,1,S,S] (depth) | int64 [B,S/4,S/4] (semseg)}."""
    _need_cuda(dev)
    assert host.dtype == torch.uint8 and dev.dtype == torch.uint8 and host.numel() == dev.numel()
    kinds = [AUGMENT_KINDS[t] for t in tasks]
    T, S = len(tasks), int(size)
    outs = {}
    for t, k in zip(tasks, kinds):
        shape = (batch, S // 4, S // 4) if k == 2 else (batch, 3 if k == 0 else 1, S, S)
        outs[t] = torch.empty(shape, dtype=torch.int64 if k == 2 else torch.float32, device=dev.device)
    scratch = torch.empty(max(int(scratch_bytes), 16), dtype=torch.uint8, device=dev.device)
    ptrs = (ctypes.c_void_p * T)(*[outs[t].data_ptr() for t in tasks])
    L.check(L.lib().mmae_augment_batch(host.data_ptr(), dev.data_ptr(), host.numel(), batch, T, (ctypes.c_int * T)(*kinds),
                                       S, int(map4), scratch.data_ptr(), int(scratch_bytes), ptrs,
                                       (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std), L.current_stream()),
            "mmae_augment_batch")
    return outs


def cls_scratch_bytes(inter_bytes, batch, size, layers):
    """Scratch of mmae_cls_augment_batch: the horizontal pass's intermediates, then (with RandAugment layers) two uint8
    [B, S, S, 3] images and int32 [B, 1024] of per-sample tables, each 256-byte aligned."""
    a = lambda n: (int(n) + 255) // 256 * 256  # noqa: E731
    return a(inter_bytes) + (2 * a(batch * size * size * 3) + batch * 1024 * 4 if layers else 0)


def cls_augment_batch(host, dev, batch, size, layers, ops_offset, inter_bytes, mean, std, fill):
    """Resample, flip, RandAugment and normalise one packed classification batch (multimae_b200.data.pack_cls_batch) on
    the current stream: fp32 [B, 3, S, S]."""
    _need_cuda(dev)
    assert host.dtype == torch.uint8 and dev.dtype == torch.uint8 and host.numel() == dev.numel()
    S = int(size)
    out = torch.empty((batch, 3, S, S), dtype=torch.float32, device=dev.device)
    nbytes = cls_scratch_bytes(inter_bytes, batch, S, layers)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev.device)
    L.check(L.lib().mmae_cls_augment_batch(host.data_ptr(), dev.data_ptr(), host.numel(), batch, int(layers),
                                           int(ops_offset), S, (ctypes.c_int * 3)(*fill), scratch.data_ptr(), nbytes,
                                           out.data_ptr(), (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std),
                                           L.current_stream()), "mmae_cls_augment_batch")
    return out
