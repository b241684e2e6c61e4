"""GPU: every primitive of the C ABI against a plain PyTorch fp32 computation of the same op on the same inputs.

Tolerances: fp32-accumulating GEMM on bf16 inputs vs fp32 matmul of the same bf16 values: 3e-5 relative L2 (accumulation
order only); outputs rounded to bf16: 4e-3; fp32 element-wise kernels: 1e-5.  Attention, both tiers, is held to float64
element by element in test_cuda_attention_float64.py."""
import os

import pytest
import torch

from helpers import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    torch.manual_seed(0)
    return torch.device("cuda:0")


def _bf16(dev, *shape, scale=0.5):
    return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)


@pytest.fixture()
def KN():
    from multimae_b200 import _lib as L
    from multimae_b200 import kernels
    yield kernels
    L.lib().mmae_gemm_set_variant(-1)
    L.lib().mmae_gemm_set_tma_store(1)
    L.lib().mmae_attention_set_tc(-1)
    L.lib().mmae_set_sm_budget(int(os.environ.get("MMAE_SM_BUDGET", 0)))


@pytest.mark.parametrize("variant", [1, 2, 3])
@pytest.mark.parametrize("shape", [(128, 128, 64), (256, 384, 768), (200, 136, 200), (396, 2128, 256), (1000, 768, 512),
                                   (2560, 2304, 768)])
def test_gemm_all_operand_majors(dev, KN, variant, shape):
    from multimae_b200 import _lib as L
    L.check(L.lib().mmae_gemm_set_variant(variant))
    M, N, K = shape
    A, B = _bf16(dev, M, K), _bf16(dev, N, K)
    ref = A.float() @ B.float().t()
    for a_mn in (False, True):
        for b_mn in (False, True):
            if a_mn and M % 8:
                continue
            out = torch.zeros(M, N, device=dev)
            KN.gemm(A.t().contiguous() if a_mn else A, B.t().contiguous() if b_mn else B, a_mn=a_mn, b_mn=b_mn, out_f32=out)
            assert rel_l2(out, ref) < 3e-5, (variant, shape, a_mn, b_mn, rel_l2(out, ref))


@pytest.mark.parametrize("variant", [1, 2, 3, -1])
def test_gemm_split_k_wgrad_shapes(dev, KN, variant):
    from multimae_b200 import _lib as L
    L.check(L.lib().mmae_gemm_set_variant(variant))
    for (M, N, K, split) in [(768, 768, 12672, 1), (768, 768, 12672, 4), (768, 3072, 1280, 3), (256, 256, 25088, 16),
                             (256, 256, 25088, 0), (2304, 768, 12672, 0)]:          # 0 = automatic split + tile choice
        A, B = _bf16(dev, M, K), _bf16(dev, N, K)
        out = torch.zeros(M, N, device=dev)
        KN.gemm(A.t().contiguous(), B.t().contiguous(), a_mn=True, b_mn=True, out_f32=out, split_k=split)
        assert rel_l2(out, A.float() @ B.float().t()) < 3e-5


@pytest.mark.parametrize("variant", [1, 2, 3])
def test_gemm_fused_epilogues(dev, KN, variant):
    from multimae_b200 import _lib as L
    L.check(L.lib().mmae_gemm_set_variant(variant))
    M, N, K = 384, 512, 256
    A, B = _bf16(dev, M, K), _bf16(dev, N, K)
    bias, resid = torch.randn(N, device=dev), torch.randn(M, N, device=dev)
    acc = A.float() @ B.float().t()
    out = torch.empty(M, N, device=dev)
    KN.gemm(A, B, bias=bias, out_f32=out)
    assert rel_l2(out, acc + bias) < 3e-5
    outb = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    pre = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    KN.gemm(A, B, bias=bias, act=1, preact=pre, out_bf16=outb)
    assert rel_l2(outb, torch.nn.functional.gelu(acc + bias)) < 4e-3 and rel_l2(pre, acc + bias) < 4e-3
    KN.gemm(A, B, bias=bias, residual=resid, out_f32=out)
    assert rel_l2(out, acc + bias + resid) < 3e-5
    z = torch.randn(M, N, device=dev).to(torch.bfloat16)
    zf = z.float().requires_grad_(True)
    torch.nn.functional.gelu(zf).sum().backward()
    KN.gemm(A, B, dgelu_z=z, out_bf16=outb)
    assert rel_l2(outb, acc * zf.grad) < 4e-3
    out = torch.ones(M, N, device=dev)
    KN.gemm(A, B, out_f32=out, accumulate=True, alpha=0.5)
    assert rel_l2(out, 1 + 0.5 * acc) < 3e-5


@pytest.mark.parametrize("variant", [1, 2, 3])
@pytest.mark.parametrize("shape", [(128, 128, 64), (200, 136, 200), (396, 2128, 256), (1000, 776, 512), (2560, 2304, 768),
                                   (25088, 256, 256)])
def test_gemm_tma_store_epilogue(dev, KN, variant, shape):
    """bf16 outputs through shared memory + TMA tile stores: ragged M / N edges, a strided output view, bias and GELU;
    bit-identical to the per-thread store path and untouched bytes outside the [M, N] view.  Both paths also run with an
    SM budget of 1 (one CTA walks every tile, reusing its staging boxes across tiles) and must give the same
    bits as with every SM."""
    from multimae_b200 import _lib as L
    L.check(L.lib().mmae_gemm_set_variant(variant))
    M, N, K = shape
    A, B = _bf16(dev, M, K), _bf16(dev, N, K)
    bias = torch.randn(N, device=dev)
    acc = A.float() @ B.float().t()
    for kw, ref in (({}, acc), ({"bias": bias}, acc + bias), ({"bias": bias, "act": 1}, torch.nn.functional.gelu(acc + bias)),
                    ({"alpha": 0.25}, 0.25 * acc)):
        outs = []
        for budget in (0, 1):
            L.lib().mmae_set_sm_budget(budget)
            for tma in (1, 0):
                L.lib().mmae_gemm_set_tma_store(tma)
                buf = torch.full((M + 3, N + 16), 7.0, device=dev, dtype=torch.bfloat16)
                KN.gemm(A, B, out_bf16=buf[:M, :N], **kw)
                assert bool((buf[M:] == 7).all()) and bool((buf[:, N:] == 7).all()), (variant, shape, kw.keys(), tma, budget)
                outs.append(buf[:M, :N].clone())
        assert rel_l2(outs[0], ref) < 4e-3, (variant, shape, list(kw), rel_l2(outs[0], ref))
        for o in outs[1:]:
            assert torch.equal(outs[0], o), (variant, shape, list(kw))
    # fp32 outputs: plain tile stores, and reduce-add tiles for accumulate / split-K (margins stay untouched)
    for kw, ref in (({"bias": bias}, acc + bias), ({"accumulate": True, "alpha": 0.5}, 1 + 0.5 * acc),
                    ({"accumulate": True, "split_k": 3, "bias": bias}, 1 + acc + bias)):
        outs = []
        for budget in (0, 1):
            L.lib().mmae_set_sm_budget(budget)
            for tma in (1, 0):
                L.lib().mmae_gemm_set_tma_store(tma)
                buf = torch.full((M + 3, N + 8), 1.0, device=dev)
                KN.gemm(A, B, out_f32=buf[:M, :N], **kw)
                assert bool((buf[M:] == 1).all()) and bool((buf[:, N:] == 1).all()), (variant, shape, list(kw), tma, budget)
                assert rel_l2(buf[:M, :N], ref) < 3e-5, (variant, shape, list(kw), tma, budget, rel_l2(buf[:M, :N], ref))
                outs.append(buf[:M, :N].clone())
        if "split_k" not in kw:
            for o in outs[1:]:
                assert torch.equal(outs[0], o), (variant, shape, list(kw))


def test_gemm_heuristic_agrees_with_every_tile(dev, KN):
    """On the big encoder shapes the heuristic's choice and the 128 x 128, 128 x 256 and 128 x 192 tiles give the same
    results."""
    from multimae_b200 import _lib as L
    for (M, N, K, b_mn) in [(12672, 3072, 768, False), (12672, 3072, 768, True), (12672, 768, 3072, False)]:
        A, B = _bf16(dev, M, K), _bf16(dev, N, K)
        bias = torch.randn(N, device=dev)
        outs = []
        for variant in (-1, 1, 2, 3):
            L.check(L.lib().mmae_gemm_set_variant(variant))
            o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            KN.gemm(A, B.t().contiguous() if b_mn else B, b_mn=b_mn, bias=bias, out_bf16=o)
            outs.append(o)
        for o in outs[1:]:
            assert rel_l2(outs[0], o) < 1e-4, (M, N, K, b_mn)


def test_gemm_rejects_bad_arguments(dev, KN):
    from multimae_b200 import _lib as L
    A, B = _bf16(dev, 128, 64), _bf16(dev, 130, 64)          # N = 130 is not a multiple of 8
    with pytest.raises(L.MmaeError):
        KN.gemm(A, B, out_f32=torch.empty(128, 130, device=dev))
    with pytest.raises(L.MmaeError):                          # no output
        KN.gemm(A, _bf16(dev, 128, 64))


def test_elementwise(dev, KN):
    x = torch.randn(1000, 776, device=dev)
    assert rel_l2(KN.cast_bf16(x), x.to(torch.bfloat16)) == 0.0
    dst = torch.empty(1000, 776, device=dev, dtype=torch.bfloat16)
    cs = torch.zeros(776, device=dev)
    KN.cast_colsum(x, dst, cs)
    assert rel_l2(dst, x.to(torch.bfloat16)) == 0.0 and rel_l2(cs, x.sum(0)) < 1e-5
    cs2 = torch.zeros(776, device=dev)
    KN.colsum_bf16(dst, cs2)
    assert rel_l2(cs2, dst.float().sum(0)) < 1e-5
    assert rel_l2(KN.transpose_bf16(dst), dst.t()) == 0.0


# every supported width (D = 128 .. 1024 in steps of 128); M = 12672 / 25088 (the encoder / decoder token counts at batch
# 128) give every warp of the one-wave backward grid several rows, so that the next-row prefetch runs
@pytest.mark.parametrize("shape", [(1000, 768), (396, 256), (130, 1024), (7, 128), (33, 384), (1000, 512), (31, 640),
                                   (200, 896), (12672, 768), (25088, 256), (12672, 1024), (25088, 128)])
def test_layernorm(dev, KN, shape):
    """Forward and backward against float64; dgamma / dbeta accumulate (+=) onto non-zero values."""
    M, D = shape
    x = torch.randn(M, D, device=dev) * 2 + 0.5
    gam, bet = torch.randn(D, device=dev), torch.randn(D, device=dev)
    yb, yf, mean, rstd = KN.layernorm_fwd(x, gam, bet, 1e-6, out_bf16=True, out_f32=True)
    xr, gr, br = (t.double().requires_grad_(True) for t in (x, gam, bet))
    ref = torch.nn.functional.layer_norm(xr, (D,), gr, br, 1e-6)
    assert rel_l2(yf, ref) < 1e-5 and rel_l2(yb, ref) < 4e-3
    dy, resid = torch.randn(M, D, device=dev), torch.randn(M, D, device=dev)
    ref.backward(dy.double())
    g0, b0 = torch.randn(D, device=dev), torch.randn(D, device=dev)
    dgam, dbet = g0.clone(), b0.clone()
    dx = KN.layernorm_bwd(dy, x, mean, rstd, gam, dgam, dbet, dx_resid=resid)
    assert rel_l2(dx, xr.grad + resid.double()) < 1e-5
    assert rel_l2(dgam, gr.grad + g0.double()) < 1e-4 and rel_l2(dbet, br.grad + b0.double()) < 1e-4


@pytest.mark.parametrize("case", [(3, 3, 14, 14, 16), (2, 1, 14, 14, 16), (2, 133, 14, 14, 4), (2, 5, 3, 7, 8), (1, 2, 2, 3, 4)])
def test_unpatchify_and_patchify_bf16(dev, case):
    """tokens [B*nh*nw, C*P*P] (c, py, px) <-> image [B, C, nh*P, nw*P] (output_adapters.py:277-280), strided token rows."""
    from multimae_b200 import _lib as L
    B, C, nh, nw, P = case
    cols = C * P * P
    tok = torch.full((B * nh * nw, cols + 8), 3.0, device=dev, dtype=torch.bfloat16)
    tok[:, :cols] = _bf16(dev, B * nh * nw, cols)
    img = torch.empty(B, C, nh * P, nw * P, device=dev)
    L.check(L.lib().mmae_unpatchify_bf16(tok.data_ptr(), tok.stride(0), img.data_ptr(), B, C, nh, nw, P, L.current_stream()))
    ref = tok[:, :cols].float().reshape(B, nh, nw, C, P, P).permute(0, 3, 1, 4, 2, 5).reshape(B, C, nh * P, nw * P)
    assert torch.equal(img, ref)
    back = torch.full_like(tok, 5.0)
    L.check(L.lib().mmae_patchify_bf16(img.data_ptr(), back.data_ptr(), back.stride(0), B, C, nh, nw, P, L.current_stream()))
    assert torch.equal(back[:, :cols], tok[:, :cols]) and bool((back[:, cols:] == 5).all())


def _depth_cases():
    g = torch.Generator().manual_seed(17)
    a = torch.randn(4, 1, 224, 224, generator=g)
    a[1] = a[1].abs() * 3 + 0.5                      # metric-depth-like: positive, skewed, few exponent bins
    a[2] = torch.round(a[2] * 4) / 4                 # heavy ties, also across both cut points
    a[3, :, :120] = -2.5                             # one value covering more than half of the map (L == H side cases)
    yield "224", a
    yield "448 (global-memory passes)", torch.randn(2, 1, 448, 448, generator=g) * 5 - 1
    yield "odd length (scalar path)", torch.randn(3, 1, 13, 77, generator=g)
    c = torch.full((2, 1, 32, 32), 0.75)
    c[0, 0, 0, :20] = torch.randn(20, generator=g)    # both cut values fall into the constant run (L == H, variance 0)
    yield "mostly constant", c
    yield "tiny", torch.tensor([[3.0, 1.0, 2.0, 2.0, 5.0, -1.0, 0.0, -0.0, 4.0, 2.0]]).reshape(1, 1, 2, 5)


@pytest.mark.parametrize("variant", [2, 1])     # 2: the default (histogram copies + cluster split), 1: the single-CTA kernel
def test_standardize_depth_against_oracle_and_golden(dev, golden_dir, variant):
    """mmae_standardize_depth (radix select of the two cut values) against the sort-based oracle
    (run_pretraining_multimae.py:487-492): fp32, differences only from the summation order -> 2e-5 absolute on O(1)
    outputs, 1e-5 relative on mean / variance; in-place operation; fixture recorded from the reference's own lines."""
    import os
    from multimae_b200 import functional as Fn
    from oracle import multimae_oracle as O
    fx = torch.load(os.path.join(golden_dir, "depth_std.pt"), map_location="cpu", weights_only=False)
    Fn.L.check(Fn.L.lib().mmae_standardize_depth_set_variant(variant))
    got = Fn.standardize_depth(fx["depth"].to(dev))
    assert got.shape == fx["standardized"].shape
    assert float((got.cpu() - fx["standardized"]).abs().max()) < 2e-5
    for name, x in _depth_cases():
        ref = O.standardize_depth(x)
        flat = x.reshape(x.shape[0], -1)
        n = flat.shape[1]
        trunc = torch.sort(flat, dim=1)[0][:, int(0.1 * n):int(0.9 * n)]
        xd = x.to(dev)
        out, stats = Fn.standardize_depth(xd, return_stats=True)
        assert out.shape == x.shape and torch.equal(xd.cpu(), x), name           # input untouched
        torch.testing.assert_close(stats[:, 0].cpu(), trunc.mean(1), rtol=1e-5, atol=1e-6, msg=name)
        torch.testing.assert_close(stats[:, 1].cpu(), trunc.var(1), rtol=1e-5, atol=1e-7, msg=name)
        scale = max(1.0, float(ref.abs().max()))
        assert float((out.cpu() - ref).abs().max()) < 2e-5 * scale, (name, float((out.cpu() - ref).abs().max()))
        same = Fn.standardize_depth(xd, out=xd)                                   # in place
        assert same.data_ptr() == xd.data_ptr() and torch.equal(same, out), name
    with pytest.raises(TypeError):
        Fn.standardize_depth(torch.zeros(2, 1, 8, 8, device=dev, dtype=torch.float16))
    Fn.L.check(Fn.L.lib().mmae_standardize_depth_set_variant(2))


# ---------------------------------------------------------------------------------------------------------------------
# fp32 tier primitives (fp32_output_adapters): 3 x bf16 split Linear, fp32 GELU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(48, 2128, 128), (392, 256, 768), (1000, 1024, 256), (48, 128, 128)])
def test_linear_f32_split_gemm(dev, shape):
    from multimae_b200 import _lib as L
    lib = L.lib()
    M, N, K = shape
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).to(dev)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    res = torch.randn(M, N, generator=g).to(dev)
    dy = torch.randn(M, N, generator=g).to(dev)
    ws = torch.empty(lib.mmae_linear_f32_workspace_bytes(M, N, K), dtype=torch.uint8, device=dev)
    y = torch.empty(M, N, device=dev)
    L.check(lib.mmae_linear_f32_forward(x.data_ptr(), W.data_ptr(), b.data_ptr(), res.data_ptr(), y.data_ptr(), M, N, K,
                                        ws.data_ptr(), L.current_stream()))
    ref = (x.double() @ W.double().t() + b.double() + res.double())
    assert rel_l2(y, ref.float()) < 2e-5, rel_l2(y, ref.float())
    dx = torch.empty(M, K, device=dev)
    dW = torch.full((N, K), 0.5, device=dev)          # accumulated into
    db = torch.full((N,), 0.25, device=dev)
    L.check(lib.mmae_linear_f32_backward(x.data_ptr(), W.data_ptr(), dy.data_ptr(), dx.data_ptr(), dW.data_ptr(), db.data_ptr(),
                                         M, N, K, ws.data_ptr(), L.current_stream()))
    assert rel_l2(dx, (dy.double() @ W.double()).float()) < 2e-5
    assert rel_l2(dW - 0.5, (dy.double().t() @ x.double()).float()) < 2e-5
    assert rel_l2(db - 0.25, dy.double().sum(0).float()) < 1e-5


def test_gelu_f32(dev):
    from multimae_b200 import _lib as L
    lib = L.lib()
    z = (torch.randn(1000, 64, device=dev) * 2).requires_grad_(True)
    a = torch.empty_like(z)
    L.check(lib.mmae_gelu_f32(z.data_ptr(), a.data_ptr(), z.numel(), 0, L.current_stream()))
    ref = torch.nn.functional.gelu(z)
    assert rel_l2(a, ref.detach()) < 1e-6
    g = torch.randn_like(z)
    ref.backward(g)
    gz = g.clone()
    L.check(lib.mmae_gelu_f32(z.data_ptr(), gz.data_ptr(), z.numel(), 1, L.current_stream()))
    assert rel_l2(gz, z.grad) < 1e-5
