"""GPU: the asynchronous-epilogue wgmma GEMM (variants 8 / 9 / 10: 128 x 128 / 192 / 256 tiles) against the cooperative
kernel of the same tile (variants 1 / 3 / 2).

Both kernels run the same items in the same order with the same wgmma sequence per 64-row slab, and compute each output
element as alpha * acc (+ bias) before the one rounding to the output type; only the way the slab reaches global memory
differs (whole-slab 128B-swizzled staging and one bulk group per item against 64 x 32 boxes).  So the output bits must
be equal, margins included, for every epilogue form the kernel takes (bf16 or fp32 output, with or without a bias,
alpha != 1), operand-major pair, SM budget and tile width, and within the float64 budgets of test_cuda_gemm_schedule.py.

Shapes: one item; 63 items with M % 128, N % BN and K % 64 all != 0; 288 items of 3 ragged k-blocks, several per CTA at
every budget, so each warpgroup restages its slab region while the stores of its previous item may still be reading it."""
import ctypes

import pytest
import torch

from test_cuda_gemm_schedule import (BF16_LOCAL, BF16_TOL, F32_LOCAL, F32_TOL, FULL, KN, MAJORS,  # noqa: F401
                                     Worst, bf16_randn, canvas, check_local, dev, knobs, margins_intact, operand)

pytestmark = pytest.mark.gpu

COOP = {8: 1, 9: 3, 10: 2}              # asynchronous-epilogue variant -> cooperative variant of the same tile
STAGES = {8: 6, 9: 4, 10: 3}            # ring depth of its bf16 form (AsyncEpiCfg); the fp32 form (variant 8) has 5
ASYNC_FLAG = 16                         # profile-flag bit

# (name, output dtype, bias, alpha)
FORMS = [("bf16", torch.bfloat16, False, 1.0), ("bf16_bias", torch.bfloat16, True, 1.0),
         ("bf16_bias_alpha", torch.bfloat16, True, 0.75), ("f32", torch.float32, False, 1.0),
         ("f32_bias", torch.float32, True, 1.0), ("f32_alpha", torch.float32, False, -1.5)]


def forms_of(variant):
    """The fp32 forms for the 128-column kernel only: variants 9 / 10 hand fp32 outputs to the cooperative kernel."""
    return [f for f in FORMS if f[1] == torch.bfloat16 or variant == 8]


def compare_case(KN, knobs, dev, A, B, acc, variant, budget, worst, tag, forms=None):
    """Every form x operand-major pair: `variant` and its cooperative twin write the same bits into identical canvases,
    leave the margins alone, and are within the float64 budgets."""
    M, N = acc.shape
    for a_mn, b_mn in MAJORS:
        Aop, Bop = operand(A, a_mn), operand(B, b_mn)
        for name, dt, has_bias, alpha in forms or forms_of(variant):
            bias = torch.randn(N, device=dev) if has_bias else None
            ref = alpha * acc + (bias.double() if has_bias else 0.0)
            fill = 7.0 if dt == torch.bfloat16 else 1.0
            res = {}
            for v in (COOP[variant], variant):
                buf, view = canvas(M, N, dt, 16, fill, dev)
                knobs(budget=budget, variant=v)
                kw = dict(out_bf16=view) if dt == torch.bfloat16 else dict(out_f32=view)
                KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, bias=bias, alpha=alpha, split_k=1, **kw)
                res[v] = (buf, view)
            what = "%s %s (%d, %d) a_mn=%d b_mn=%d variant=%d budget=%d" % (tag, name, M, N, a_mn, b_mn, variant, budget)
            (cb, _), (nb, nv) = res[COOP[variant]], res[variant]
            assert torch.equal(cb, nb), (what, "differs from the cooperative kernel", int((cb != nb).sum()), "elements")
            assert margins_intact(nb, M, N, fill), (what, "margin written")
            is_bf16 = dt == torch.bfloat16
            check_local(nv, ref, BF16_TOL if is_bf16 else F32_TOL, BF16_LOCAL if is_bf16 else F32_LOCAL, worst, what)


def operands(M, N, K, dev):
    torch.manual_seed(M * 7 + N * 3 + K)
    s = K ** -0.25
    A, B = bf16_randn(M, K, scale=s, dev=dev), bf16_randn(N, K, scale=s, dev=dev)
    return A, B, A.double() @ B.double().t()


SHAPES = [pytest.param((96, 64, 200), id="1item"),
          pytest.param((1096, 776, 456), id="ragged-MNK"),
          pytest.param((4000, 1032, 136), id="288items-3kb")]


@pytest.mark.parametrize("variant", [8, 9, 10])
@pytest.mark.parametrize("budget", [FULL, 1, 3])
@pytest.mark.parametrize("shape", SHAPES)
def test_bitwise_equal_to_cooperative(dev, knobs, KN, shape, budget, variant):
    M, N, K = shape
    A, B, acc = operands(M, N, K, dev)
    worst = Worst()
    compare_case(KN, knobs, dev, A, B, acc, variant, budget, worst, "%s" % (shape,))
    worst.report("async epilogue %s budget %d variant %d" % (shape, budget, variant))


@pytest.mark.parametrize("variant", [8, 9, 10])
def test_ring_depth(dev, knobs, KN, variant):
    """Items of STAGES - 1, STAGES and STAGES + 1 k-blocks (ragged K), and for the fp32 form of its depth, 5: the
    producer wraps the ring inside an item, exactly at its end, or not at all."""
    worst = Worst()
    depths = {STAGES[variant]} | ({5} if variant == 8 else set())
    for S in sorted(depths):
        for K in (64 * (S - 2) + 40, 64 * S - 24, 64 * S + 8):
            A, B, acc = operands(1000, 520, K, dev)
            for budget in (FULL, 1):
                compare_case(KN, knobs, dev, A, B, acc, variant, budget, worst, "K=%d" % K)
    worst.report("async epilogue ring depth variant %d" % variant)


def test_bitwise_same_across_budgets_and_launches(dev, knobs, KN):
    """The output bits depend neither on the SM budget (grid size, items per CTA) nor on the launch."""
    torch.manual_seed(8)
    for (M, N, K) in [(1000, 776, 200), (648, 1024, 512)]:
        A, B = bf16_randn(M, K, scale=0.5, dev=dev), bf16_randn(N, K, scale=0.5, dev=dev)
        bias = torch.randn(N, device=dev)
        for variant in (8, 9, 10):
            for a_mn, b_mn in MAJORS:
                Aop, Bop = operand(A, a_mn), operand(B, b_mn)
                first = None
                for budget in (FULL, FULL, 1, 3, 17):
                    knobs(budget=budget, variant=variant)
                    o32 = torch.empty(M, N, device=dev)
                    o16 = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
                    KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, out_f32=o32)
                    KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, bias=bias, out_bf16=o16)
                    if first is None:
                        first = (o32, o16)
                        assert float((o32.double() - A.double() @ B.double().t()).norm()) < F32_TOL * float(o32.norm())
                    else:
                        assert torch.equal(o32, first[0]) and torch.equal(o16, first[1]), (M, N, K, variant, a_mn,
                                                                                            b_mn, budget)


ENC, DQ, DC = 128 * 99, 128 * 196, 128 * 99
# the bench step's forward (bf16 out + bias) and dgrad (bf16 out, MN-major weight) shapes
FWD = [(ENC, 2304, 768), (ENC, 768, 768), (ENC, 3072, 768), (ENC, 768, 3072), (DQ, 256, 256), (DC, 512, 256),
       (DQ, 1024, 256), (DQ, 256, 1024), (DQ, 768, 256), (DQ, 2128, 256)]
DGRAD = [(ENC, 3072, 768), (ENC, 768, 768), (ENC, 768, 3072), (ENC, 768, 2304), (DQ, 256, 256), (DC, 256, 512),
         (DQ, 1024, 256), (DQ, 256, 1024)]
WGRAD = [(768, 768, ENC), (3072, 768, ENC), (768, 3072, ENC), (256, 1024, DQ)]


def test_heuristic_runs_async_epilogue_at_bench_shapes(dev, knobs, KN):
    """Under the automatic choice the step's forward and dgrad GEMMs run the asynchronous-epilogue kernel (flag bit 4),
    and the weight gradients still split on the cooperative kernel."""
    from multimae_b200 import _lib as L
    lib = L.lib()
    knobs(budget=FULL, variant=-1)
    lib.mmae_profile_gemm(1)
    try:
        for M, N, K in FWD:
            A, B = bf16_randn(M, K, scale=0.5, dev=dev), bf16_randn(N, K, scale=0.5, dev=dev)
            KN.gemm(A, B, bias=torch.randn(N, device=dev), out_bf16=torch.empty(M, N, device=dev, dtype=torch.bfloat16))
        for M, N, K in DGRAD:
            A, B = bf16_randn(M, K, scale=0.5, dev=dev), bf16_randn(K, N, scale=0.5, dev=dev)
            KN.gemm(A, B, b_mn=True, out_bf16=torch.empty(M, N, device=dev, dtype=torch.bfloat16))
        for M, N, K in WGRAD:
            A, B = bf16_randn(K, M, scale=0.5, dev=dev), bf16_randn(K, N, scale=0.5, dev=dev)
            KN.gemm(A, B, a_mn=True, b_mn=True, out_f32=torch.zeros(M, N, device=dev), accumulate=True, split_k=0)
        buf = ctypes.create_string_buffer(1 << 16)
        n = lib.mmae_profile_gemm_dump(buf, len(buf))
    finally:
        lib.mmae_profile_gemm(0)
    flags = [int(line.split()[3]) for line in buf.raw[:max(n, 0)].decode().splitlines()]
    nf = len(FWD) + len(DGRAD)
    assert len(flags) == nf + len(WGRAD)
    assert all(f & ASYNC_FLAG for f in flags[:nf]), list(zip(FWD + DGRAD, flags[:nf]))
    assert all(f >> 8 > 1 and not f & ASYNC_FLAG for f in flags[nf:]), list(zip(WGRAD, flags[nf:]))
