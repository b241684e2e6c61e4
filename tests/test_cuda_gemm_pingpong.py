"""GPU: the ping-pong wgmma GEMM (variant 7) against the cooperative kernel of the same 128 x 128 tile (variant 1).

In the ping-pong kernel each consumer warpgroup owns whole 128 x 128 tiles and the two take turns on the tensor cores; in
the cooperative kernel both work on one tile, 64 rows each.  Each 64-row slab of a tile sees the same wgmma sequence (same
k order, same instruction shape) and the same epilogue code in both, so with split_k = 1 the outputs must be bitwise
equal, margins included, for every operand-major pair, epilogue form, output path (TMA store on / off) and SM budget.
The split-K forms add partial tiles in an order that is not fixed: they are held to the float64 budgets of
test_cuda_gemm_schedule.py instead, as is every variant-7 output.

Shapes: one item; 9 items (odd per CTA at budgets 1 and 3); 12 and 64 items (fewer than the SMs at full budget, 64 split
22 / 21 / 21 at budget 3); 288 items of 3 ragged k-blocks (two or three per CTA at full budget, the producer items ahead
of the consumers).  M % 128 != 0, N % 128 in {8, 64} and K % 64 != 0 throughout."""
import ctypes

import pytest
import torch

from test_cuda_gemm_schedule import (BF16_LOCAL, BF16_TOL, EPILOGUES, F32_LOCAL, F32_TOL, FULL, KN, MAJORS,  # noqa: F401
                                     Worst, bf16_randn, check_local, dev, epilogue_case, knobs, margins_intact,
                                     operand, run_gemm_case)

pytestmark = pytest.mark.gpu

PINGPONG, COOP128 = 7, 1
SPLIT_KINDS = ["split_bias", "split_bias_residual"]     # epilogue_case runs these with split_k = 3
UNSPLIT_KINDS = [k for k in EPILOGUES if k not in SPLIT_KINDS]

SHAPES = [pytest.param((96, 64, 200), id="1item"),
          pytest.param((1096, 64, 456), id="9items"),
          pytest.param((648, 136, 320), id="12items"),
          pytest.param((2000, 392, 712), id="64items"),
          pytest.param((4000, 1032, 136), id="288items-3kb")]


@pytest.mark.parametrize("budget", [FULL, 1, 3])
@pytest.mark.parametrize("shape", SHAPES)
def test_bitwise_equal_to_cooperative(dev, knobs, KN, shape, budget):
    """Every split_k = 1 epilogue form x operand-major pair x TMA store on / off: variant 7 writes exactly the bits
    variant 1 writes, into canvases that start out the same; variant 7 also within the float64 budgets."""
    M, N, K = shape
    torch.manual_seed(M * 7 + N * 3 + K)
    s = K ** -0.25
    A, B = bf16_randn(M, K, scale=s, dev=dev), bf16_randn(N, K, scale=s, dev=dev)
    acc = A.double() @ B.double().t()
    worst = Worst()
    for tma in (1, 0):
        for a_mn, b_mn in MAJORS:
            Aop, Bop = operand(A, a_mn), operand(B, b_mn)
            for kind in UNSPLIT_KINDS:
                kw, outs, sp = epilogue_case(kind, acc, 1, dev)
                assert sp == 1
                start = [buf.clone() for _, buf, _, _, _, _ in outs]
                res = {}
                for variant in (COOP128, PINGPONG):
                    for (_, buf, _, _, _, _), b0 in zip(outs, start):
                        buf.copy_(b0)
                    knobs(budget=budget, variant=variant, tma_store=tma)
                    KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, split_k=1, **kw)
                    res[variant] = [buf.clone() for _, buf, _, _, _, _ in outs]
                for (name, buf, view, fill, ref, is_bf16), c, p in zip(outs, res[COOP128], res[PINGPONG]):
                    what = "%s (%d, %d, %d) a_mn=%d b_mn=%d tma=%d budget=%d %s" % (kind, M, N, K, a_mn, b_mn, tma,
                                                                                   budget, name)
                    assert torch.equal(c, p), (what, "differs from the cooperative kernel",
                                               int((c != p).sum()), "elements")
                    assert margins_intact(buf, M, N, fill), (what, "margin written")
                    check_local(view, ref, BF16_TOL if is_bf16 else F32_TOL, BF16_LOCAL if is_bf16 else F32_LOCAL,
                                worst, what)
    worst.report("ping-pong %s budget %d" % (shape, budget))


@pytest.mark.parametrize("budget", [FULL, 1, 3])
@pytest.mark.parametrize("shape", SHAPES)
def test_split_k_within_float64_budgets(dev, knobs, KN, shape, budget):
    """Split-K (3 splits: bias and residual exactly once, TMA reduce-add or red.global adds) on the ping-pong kernel."""
    M, N, K = shape
    worst = Worst()
    for tma in (1, 0):
        knobs(budget=budget, variant=PINGPONG, tma_store=tma)
        run_gemm_case(KN, dev, M, N, K, SPLIT_KINDS, worst, tag="v7 b%d tma%d" % (budget, tma))
    worst.report("ping-pong split-K %s budget %d" % (shape, budget))


def test_bitwise_same_across_budgets_and_launches(dev, knobs, KN):
    """As for variants 0-6 in test_cuda_gemm_schedule.py: one warpgroup sums each tile in a fixed k order, so the output
    bits may not depend on the SM budget (grid size, items per CTA, which warpgroup takes an item) or on the launch."""
    torch.manual_seed(PINGPONG)
    for (M, N, K) in [(1000, 776, 200), (648, 1024, 512)]:
        A, B = bf16_randn(M, K, scale=0.5, dev=dev), bf16_randn(N, K, scale=0.5, dev=dev)
        bias = torch.randn(N, device=dev)
        for a_mn, b_mn in MAJORS:
            Aop, Bop = operand(A, a_mn), operand(B, b_mn)
            first = None
            for budget in (FULL, FULL, 1, 3, 17):
                knobs(budget=budget, variant=PINGPONG)
                o32 = torch.empty(M, N, device=dev)
                o16 = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
                KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, out_f32=o32)
                KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, bias=bias, act=1, out_bf16=o16)
                if first is None:
                    first = (o32, o16)
                    assert float((o32.double() - A.double() @ B.double().t()).norm()) < F32_TOL * float(o32.norm())
                else:
                    assert torch.equal(o32, first[0]) and torch.equal(o16, first[1]), (M, N, K, a_mn, b_mn, budget)


# (M, N, K) of the bench step's weight gradients: both operands MN-major, long K, fp32 accumulate, automatic split
ENC, DQ = 128 * 99, 128 * 196
WGRAD = [(768, 768, ENC), (3072, 768, ENC), (768, 3072, ENC), (256, 1024, DQ)]


def test_heuristic_never_picks_pingpong(dev, knobs, KN):
    """The automatic choice does not run the ping-pong kernel (bit 2 of the profile flags): it measured slower than the
    cooperative tiles over the bench step.  The weight gradients split at full budget."""
    from multimae_b200 import _lib as L
    lib = L.lib()
    knobs(budget=FULL, variant=-1)
    fwd = [(ENC, 2304, 768), (ENC, 768, 768), (DQ, 256, 256), (DQ, 1024, 256), (DQ, 2128, 256)]
    lib.mmae_profile_gemm(1)
    try:
        for M, N, K in fwd:
            A, B = bf16_randn(M, K, scale=0.5, dev=dev), bf16_randn(N, K, scale=0.5, dev=dev)
            KN.gemm(A, B, bias=torch.randn(N, device=dev), out_bf16=torch.empty(M, N, device=dev, dtype=torch.bfloat16))
        for M, N, K in WGRAD:
            A, B = bf16_randn(K, M, scale=0.5, dev=dev), bf16_randn(K, N, scale=0.5, dev=dev)
            KN.gemm(A, B, a_mn=True, b_mn=True, out_f32=torch.zeros(M, N, device=dev), accumulate=True, split_k=0)
        buf = ctypes.create_string_buffer(1 << 16)
        n = lib.mmae_profile_gemm_dump(buf, len(buf))
    finally:
        lib.mmae_profile_gemm(0)
    flags = [int(line.split()[3]) for line in buf.raw[:max(n, 0)].decode().splitlines()]
    assert len(flags) == len(fwd) + len(WGRAD)
    assert not any(f & 4 for f in flags), flags
    assert all(f >> 8 > 1 for f in flags[len(fwd):]), list(zip(WGRAD, flags[len(fwd):]))
