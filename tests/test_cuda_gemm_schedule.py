"""GPU: the persistent wgmma GEMM's work-item schedule and the SM-count-sized reduction kernels under reduced SM budgets,
against float64.

The GEMM grid holds at most one CTA (or two-CTA cluster) per SM of the budget (mmae_set_sm_budget), and each walks a
strided sequence of work items (n-tile fastest, then m-tile, then split) with a TMA ring whose slot and phase run across
items.  The budget also sets the tile / split choice, the row blocking of the column-sum kernels and of their last-block
fold, and the LayerNorm backward grid.  Budget 1 puts every item (every row block) on one CTA; budgets 3, 7 and 17 are odd,
so that sms / 2 truncates for the cluster variants.

Error budgets, against a float64 reference of the same bf16 operands:
  * whole matrix, relative L2: fp32 outputs 3e-5 (fp32 accumulation order only), bf16 outputs 4e-3 (the suite's budgets);
  * per 64-row x 32-column box (the TMA-store box; boxes start at multiples of 64 rows / 32 columns for every tile) and per
    output row, relative L2: fp32 outputs F32_LOCAL = 1e-4.  Rounding to bf16 (round to nearest) moves an element by at
    most 2^-8 of its magnitude, so a bf16 output block is within 2^-8 (1 + d) + d of the float64 value when the fp32
    value it was rounded from is within d: BF16_LOCAL = 2^-8 + 2 * F32_LOCAL.  A box or a row that a scheduling bug
    computes wrongly (a missed or doubled split, a stale staging box, another CTA's rows) is off by far more, while the
    whole-matrix figure of a 2560 x 2304 output dilutes one 10 %-wrong box to ~2e-3.
Every test prints the worst box / row error it saw as a fraction of its budget."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

F32_TOL, BF16_TOL = 3e-5, 4e-3
F32_LOCAL = 1e-4
BF16_LOCAL = 2.0 ** -8 + 2 * F32_LOCAL
SUM_TOL = 1e-5           # column sums (bias / gamma / beta gradients) against float64, relative L2

FULL = 0                 # budget 0: every SM
MAJORS = [(False, False), (False, True), (True, False), (True, True)]

# variant -> (tile width BN, TMA ring stages), gemm_wgmma.cu variant_bn / GemmCfg
VARIANT_TILE = {0: (64, 8), 1: (128, 6), 2: (256, 4), 3: (192, 4), 4: (256, 4), 5: (192, 4), 6: (128, 6)}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.fixture()
def knobs():
    """set(budget=, variant=, tma_store=) for one test; the library defaults come back on teardown (the budget from
    MMAE_SM_BUDGET, as at library load: there is no getter), so later tests in the same process see them."""
    from multimae_b200 import _lib as L
    lib = L.lib()

    def set_(budget=None, variant=None, tma_store=None):
        if budget is not None:
            L.check(lib.mmae_set_sm_budget(budget))
        if variant is not None:
            L.check(lib.mmae_gemm_set_variant(variant))
        if tma_store is not None:
            L.check(lib.mmae_gemm_set_tma_store(tma_store))
    yield set_
    lib.mmae_set_sm_budget(int(os.environ.get("MMAE_SM_BUDGET", 0)))
    lib.mmae_gemm_set_variant(-1)
    lib.mmae_gemm_set_tma_store(1)


# ------------------------------------------------------------------------------------------------------ checking helpers
class Worst:
    """Largest per-box / per-row error of a test as a fraction of its budget (printed at the end)."""

    def __init__(self):
        self.ratio, self.what = 0.0, ""

    def add(self, r, what):
        if r > self.ratio:
            self.ratio, self.what = r, what

    def report(self, name):
        print("%s: worst box/row error %.3f of its budget (%s)" % (name, self.ratio, self.what))


def check_local(out, ref, tol, local, worst, what):
    """Relative L2 of `out` against the float64 `ref`, over the whole matrix (< tol), per 64 x 32 box and per row
    (< local)."""
    d = out.double() - ref
    whole = float(d.norm() / ref.norm().clamp_min(1e-300))
    assert whole < tol, (what, "whole", whole)
    M, N = ref.shape
    pm, pn = (-M) % 64, (-N) % 32
    d2 = F.pad(d * d, (0, pn, 0, pm)).reshape((M + pm) // 64, 64, (N + pn) // 32, 32).sum((1, 3))
    r2 = F.pad(ref * ref, (0, pn, 0, pm)).reshape((M + pm) // 64, 64, (N + pn) // 32, 32).sum((1, 3))
    box = (d2.sqrt() / r2.sqrt().clamp_min(1e-300)).flatten()
    row = (d * d).sum(1).sqrt() / (ref * ref).sum(1).sqrt().clamp_min(1e-300)
    bi, ri = int(box.argmax()), int(row.argmax())
    b, r = float(box[bi]), float(row[ri])
    worst.add(max(b, r) / local, what)
    nb = (N + pn) // 32
    assert b < local, (what, "box (rows %d.., cols %d..)" % (64 * (bi // nb), 32 * (bi % nb)), b)
    assert r < local, (what, "row %d" % ri, r)


def canvas(M, N, dtype, right, fill, dev):
    """[M, N] view into a larger buffer filled with `fill`: one margin row above, two below, 8 columns left and `right`
    on the right (leading dimension N + 8 + right, a multiple of 8).  Returns (buffer, view)."""
    buf = torch.full((M + 3, N + 8 + right), fill, dtype=dtype, device=dev)
    return buf, buf[1:1 + M, 8:8 + N]


def margins_intact(buf, M, N, fill):
    chk = buf.clone()
    chk[1:1 + M, 8:8 + N] = fill
    return bool((chk == fill).all())


def operand(x, mn):
    """What the kernel reads for the K-major [rows, K] operand x: x (K-major) or its transpose [K, rows] (MN-major), as a
    strided view (leading dimension > its width) whose padding holds NaN, so a read past the logical edge shows."""
    src = x.t() if mn else x
    r, c = src.shape
    buf = torch.full((r, c + 24), float("nan"), dtype=torch.bfloat16, device=x.device)
    buf[:, 8:8 + c] = src
    return buf[:, 8:8 + c]


def gelu64(v):
    return v * 0.5 * (1.0 + torch.erf(v / math.sqrt(2.0)))


def dgelu64(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def bf16_randn(*shape, scale, dev):
    return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------- GEMM epilogues
EPILOGUES = ["bias_bf16", "bias_gelu_bf16", "preact_act", "dgelu", "residual", "f32", "accumulate", "split_bias",
             "split_bias_residual", "f32_and_bf16"]


def epilogue_case(kind, acc, split, dev):
    """(kwargs of kernels.gemm, [(name, buffer, view, fill, float64 reference, is_bf16)], split_k) of one epilogue kind
    on the float64 product `acc`; every tensor has its own leading dimension != N."""
    M, N = acc.shape
    bias = torch.randn(N, device=dev)
    kw, outs = {}, []

    def out(name, dtype, right, fill, ref, init=None):
        buf, view = canvas(M, N, dtype, right, fill, dev)
        if init is not None:
            view.copy_(init)
        outs.append((name, buf, view, fill, ref, dtype == torch.bfloat16))
        return view

    v = acc + bias.double()
    if kind == "bias_bf16":
        kw = dict(bias=bias, out_bf16=out("out_bf16", torch.bfloat16, 16, 7.0, v))
    elif kind == "bias_gelu_bf16":
        kw = dict(bias=bias, act=1, out_bf16=out("out_bf16", torch.bfloat16, 16, 7.0, gelu64(v)))
    elif kind == "preact_act":
        kw = dict(bias=bias, act=1, preact=out("preact", torch.bfloat16, 32, 5.0, v),
                  out_bf16=out("out_bf16", torch.bfloat16, 16, 7.0, gelu64(v)))
    elif kind == "dgelu":
        zb, z = canvas(M, N, torch.bfloat16, 48, 3.0, dev)
        z.copy_(torch.randn(M, N, device=dev) * 1.5)
        kw = dict(dgelu_z=z, out_bf16=out("out_bf16", torch.bfloat16, 16, 7.0, acc * dgelu64(z.double())))
    elif kind == "residual":
        rb, res = canvas(M, N, torch.float32, 40, 3.0, dev)
        res.copy_(torch.randn(M, N, device=dev))
        kw = dict(bias=bias, residual=res, out_f32=out("out_f32", torch.float32, 24, 1.0, v + res.double()))
    elif kind == "f32":                      # a split store adds onto the destination: zero it then
        kw = dict(out_f32=out("out_f32", torch.float32, 24, 1.0, acc, None if split == 1 else torch.zeros(M, N)))
    elif kind == "accumulate":
        d0 = torch.randn(M, N, device=dev)
        kw = dict(accumulate=True, alpha=0.5, out_f32=out("out_f32", torch.float32, 24, 1.0, d0.double() + 0.5 * acc, d0))
    elif kind == "split_bias":              # the bias exactly once, whatever the split count (TMA reduce-add tiles)
        kw = dict(bias=bias, out_f32=out("out_f32", torch.float32, 24, 1.0, v, torch.zeros(M, N)))
        split = 3 if split == 1 else split
    elif kind == "split_bias_residual":     # bias and residual exactly once (a residual takes the register path)
        rb, res = canvas(M, N, torch.float32, 40, 3.0, dev)
        res.copy_(torch.randn(M, N, device=dev))
        kw = dict(bias=bias, residual=res, out_f32=out("out_f32", torch.float32, 24, 1.0, v + res.double(), torch.zeros(M, N)))
        split = 3 if split == 1 else split
    elif kind == "f32_and_bf16":
        kw = dict(bias=bias, out_f32=out("out_f32", torch.float32, 24, 1.0, v), out_bf16=out("out_bf16", torch.bfloat16, 16, 7.0, v))
    else:
        raise AssertionError(kind)
    return kw, outs, split


def run_gemm_case(KN, dev, M, N, K, kinds, worst, split=1, majors=MAJORS, tag=""):
    """Every kind x operand-major combination of one shape, each output checked against float64 (check_local) with its
    margins untouched."""
    torch.manual_seed(M * 7 + N * 3 + K)
    s = K ** -0.25                                # |acc| ~ 1 whatever K
    A, B = bf16_randn(M, K, scale=s, dev=dev), bf16_randn(N, K, scale=s, dev=dev)
    acc = A.double() @ B.double().t()
    for a_mn, b_mn in majors:
        if a_mn and M % 8:
            continue
        Aop, Bop = operand(A, a_mn), operand(B, b_mn)
        for kind in kinds:
            kw, outs, sp = epilogue_case(kind, acc, split, dev)
            KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, split_k=sp, **kw)
            for name, buf, view, fill, ref, is_bf16 in outs:
                what = "%s %s (%d, %d, %d) a_mn=%d b_mn=%d split=%d %s" % (tag, kind, M, N, K, a_mn, b_mn, sp, name)
                assert margins_intact(buf, M, N, fill), (what, "margin written")
                check_local(view, ref, BF16_TOL if is_bf16 else F32_TOL, BF16_LOCAL if is_bf16 else F32_LOCAL, worst, what)


@pytest.fixture()
def KN():
    from multimae_b200 import kernels
    return kernels


# Small shapes for the variant x epilogue x budget product; at budget 1 one CTA (cluster) runs all of their items
SMALL = [pytest.param((40, 776, 200), id="M<64-partial_box-raggedK"),
         pytest.param((648, 136, 320), id="odd_128row_tiles-N%BN-5kb"),
         pytest.param((1000, 1024, 64), id="1kb_per_item-many_items")]


@pytest.mark.parametrize("shape", SMALL)
@pytest.mark.parametrize("budget", [FULL, 1])
@pytest.mark.parametrize("variant", [0, 1, 2, 3, 4, 5, 6])
def test_epilogues_every_variant(dev, knobs, KN, variant, budget, shape):
    """Every epilogue kind, through the TMA-store and the register paths, at every explicit tile variant."""
    worst = Worst()
    M, N, K = shape
    for tma in (1, 0):
        knobs(budget=budget, variant=variant, tma_store=tma)
        run_gemm_case(KN, dev, M, N, K, EPILOGUES, worst, tag="v%d b%d tma%d" % (variant, budget, tma))
    worst.report("variant %d budget %d %s" % (variant, budget, shape))


@pytest.mark.parametrize("budget", [FULL, 1])
@pytest.mark.parametrize("variant", [0, 1, 2, 3, 4, 5, 6])
def test_ring_depth_every_variant(dev, knobs, KN, variant, budget):
    """Items of STAGES - 1, STAGES and STAGES + 1 k-blocks of the variant's ring: with fewer k-blocks than stages the
    producer runs whole items ahead of the consumers, and the ring's slot / phase wrap inside or between items."""
    worst = Worst()
    stages = VARIANT_TILE[variant][1]
    knobs(budget=budget, variant=variant)
    for kb in (stages - 1, stages, stages + 1):
        run_gemm_case(KN, dev, 520, 776, 64 * kb, ["bias_bf16", "f32", "accumulate"], worst, tag="v%d b%d" % (variant, budget))
    worst.report("ring variant %d budget %d" % (variant, budget))


# (M, N, K, split): the shape table at the heuristic's choice of tile and split
SHAPES = [pytest.param((1000, 1024, 64, 1), id="1kb-many_items"),
          pytest.param((4096, 768, 8, 1), id="K8-one_ragged_kb"),
          pytest.param((1000, 776, 200, 1), id="raggedK-partial_box"),
          pytest.param((1536, 2304, 192, 1), id="3kb"),
          pytest.param((1536, 2304, 256, 1), id="4kb"),
          pytest.param((1536, 2304, 320, 1), id="5kb"),
          pytest.param((1536, 1024, 384, 1), id="6kb"),
          pytest.param((1536, 1024, 448, 1), id="7kb"),
          pytest.param((1536, 1024, 576, 1), id="9kb"),
          pytest.param((648, 1024, 512, 1), id="M=5x128+8"),
          pytest.param((8, 768, 256, 1), id="M=8"),
          pytest.param((40, 2304, 768, 1), id="M=40"),
          pytest.param((1000, 8, 256, 1), id="N=8"),
          pytest.param((1000, 24, 512, 1), id="N=24"),
          pytest.param((1000, 776, 512, 1), id="N=776"),
          pytest.param((768, 768, 12672, 3), id="longK-split3"),
          pytest.param((768, 768, 12672, 0), id="longK-split_auto")]


@pytest.mark.parametrize("budget", [FULL, 1, 3, 17])
@pytest.mark.parametrize("shape", SHAPES)
def test_shape_table_heuristic(dev, knobs, KN, shape, budget):
    worst = Worst()
    M, N, K, split = shape
    knobs(budget=budget, variant=-1)
    kinds = ["f32", "split_bias", "split_bias_residual"] if split != 1 else ["bias_gelu_bf16", "residual", "accumulate"]
    run_gemm_case(KN, dev, M, N, K, kinds, worst, split=split, tag="b%d" % budget)
    worst.report("shape %s budget %d" % (shape, budget))


@pytest.mark.parametrize("variant", [0, 1, 2, 3, 4, 5, 6])
def test_bitwise_same_across_budgets_and_launches(dev, knobs, KN, variant):
    """With a fixed tile and split_k = 1 one CTA sums each tile in a fixed k order: the output bits may not depend on the
    SM budget (grid size, items per CTA) or on the launch."""
    torch.manual_seed(variant)
    for (M, N, K) in [(1000, 776, 200), (648, 1024, 512)]:
        A, B = bf16_randn(M, K, scale=0.5, dev=dev), bf16_randn(N, K, scale=0.5, dev=dev)
        bias = torch.randn(N, device=dev)
        for a_mn, b_mn in MAJORS:
            Aop, Bop = operand(A, a_mn), operand(B, b_mn)
            first = None
            for budget in (FULL, FULL, 1, 3, 17):
                knobs(budget=budget, variant=variant)
                o32 = torch.empty(M, N, device=dev)
                o16 = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
                KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, out_f32=o32)
                KN.gemm(Aop, Bop, a_mn=a_mn, b_mn=b_mn, bias=bias, act=1, out_bf16=o16)
                if first is None:
                    first = (o32, o16)
                    assert float((o32.double() - A.double() @ B.double().t()).norm()) < F32_TOL * float(o32.norm())
                else:
                    assert torch.equal(o32, first[0]) and torch.equal(o16, first[1]), (variant, M, N, K, a_mn, b_mn, budget)


# ------------------------------------------------------------------------------------- the heuristic at the real shapes
def _dump(lib):
    import ctypes
    buf = ctypes.create_string_buffer(1 << 20)
    n = lib.mmae_profile_gemm_dump(buf, len(buf))
    rows = []
    for line in buf.raw[:max(n, 0)].decode().splitlines():
        M, N, K, fl, _ = line.split()
        rows.append((int(M), int(N), int(K), int(fl) & 1, (int(fl) >> 1) & 1, int(fl) >> 8))
    return rows


def test_heuristic_at_model_shapes(dev, knobs, KN):
    """Every distinct GEMM launch of one eager MultiMAE-B step (BASELINE config 2 at the bench batch: 224^2, 98 visible
    tokens, B = 128), re-run on its own with the automatic split and tile into a zeroed fp32 destination at budgets full,
    120 (a data-parallel run's) and 1, against float64.  At full budget the weight-gradient GEMMs (both operands MN-major)
    must take the split-K path; at budget 1 there is nothing to fill and every launch must run unsplit."""
    from multimae_b200 import _lib as L
    from oracle import multimae_oracle as O
    from test_cuda_parity import _run_cuda_step
    from test_host_api import _build
    lib = L.lib()
    B, image, visible = 128, 224, 98
    torch.manual_seed(0)
    model = _build(("rgb", "depth", "semseg"), 768, 12, 12, 256, 2, 8, image).to(dev).train()
    cfg = O.make_config(size="base")
    cfg.posemb_grid = image // 16
    x = O.synthetic_inputs(cfg, B, image, seed=0)
    shares, noises, noise_all = O.synthetic_mask_draws(cfg, B, image, seed=1)
    m, ids_keep, ids_restore = O.sample_masks(shares, noises, noise_all, visible)
    triple = ({d.name: mm.to(dev) for d, mm in zip(cfg.in_domains, m)}, ids_keep.to(dev), ids_restore.to(dev))
    lib.mmae_profile_gemm(1)
    try:
        _run_cuda_step(model, x, triple, dev)
    finally:
        lib.mmae_profile_gemm(0)
    shapes = sorted({r[:5] for r in _dump(lib)})
    del model, x, triple
    torch.cuda.empty_cache()
    assert any(a and b for (_, _, _, a, b) in shapes), shapes
    print("%d distinct GEMM shapes in one step" % len(shapes))

    worst = Worst()
    splits = {}
    for budget in (FULL, 120, 1):
        knobs(budget=budget, variant=-1)
        lib.mmae_profile_gemm(1)
        try:
            for (M, N, K, a_mn, b_mn) in shapes:
                run_gemm_case(KN, dev, M, N, K, ["f32"], worst, split=0, majors=[(bool(a_mn), bool(b_mn))],
                              tag="b%d" % budget)
        finally:
            lib.mmae_profile_gemm(0)
        got = _dump(lib)
        assert len(got) == len(shapes)
        for shape, r in zip(shapes, got):
            assert r[:5] == shape
            splits[budget, shape] = r[5]
    worst.report("model shapes")
    for shape in shapes:
        print(shape, "split at budgets full / 120 / 1:", [splits[b, shape] for b in (FULL, 120, 1)])
    wgrad = [s for s in shapes if s[3] and s[4]]
    assert all(splits[FULL, s] > 1 for s in wgrad), [(s, splits[FULL, s]) for s in wgrad]
    assert all(splits[1, s] == 1 for s in shapes), [(s, splits[1, s]) for s in shapes if splits[1, s] != 1]


# --------------------------------------------------------------------------- column reductions and LayerNorm backward
ROWS = [1, 31, 32, 33, 1000, 12672, 25088]
BUDGETS = [FULL, 1, 7]


def rel(a, ref):
    return float((a.double() - ref).norm() / ref.norm().clamp_min(1e-300))


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("M", ROWS)
def test_layernorm_backward_ex(dev, knobs, M, budget):
    """mmae_layernorm_backward_ex: bf16 dy, dx_resid, the bf16 copy of dx and its column sums, strided leading dimensions;
    dgamma / dbeta / colsum accumulate onto non-zero values."""
    from multimae_b200 import _lib as L
    knobs(budget=budget)
    worst = Worst()
    for D in (256, 768):
        torch.manual_seed(M + D)
        xb, x = canvas(M, D, torch.float32, 4, 0.0, dev)
        x.copy_(torch.randn(M, D, device=dev) * 2 + 0.5)
        dyb, dy = canvas(M, D, torch.bfloat16, 56, 0.0, dev)
        dy.copy_(torch.randn(M, D, device=dev))
        rb, res = canvas(M, D, torch.float32, 8, 0.0, dev)
        res.copy_(torch.randn(M, D, device=dev))
        gamma = torch.randn(D, device=dev)
        x64 = x.double()
        mu = x64.mean(1, keepdim=True)
        rstd = (x64.var(1, unbiased=False, keepdim=True) + 1e-6).rsqrt()
        mean32, rstd32 = mu.float().flatten().contiguous(), rstd.float().flatten().contiguous()
        mu, rstd = mean32.double()[:, None], rstd32.double()[:, None]
        xh = (x64 - mu) * rstd
        g = dy.double() * gamma.double()
        dx_ref = rstd * (g - g.mean(1, keepdim=True) - xh * (g * xh).mean(1, keepdim=True)) + res.double()
        c0 = [torch.randn(D, device=dev) * 0.5 for _ in range(3)]
        dgam, dbet, cs = [c.clone() for c in c0]
        dxb, dx = canvas(M, D, torch.float32, 12, 9.0, dev)
        dx16b, dx16 = canvas(M, D, torch.bfloat16, 16, 9.0, dev)
        L.check(L.lib().mmae_layernorm_backward_ex(dy.data_ptr(), 1, dy.stride(0), x.data_ptr(), x.stride(0), mean32.data_ptr(),
                                                   rstd32.data_ptr(), gamma.data_ptr(), res.data_ptr(), res.stride(0),
                                                   dx.data_ptr(), dx.stride(0), dgam.data_ptr(), dbet.data_ptr(),
                                                   dx16.data_ptr(), dx16.stride(0), cs.data_ptr(), M, D, L.current_stream()))
        what = "M=%d D=%d budget %d" % (M, D, budget)
        assert margins_intact(dxb, M, D, 9.0) and margins_intact(dx16b, M, D, 9.0), what
        check_local(dx, dx_ref, 1e-5, F32_LOCAL, worst, what + " dx")
        check_local(dx16, dx_ref, BF16_TOL, BF16_LOCAL, worst, what + " dx_bf16")
        for got, c, ref, name in ((dgam, c0[0], (dy.double() * xh).sum(0), "dgamma"), (dbet, c0[1], dy.double().sum(0), "dbeta"),
                                  (cs, c0[2], dx_ref.sum(0), "dx_colsum")):
            assert rel(got, c.double() + ref) < SUM_TOL, (what, name, rel(got, c.double() + ref))
    worst.report("layernorm_backward_ex M=%d budget %d" % (M, budget))


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("M", ROWS)
def test_add_layernorm_forward(dev, knobs, M, budget):
    """x_sum = x + bf16 addend (written when given), then LayerNorm(x_sum) -> bf16, mean, rstd."""
    from multimae_b200 import _lib as L
    knobs(budget=budget)
    worst = Worst()
    D = 768
    torch.manual_seed(M)
    xb, x = canvas(M, D, torch.float32, 4, 0.0, dev)
    x.copy_(torch.randn(M, D, device=dev) * 2 + 0.5)
    ab, a = canvas(M, D, torch.bfloat16, 8, 0.0, dev)
    a.copy_(torch.randn(M, D, device=dev))
    gamma, beta = torch.randn(D, device=dev), torch.randn(D, device=dev)
    xs = x.double() + a.double()
    mu = xs.mean(1)
    rs = (xs.var(1, unbiased=False) + 1e-6).rsqrt()
    y_ref = (xs - mu[:, None]) * rs[:, None] * gamma.double() + beta.double()
    for with_sum in (True, False):
        sb, xsum = canvas(M, D, torch.float32, 12, 9.0, dev)
        yb, y = canvas(M, D, torch.bfloat16, 16, 9.0, dev)
        mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
        L.check(L.lib().mmae_add_layernorm_forward(x.data_ptr(), x.stride(0), a.data_ptr(), a.stride(0),
                                                   xsum.data_ptr() if with_sum else None, xsum.stride(0), gamma.data_ptr(),
                                                   beta.data_ptr(), y.data_ptr(), y.stride(0), mean.data_ptr(), rstd.data_ptr(),
                                                   M, D, 1e-6, L.current_stream()))
        what = "M=%d budget %d x_sum %s" % (M, budget, with_sum)
        assert margins_intact(yb, M, D, 9.0) and margins_intact(sb, M, D, 9.0), what
        if with_sum:
            assert rel(xsum, xs) < 1e-7, (what, rel(xsum, xs))
        else:
            assert bool((xsum == 9.0).all()), what
        check_local(y, y_ref, BF16_TOL, BF16_LOCAL, worst, what)
        assert rel(mean, mu) < 1e-5 and rel(rstd, rs) < 1e-5, (what, rel(mean, mu), rel(rstd, rs))
    worst.report("add_layernorm_forward M=%d budget %d" % (M, budget))


@pytest.mark.parametrize("budget", BUDGETS)
@pytest.mark.parametrize("M", ROWS)
def test_column_sums(dev, knobs, M, budget):
    """mmae_colsum_bf16 on its wide path (8 columns per thread) and its 128-column path (N % 8 != 0, or ld % 8 != 0),
    mmae_cast_colsum_f32 with and without the bf16 copy, and mmae_dgelu_colsum_bf16, each onto non-zero column sums.
    Budget and M set the row blocking: one row block (direct add), or many folded by the last block to finish."""
    from multimae_b200 import _lib as L
    lib, st = L.lib(), L.current_stream()
    knobs(budget=budget)
    torch.manual_seed(M)
    worst = Worst()
    for N, right in ((776, 8), (772, 12), (768, 4)):      # wide; N % 8 != 0; ld % 8 != 0
        sb, src = canvas(M, N, torch.bfloat16, right, 0.0, dev)
        src.copy_(torch.randn(M, N, device=dev))
        c0 = torch.randn(N, device=dev)
        cs = c0.clone()
        L.check(lib.mmae_colsum_bf16(src.data_ptr(), src.stride(0), cs.data_ptr(), M, N, st))
        ref = c0.double() + src.double().sum(0)
        assert rel(cs, ref) < SUM_TOL, ("colsum_bf16", M, N, src.stride(0), rel(cs, ref))

    N = 776
    fb, f = canvas(M, N, torch.float32, 4, 0.0, dev)
    f.copy_(torch.randn(M, N, device=dev))
    for with_dst in (True, False):
        c0 = torch.randn(N, device=dev)
        cs = c0.clone()
        db, dst = canvas(M, N, torch.bfloat16, 16, 9.0, dev)
        L.check(lib.mmae_cast_colsum_f32(f.data_ptr(), f.stride(0), dst.data_ptr() if with_dst else None, dst.stride(0),
                                         cs.data_ptr(), M, N, st))
        ref = c0.double() + f.double().sum(0)
        assert rel(cs, ref) < SUM_TOL, ("cast_colsum_f32", M, with_dst, rel(cs, ref))
        assert margins_intact(db, M, N, 9.0)
        if with_dst:
            assert torch.equal(dst, f.to(torch.bfloat16)), ("cast_colsum_f32 copy", M)
        else:
            assert bool((dst == 9.0).all())

    for N in (776, 3072):
        zb, z = canvas(M, N, torch.bfloat16, 8, 0.0, dev)        # z and dz share the leading dimension
        z.copy_(torch.randn(M, N, device=dev) * 1.5)
        dzb, dz = canvas(M, N, torch.bfloat16, 8, 9.0, dev)
        dz.copy_(torch.randn(M, N, device=dev))
        ref_dz = dz.double() * dgelu64(z.double())
        c0 = torch.randn(N, device=dev)
        cs = c0.clone()
        L.check(lib.mmae_dgelu_colsum_bf16(z.data_ptr(), dz.data_ptr(), dz.stride(0), cs.data_ptr(), M, N, st))
        what = "dgelu_colsum M=%d N=%d budget %d" % (M, N, budget)
        assert margins_intact(dzb, M, N, 9.0), what
        check_local(dz, ref_dz, BF16_TOL, BF16_LOCAL, worst, what)
        ref = c0.double() + dz.double().sum(0)                     # the sum of the stored (bf16-rounded) gradient
        assert rel(cs, ref) < SUM_TOL, (what, rel(cs, ref))
    worst.report("column sums M=%d budget %d" % (M, budget))
