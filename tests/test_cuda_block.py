"""GPU: the transformer-block entry points through the C ABI, as functional.BlockFunction calls them, against float64.

1. mmae_block_forward / mmae_block_backward (bf16 tier) against block_oracle.block_reference, which rounds to bf16
   wherever the kernels store bf16 (values and gradient operands, both GELU modes of mmae_set_fuse_gelu) and forms each
   bias gradient's column sum before or after the rounding exactly as the kernels do.  What it does NOT mirror:
     * attention's bf16 P (forward, and P / dS in backward): one bf16 rounding, relative u = 2^-8, per element;
     * __expf, fp32 accumulation order (GEMM k-loop, split-K, column sums), LayerNorm's fp32 arithmetic, the GELU
       approximation, the fp32 residual sums x_mid / x_out: < 1e-6 relative.
   A difference before a bf16 store can move the stored value to its neighbour: one ulp = 2u.  Forward: u (P) + 2u (o
   re-rounded) + the later stores' flips -> 4u (FWD_ROW), as for the decoder head in test_cuda_pretrain_io.py.  Backward
   adds P / dS (2u) and the re-rounding of dq / dk / dv (2u) -> 8u (GRAD_ROW).  Checked on their own, each as a relative
   L2 error:
     * the branch outputs x_mid - x_in (read through mmae_block_saved_x_mid) and x_out - x_mid, per token row - not the
       residual stream, whose size would hide a branch's error;
     * dx_in - dx_out (the gradient through both branches) per token row;
     * each weight gradient per output row and as a whole, qkv_w / qkv_b also per (q|k|v, head) slice of 64 (or 32) rows;
     * each bias and LayerNorm gradient as a whole.  The key part of qkv_b's gradient, colsum(dk), is 0 in exact
       arithmetic (softmax is invariant to a common shift of a query's scores), so a relative check of its slices means
       nothing: each of its elements is held to 8u of the sum of its terms' magnitudes instead.
   Every gradient buffer starts at non-zero values and the check is on grad - prior.  `saved` is filled with NaN bytes
   before forward, `ws` and every output before each call: a read of anything never written shows up as NaN.
   Per-sample drop-path factors 0, 1, 1/(1-0.1) and 2.5 on both branches; a sample with both factors 0 must pass x and
   its gradient through bitwise.
   Sensitivity: references with the neighbouring sample's keys, q of head h against k / v of head h+1, or the
   neighbouring sample's factors must miss by >= 10x the budget.
2. Three blocks chained as BlockFunction chains them (y_out -> x_add with s_prev; dx_in_bf16 / dx_in_colsum -> the next
   call's dx_out_bf16 and the previous block's fc2_b gradient).  Each block against block_reference on the inputs it was
   handed (x_in + s_prev x_add, dx_out) with the budgets of 1; the whole stack against the float64 three-block stack,
   where an error of a lower block's output reaches the branches above it at about the same relative size: forward of
   block i within (i + 1) x FWD_ROW, gradients within 3 x GRAD_ROW; and against the same blocks run unchained.  Both
   forms compute x + s * y as one fma (the LayerNorm kernel's `v += sc * a`, add_scaled_f32's `a + s * y`) and cast
   s * dx from the same fp32 value, so activations, dx_in and every
   gradient but the hand-off ones are held bitwise (weight gradients: see 3).  The hand-off fc2_b gradient of the lower
   blocks differs only in the order of its column sum: within 1e-6 of the sum of its terms' magnitudes per element.
   References with that column sum counted twice or left out must miss by >= 10x.
3. Switches, each restored to the library default after the test: the weight-gradient side stream (MMAE_WGRAD_STREAM)
   and the weight mirror (none; one registered flat buffer; one weight at a 4-float offset, which takes the cast
   fallback) against the plain run; two launches against each other.  Everything is compared bitwise except the weight
   gradients: their GEMMs may split K and add the splits onto the gradient with fp32 atomics in arrival order, so they
   are held to 1e-6 per row (fp32 reassociation).  MMAE_ATTN_TC = 7 (wgmma attention forward and backward) against the
   reference with the budgets of 1.
4. The fp32 tier (mmae_block_f32_*, mmae_dechead_f32_*, mmae_dectail_f32_*) against plain float64 (round=False).  Every
   Linear is the 3 x bf16 split GEMM of fp32_ops.cu, whose error per product is at most the two operand split residuals
   and the dropped lo x lo term, each <= v = 2^-16 relative: 3v per Linear.  Attention, GELU and LayerNorm in fp32 add
   < 1e-6.  The errors of the Linears on one path add: block forward 4 Linears (qkv, proj, fc1, fc2) -> 12v, its
   gradients 8 (the 4 forward and at most 4 dgrad / wgrad) -> 24v; decoder head forward 5 on the longest path
   (proj_context, kv, proj, fc1, fc2) -> 15v, gradients 10 -> 30v; decoder tail 1 -> 3v.  All per row, and as a whole."""
import ctypes
import os

import pytest
import torch

import block_oracle as BO
import pretrain_io_oracle as R
from multimae_b200 import _lib as L
from test_cuda_pretrain_io import DD, DE, HEAD_CASES, HEAD_VEC, HEAD_W, HEADS, HIDDEN, _Head, _head_inputs, _rel_rows, \
    _report

pytestmark = pytest.mark.gpu

U = 2.0 ** -8                      # bf16 unit roundoff
FWD_ROW = 4 * U                    # branch outputs, per token row and whole tensor
GRAD_ROW = 8 * U                   # gradients, per row / slice and whole tensor
V = 2.0 ** -16                     # split error of the fp32 tier's 3 x bf16 GEMM
BLOCK32_FWD, BLOCK32_GRAD = 12 * V, 24 * V
HEAD32_FWD, HEAD32_GRAD = 15 * V, 30 * V
TAIL32 = 3 * V
REASSOC = 1e-6                     # fp32 reassociation only
EPS = 1e-6
FACTORS = [0.0, 1.0, 1.0 / (1.0 - 0.1), 2.5]

SHAPES = {                         # B, N, D, H, hidden
    "enc_cfg2": (128, 99, 768, 12, 3072),
    "enc_cfg4": (64, 99, 1024, 16, 4096),
    "enc_cfg5": (32, 393, 768, 12, 3072),       # > 256 keys: delta + dQ + dK/dV backward
    "dec_cfg2": (128, 196, 256, 8, 1024),
    "dec_cfg5": (32, 784, 256, 8, 1024),
    "ft_cls": (32, 197, 768, 12, 3072),
    "ft_512": (4, 1025, 768, 12, 3072),
    "segmenter": (4, 1175, 768, 12, 3072),      # 1024 patches + 151 class tokens
    "n256": (8, 256, 768, 12, 3072),            # the fused attention backward's last size ...
    "n257": (8, 257, 768, 12, 3072),            # ... and the first past it
    "n1": (4, 1, 768, 12, 3072),
    "n7_b3": (3, 7, 768, 12, 3072),
    "n7_b3_dec": (3, 7, 256, 8, 1024),
}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(params=[0, 1], ids=["gelu_stream", "gelu_fused"])
def fuse_gelu(request):
    lib = L.lib()
    L.check(lib.mmae_set_fuse_gelu(request.param), "mmae_set_fuse_gelu")
    yield request.param
    lib.mmae_set_fuse_gelu(int(os.environ.get("MMAE_FUSE_GELU", "0")))      # the library's default


@pytest.fixture
def wgrad_stream():
    """set(on) switches the weight-gradient side stream; the library default is back after the test"""
    lib = L.lib()
    yield lambda on: L.check(lib.mmae_set_wgrad_stream(int(on)), "mmae_set_wgrad_stream")
    lib.mmae_set_wgrad_stream(int(os.environ.get("MMAE_WGRAD_STREAM", "0")))


@pytest.fixture
def attn_tc():
    lib = L.lib()
    yield lambda mask: L.check(lib.mmae_attention_set_tc(mask), "mmae_attention_set_tc")
    lib.mmae_attention_set_tc(-1)                                             # the start-up default


@pytest.fixture
def mirrors():
    """register(f32, bf16) registers a weight mirror; every one is unregistered (n = 0) after the test"""
    lib, done = L.lib(), []

    def register(f32, b16):
        L.check(lib.mmae_weight_mirror_register(f32.data_ptr(), b16.data_ptr(), f32.numel()), "mirror register")
        done.append(f32)
    yield register
    for f32 in done:
        lib.mmae_weight_mirror_register(f32.data_ptr(), None, 0)


# ------------------------------------------------------------------------------------------------------------ inputs
def _params(D, hid, gen, dev):
    """float64 parameters (fp32 values) scaled so that each branch is about as large as the residual stream: weights by
    1/sqrt(fan-in), q / k rows by a further 1.5 so that attention is peaked and depends on which key is which"""
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    qkv = r(3 * D, D) / D ** 0.5
    qkv[:2 * D] *= 1.5
    p = {"norm1_w": 1 + 0.1 * r(D), "norm1_b": 0.1 * r(D), "qkv_w": qkv, "qkv_b": 0.1 * r(3 * D),
         "proj_w": r(D, D) / D ** 0.5, "proj_b": 0.1 * r(D), "norm2_w": 1 + 0.1 * r(D), "norm2_b": 0.1 * r(D),
         "fc1_w": r(hid, D) / D ** 0.5, "fc1_b": 0.1 * r(hid), "fc2_w": r(D, hid) / hid ** 0.5, "fc2_b": 0.1 * r(D)}
    return {k: v.float().double().to(dev) for k, v in p.items()}


def _randn(shape, gen, dev):
    return torch.randn(*shape, generator=gen, dtype=torch.float64).float().double().to(dev)


def _factors(B, dev, shift=0):
    """(s_attn, s_mlp) float64 [B]: 0, 1, 1/(1-0.1), 2.5 on each branch; sample `shift` has both 0, and from B = 8 on
    some samples drop one branch only"""
    sa = [FACTORS[(i - shift) % 4] for i in range(B)]
    sm = [FACTORS[((i - shift) + (i - shift) // 4) % 4] for i in range(B)]
    return (torch.tensor(sa, dtype=torch.float64, device=dev), torch.tensor(sm, dtype=torch.float64, device=dev))


def _nan(shape, dev, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


class _Blk:
    """fp32 device copies of one block's parameters and gradient slots (starting at `prior`), its saved / ws buffers,
    and the ctypes calls of one tier."""

    def __init__(self, prm, prior, shape, dev, f32=False, p32=None):
        self.dims = shape
        self.f32 = f32
        self.p32 = p32 or {k: v.float().contiguous() for k, v in prm.items()}
        self.prior = prior
        self.g32 = {k: v.float().contiguous() for k, v in prior.items()}
        self.prm = L.BlockParams(*[self.p32[k].data_ptr() for k in BO.PARAMS])
        self.grd = L.BlockGrads(*[self.g32[k].data_ptr() for k in BO.PARAMS])
        lib, tier = L.lib(), "_f32" if f32 else ""
        self.saved = torch.empty(getattr(lib, "mmae_block%s_saved_bytes" % tier)(*shape), dtype=torch.uint8, device=dev)
        self.ws = torch.empty(getattr(lib, "mmae_block%s_workspace_bytes" % tier)(*shape), dtype=torch.uint8, device=dev)
        self.dev = dev

    def reset_grads(self):
        for k, v in self.prior.items():
            self.g32[k].copy_(v)

    def grads(self):
        return {k: self.g32[k].double() - self.prior[k] for k in BO.PARAMS}

    def x_mid(self):
        B, N, D = self.dims[:3]
        off = L.lib().mmae_block_saved_x_mid(self.saved.data_ptr(), *self.dims) - self.saved.data_ptr()
        return self.saved[off:off + 4 * B * N * D].view(torch.float32).view(B, N, D)

    def forward(self, x_in, s=(None, None), x_add=None, s_prev=None, chained=False):
        """returns (x_sum or None, x_out or None, y_out or None)"""
        B, N, D, H, hid = self.dims
        self.saved.fill_(0xFF)
        self.ws.fill_(0xFF)
        st = L.current_stream()
        if self.f32:
            x_out = _nan((B, N, D), self.dev)
            L.check(L.lib().mmae_block_f32_forward(x_in.data_ptr(), x_out.data_ptr(), B, N, D, H, hid, EPS, L.ptr(s[0]),
                                                   L.ptr(s[1]), ctypes.byref(self.prm), self.saved.data_ptr(),
                                                   self.ws.data_ptr(), st), "mmae_block_f32_forward")
            return None, x_out, None
        x_sum = _nan((B, N, D), self.dev) if x_add is not None else None
        x_out = None if chained else _nan((B, N, D), self.dev)
        y_out = _nan((B, N, D), self.dev, torch.bfloat16) if chained else None
        L.check(L.lib().mmae_block_forward(x_in.data_ptr(), L.ptr(x_add), L.ptr(x_sum), L.ptr(x_out), L.ptr(y_out), B, N, D,
                                           H, hid, EPS, L.ptr(s[0]), L.ptr(s[1]), L.ptr(s_prev), None,
                                           ctypes.byref(self.prm), self.saved.data_ptr(), self.ws.data_ptr(), st),
                "mmae_block_forward")
        return x_sum, x_out, y_out

    def backward(self, x_in, dx_out, s=(None, None), dx_out_b=None, handoff=None, s_prev=None):
        """handoff: the previous block's fc2_b gradient slot (chained); returns (dx_in, dx_in_bf16 or None)"""
        B, N, D, H, hid = self.dims
        self.ws.fill_(0xFF)
        st = L.current_stream()
        dx_in = _nan((B, N, D), self.dev)
        if self.f32:
            L.check(L.lib().mmae_block_f32_backward(x_in.data_ptr(), dx_out.data_ptr(), dx_in.data_ptr(), B, N, D, H, hid,
                                                    L.ptr(s[0]), L.ptr(s[1]), ctypes.byref(self.prm),
                                                    ctypes.byref(self.grd), self.saved.data_ptr(), self.ws.data_ptr(), st),
                    "mmae_block_f32_backward")
            return dx_in, None
        dx_in_b = _nan((B, N, D), self.dev, torch.bfloat16) if handoff is not None else None
        L.check(L.lib().mmae_block_backward(x_in.data_ptr(), dx_out.data_ptr(), L.ptr(dx_out_b), dx_in.data_ptr(),
                                            L.ptr(dx_in_b), L.ptr(handoff), B, N, D, H, hid, L.ptr(s[0]), L.ptr(s[1]),
                                            L.ptr(s_prev), None, ctypes.byref(self.prm), ctypes.byref(self.grd),
                                            self.saved.data_ptr(), self.ws.data_ptr(), st), "mmae_block_backward")
        return dx_in, dx_in_b


def _f32(t):
    return None if t is None else t.float().contiguous()


def _case(name, dev, seed=41, with_factors=True):
    B, N, D, H, hid = SHAPES[name]
    gen = torch.Generator().manual_seed(seed)
    prm = _params(D, hid, gen, dev)
    prior = {k: _randn(v.shape, gen, dev) for k, v in prm.items()}
    x = _randn((B, N, D), gen, dev)
    dout = _randn((B, N, D), gen, dev)
    sc = _factors(B, dev) if with_factors else (None, None)
    return prm, prior, x, dout, sc


# ------------------------------------------------------------------------------------------------------------ checks
ACT = ("attn", "mlp", "branches")


def _got(blk, x_in, x_mid, x_out, dx_in, dx_out):
    """the quantities that are checked, float64"""
    g = {"dbranch": dx_in.double() - dx_out.double()}
    if x_mid is None:
        g["branches"] = x_out.double() - x_in.double()
    else:
        g["attn"] = x_mid.double() - x_in.double()
        g["mlp"] = x_out.double() - x_mid.double()
    g.update(blk.grads())
    return g


def _view(ref, dout, keys):
    r = {"attn": ref["attn"], "mlp": ref["mlp"], "branches": ref["x_out"] - ref["x"], "dbranch": ref["dx_in"] - dout}
    r.update({k: ref[k] for k in BO.PARAMS})
    out = {k: r[k] for k in keys}
    out["dk_abs"] = ref["dk_abs"]
    return out


def _checks(got, ref, H, fwd, grad, N):
    """[(label, error, budget)]: everything as a whole; activations per token row, weight gradients per output row,
    qkv_w / qkv_b per (q|k|v, head) slice.  With one token per sample (N = 1) softmax is 1 whatever q and k are: their
    gradients are 0 in exact arithmetic and the kernels' are rounding noise, so the q and k rows are held only within
    the whole-tensor checks."""
    out = []
    for k, g in got.items():
        r = ref[k]
        if k == "dk_abs":
            continue
        whole, row = _rel_rows(g, r)
        b = fwd if k in ACT else grad
        out.append((k, whole, b))
        if k in ACT or k == "dbranch" or (k.endswith("_w") and g.dim() == 2):
            if k == "qkv_w" and N == 1:
                row = _rel_rows(g[2 * g.shape[1]:], r[2 * g.shape[1]:])[1]
            out.append((k + " row", row, b))
    for k in ("qkv_w", "qkv_b"):
        g, r = got[k].reshape(3, H, -1), ref[k].reshape(3, H, -1)
        if N == 1:
            g, r = g[2:], r[2:]
        elif k == "qkv_b":                     # q and v slices; the key slices are ~0, held to the size of their terms
            D = ref["dk_abs"].numel()
            err = (got[k][D:2 * D] - ref[k][D:2 * D]).abs() / ref["dk_abs"].clamp_min(1e-300)
            out.append(("qkv_b key part / sum|dk|", float(err.max()), grad))
            g, r = g[0::2], r[0::2]
        out.append((k + " head", _rel_rows(g.flatten(0, 1), r.flatten(0, 1))[1], grad))
    return out


def _assert_within(name, errs):
    frac = _report(name, errs)
    assert frac <= 1.0, [e for e in errs if e[1] > e[2]]


def _assert_dropped(x_in, x_out, dx_in, dx_out, sc):
    """a sample with both factors 0 passes its input and its gradient through bitwise"""
    if sc[0] is None:
        return
    both = ((sc[0] == 0) & (sc[1] == 0)).nonzero().flatten().tolist()
    assert both
    for b in both:
        assert torch.equal(x_out[b], x_in[b].float()), b
        assert torch.equal(dx_in[b], dx_out[b].float()), b


def _run_single(dev, name, fuse, with_factors=True, mutations=()):
    B, N, D, H, hid = SHAPES[name]
    prm, prior, x, dout, sc = _case(name, dev, with_factors=with_factors)
    blk = _Blk(prm, prior, SHAPES[name], dev)
    x32, d32, s32 = _f32(x), _f32(dout), (_f32(sc[0]), _f32(sc[1]))
    _, x_out, _ = blk.forward(x32, s32)
    dx_in, _ = blk.backward(x32, d32, s32)
    torch.cuda.synchronize()
    got = _got(blk, x32, blk.x_mid(), x_out, dx_in, d32)
    ref = BO.block_reference(x, prm, H, EPS, dout, bool(fuse), True, sc[0], sc[1])
    _assert_within("block %s fuse=%d" % (name, fuse), _checks(got, _view(ref, dout, got), H, FWD_ROW, GRAD_ROW, N))
    _assert_dropped(x32, x_out, dx_in, d32, sc)
    for m in mutations:
        wrong = BO.block_reference(x, prm, H, EPS, dout, bool(fuse), True, sc[0], sc[1], mutate=m)
        wf = max(e[1] / e[2] for e in _checks(got, _view(wrong, dout, got), H, FWD_ROW, GRAD_ROW, N))
        print("  wrong reference %s: %.1f x budget" % (m, wf))
        assert wf >= 10.0, (m, wf)


# ============================================================================================= 1. one block, bf16 tier
@pytest.mark.parametrize("name", [n for n in SHAPES if n != "n7_b3_dec"])
def test_block_against_rounding_reference(dev, fuse_gelu, name):
    muts = BO.MUTATIONS if name in ("enc_cfg2", "dec_cfg2") and fuse_gelu == 0 else ()
    _run_single(dev, name, fuse_gelu, mutations=muts)


def test_block_without_factors(dev):
    """null s_attn / s_mlp: factor 1, the kernels' plain residual adds"""
    _run_single(dev, "enc_cfg2", 0, with_factors=False)


# ============================================================================================================ 2. chain
def _chain_inputs(name, dev):
    B, N, D, H, hid = SHAPES[name]
    gen = torch.Generator().manual_seed(43)
    prms = [_params(D, hid, gen, dev) for _ in range(3)]
    priors = [{k: _randn(v.shape, gen, dev) for k, v in p.items()} for p in prms]
    x = _randn((B, N, D), gen, dev)
    dout = _randn((B, N, D), gen, dev)
    scales = [_factors(B, dev), _factors(B, dev, shift=1), None]
    return prms, priors, x, dout, scales


@pytest.mark.parametrize("name", ["enc_cfg2", "dec_cfg2", "n7_b3"])
def test_block_chain(dev, name):
    B, N, D, H, hid = SHAPES[name]
    prms, priors, x, dout, scales = _chain_inputs(name, dev)
    s32 = [(None, None) if s is None else (_f32(s[0]), _f32(s[1])) for s in scales]
    x32, d32 = _f32(x), _f32(dout)

    # chained, as BlockFunction runs a stack
    ch = [_Blk(p, q, SHAPES[name], dev) for p, q in zip(prms, priors)]
    xs, ys, x_ptr, add, s_prev = [], [], x32, None, None
    for i, b in enumerate(ch):
        x_sum, x_out, y = b.forward(x_ptr, s32[i], add, s_prev, chained=i < 2)
        xs.append(x_ptr if x_sum is None else x_sum)
        ys.append(y)
        if i < 2:
            x_ptr, add, s_prev = b.x_mid(), y, s32[i][1]
    c_out = x_out
    c_dx, d, g_in = [None] * 3, d32, None
    for i in reversed(range(3)):
        handoff = ch[i - 1].g32["fc2_b"] if i > 0 else None
        dx, g_out = ch[i].backward(xs[i], d, s32[i], g_in, handoff, s32[i - 1][1] if i > 0 else None)
        c_dx[i], d, g_in = dx, dx, g_out
    torch.cuda.synchronize()

    # the same blocks, one call each, nothing handed off
    un = [_Blk(p, q, SHAPES[name], dev) for p, q in zip(prms, priors)]
    u_in, h = [], x32
    for i, b in enumerate(un):
        u_in.append(h)
        _, h, _ = b.forward(h, s32[i])
    u_dx, d = [None] * 3, d32
    for i in reversed(range(3)):
        u_dx[i], _ = un[i].backward(u_in[i], d, s32[i])
        d = u_dx[i]
    torch.cuda.synchronize()
    assert torch.equal(c_out, h)
    for i in range(3):
        assert torch.equal(xs[i], u_in[i]) and torch.equal(ch[i].x_mid(), un[i].x_mid()), i
        assert torch.equal(c_dx[i], u_dx[i]), i
        for k in BO.PARAMS:
            a, b = ch[i].grads()[k], un[i].grads()[k]
            if k == "fc2_b" and i < 2:          # the hand-off column sum: same terms, another order
                terms = (u_dx[i + 1].double() * (1.0 if scales[i] is None else scales[i][1].reshape(-1, 1, 1))).abs()
                bound = REASSOC * (terms.sum((0, 1)) + priors[i][k].abs())
                assert bool(((a - b).abs() <= bound).all()), (i, float(((a - b).abs() / bound).max()))
            elif k.endswith("_w") and a.dim() == 2:
                assert _rel_rows(a, b)[1] <= REASSOC, (i, k, _rel_rows(a, b))
            else:
                assert torch.equal(a, b), (i, k)

    # against float64, each block on the inputs it was handed (x_mid and y_out of the block below, the dx_in of the block
    # above): the single-block budgets; the fc2_b gradient of the lower blocks is the hand-off column sum alone
    dxo = [c_dx[1], c_dx[2], d32]
    outs = [xs[1], xs[2], c_out]
    got = [_got(ch[i], xs[i], ch[i].x_mid(), outs[i], c_dx[i], dxo[i]) for i in range(3)]
    refs = []
    for i in range(3):
        s = scales[i] or (None, None)
        hand = {} if i == 0 else {"x_add": ys[i - 1].double(), "s_prev": None if scales[i - 1] is None else scales[i - 1][1]}
        x_in = x32 if i == 0 else ch[i - 1].x_mid()
        refs.append(_view(BO.block_reference(x_in.double(), prms[i], H, EPS, dxo[i].double(), s_attn=s[0], s_mlp=s[1],
                                             **hand), dxo[i].double(), got[i]))

    def checks(refs, fwd, grad):
        return [("block %d %s" % (i, e[0]), e[1], e[2])
                for i in range(3) for e in _checks(got[i], refs[i], H, fwd, grad, N)]

    _assert_within("chain %s, block by block" % name, checks(refs, FWD_ROW, GRAD_ROW))
    if name != "n7_b3":
        for m in ("handoff_twice", "handoff_missing"):
            wrong = [dict(r, fc2_b=r["fc2_b"] * (2 if m == "handoff_twice" else 0)) if i < 2 else r
                     for i, r in enumerate(refs)]
            wf = max(e[1] / e[2] for e in checks(wrong, FWD_ROW, GRAD_ROW))
            print("  wrong reference %s: %.1f x budget" % (m, wf))
            assert wf >= 10.0, (m, wf)
    # against the float64 stack: an error of a block's output carries into the input of every block above it, where,
    # with branches about as large as the residual stream, it is about as large relative to their branches.  Forward of
    # block i: the budgets of i + 1 blocks; gradients pass through every block's forward and the backward of the
    # blocks above: the budgets of 3.
    stack = BO.chain_reference(x, prms, H, EPS, dout, scales=scales)
    errs = []
    for i in range(3):
        r = _view(stack[i], stack[i + 1]["dx_in"] if i < 2 else dout, got[i])
        errs += [("block %d %s" % (i, e[0]), e[1], e[2])
                 for e in _checks(got[i], r, H, (i + 1) * FWD_ROW, 3 * GRAD_ROW, N)]
    _assert_within("chain %s, whole stack" % name, errs)


# ========================================================================================================= 3. switches
def _outputs(blk, x_out, dx_in):
    return {"x_out": x_out, "x_mid": blk.x_mid().clone(), "dx_in": dx_in, **{k: v.clone() for k, v in blk.g32.items()}}


def _assert_same(a, b, what):
    """bitwise, except weight gradients (split-K atomics): 1e-6 per row"""
    for k in a:
        if k.endswith("_w") and a[k].dim() == 2:
            assert _rel_rows(a[k], b[k].double())[1] <= REASSOC, (what, k)
        else:
            assert torch.equal(a[k], b[k]), (what, k, float((a[k].double() - b[k].double()).abs().max()))


def _fwd_bwd(blk, x32, d32, s32, backwards=1):
    _, x_out, _ = blk.forward(x32, s32)
    for _ in range(backwards):
        dx_in, _ = blk.backward(x32, d32, s32)
    torch.cuda.synchronize()
    return _outputs(blk, x_out, dx_in)


@pytest.mark.parametrize("name", ["enc_cfg2", "dec_cfg2"])
def test_wgrad_side_stream(dev, wgrad_stream, name):
    """the four weight-gradient GEMMs on the library's side stream: the same results; backward twice, so that the side
    stream and its events are reused"""
    prm, prior, x, dout, sc = _case(name, dev)
    x32, d32, s32 = _f32(x), _f32(dout), (_f32(sc[0]), _f32(sc[1]))
    runs = []
    for on in (0, 1):
        wgrad_stream(on)
        runs.append(_fwd_bwd(_Blk(prm, prior, SHAPES[name], dev), x32, d32, s32, backwards=2))
    _assert_same(runs[0], runs[1], "side stream")


@pytest.mark.parametrize("name", ["enc_cfg2", "dec_cfg2", "ft_cls", "n256", "enc_cfg5"])
def test_wgmma_attention_in_block(dev, attn_tc, name):
    attn_tc(7)
    _run_single(dev, name, 0)


@pytest.mark.parametrize("name", ["enc_cfg2", "dec_cfg2"])
def test_weight_mirror(dev, mirrors, name):
    """no mirror; a registered bf16 mirror of one flat buffer holding the four weights; the same with proj_w at a 4-float
    offset, whose mirror lookup falls back to the per-call cast.  All bitwise (weight gradients: see the docstring)."""
    B, N, D, H, hid = SHAPES[name]
    prm, prior, x, dout, sc = _case(name, dev)
    x32, d32, s32 = _f32(x), _f32(dout), (_f32(sc[0]), _f32(sc[1]))
    plain = _fwd_bwd(_Blk(prm, prior, SHAPES[name], dev), x32, d32, s32)
    W = ["qkv_w", "proj_w", "fc1_w", "fc2_w"]
    for pad in (0, 4):
        sizes = [prm[k].numel() for k in W]
        offs, o = [], 0
        for i, n in enumerate(sizes):
            o += pad if i in (1, 2) else 0      # proj_w at pad, fc1_w back on a multiple of 8
            offs.append(o)
            o += n
        flat = torch.zeros(o, dtype=torch.float32, device=dev)
        p32 = {k: v.float().contiguous() for k, v in prm.items()}
        for k, off, n in zip(W, offs, sizes):
            flat[off:off + n] = prm[k].flatten().float()
            p32[k] = flat[off:off + n].view(prm[k].shape)
        mirror = flat.to(torch.bfloat16)
        mirrors(flat, mirror)
        assert [off % 8 for off in offs] == ([0, 0, 0, 0] if pad == 0 else [0, 4, 0, 0])
        got = _fwd_bwd(_Blk(prm, prior, SHAPES[name], dev, p32=p32), x32, d32, s32)
        _assert_same(plain, got, "mirror pad %d" % pad)
        L.check(L.lib().mmae_weight_mirror_register(flat.data_ptr(), None, 0), "mirror unregister")


def test_repeatable(dev):
    name = "enc_cfg2"
    prm, prior, x, dout, sc = _case(name, dev)
    x32, d32, s32 = _f32(x), _f32(dout), (_f32(sc[0]), _f32(sc[1]))
    blk = _Blk(prm, prior, SHAPES[name], dev)
    fwd = []
    for _ in range(2):
        _, x_out, _ = blk.forward(x32, s32)
        torch.cuda.synchronize()
        fwd.append((x_out, blk.saved.clone()))
    assert torch.equal(fwd[0][0], fwd[1][0]) and torch.equal(fwd[0][1], fwd[1][1])
    bwd = []
    for _ in range(2):
        blk.reset_grads()
        dx_in, _ = blk.backward(x32, d32, s32)
        torch.cuda.synchronize()
        bwd.append(_outputs(blk, fwd[1][0], dx_in))
    _assert_same(bwd[0], bwd[1], "two launches")


# ========================================================================================================= 4. fp32 tier
@pytest.mark.parametrize("factors", [True, False], ids=["factors", "plain"])
@pytest.mark.parametrize("name", ["dec_cfg2", "dec_cfg5", "n7_b3_dec"])
def test_block_f32(dev, name, factors):
    B, N, D, H, hid = SHAPES[name]
    prm, prior, x, dout, sc = _case(name, dev, with_factors=factors)
    blk = _Blk(prm, prior, SHAPES[name], dev, f32=True)
    x32, d32, s32 = _f32(x), _f32(dout), (_f32(sc[0]), _f32(sc[1]))
    _, x_out, _ = blk.forward(x32, s32)
    dx_in, _ = blk.backward(x32, d32, s32)
    torch.cuda.synchronize()
    got = _got(blk, x32, None, x_out, dx_in, d32)
    ref = BO.block_reference(x, prm, H, EPS, dout, round=False, s_attn=sc[0], s_mlp=sc[1])
    _assert_within("block_f32 %s" % name, _checks(got, _view(ref, dout, got), H, BLOCK32_FWD, BLOCK32_GRAD, N))
    _assert_dropped(x32, x_out, dx_in, d32, sc)


@pytest.mark.parametrize("case", [c for c, v in HEAD_CASES.items() if v[5] is None])
def test_dechead_f32(dev, case):
    B, n, T, mode, own, _ = HEAD_CASES[case]
    gen = torch.Generator().manual_seed(22)
    prm, ix = _head_inputs(B, n, T, mode, own, gen, dev, False)
    Nc = T + 1
    h = _Head(prm, ix, B, DE, dev)
    for k, v in h.g32.items():                       # gradients accumulate onto non-zero values
        for t in (v if k == "task_emb" else [v]):
            t.copy_(torch.randn(t.shape, generator=gen))
    prior = {k: ([t.double() for t in v] if k == "task_emb" else v.double()) for k, v in h.g32.items()}
    lib, st = L.lib(), L.current_stream()
    saved = torch.full((lib.mmae_dechead_f32_saved_bytes(ctypes.byref(h.ix), DE, HEADS, HIDDEN),), 0xFF, dtype=torch.uint8,
                       device=dev)
    ws = torch.full((lib.mmae_dechead_f32_workspace_bytes(ctypes.byref(h.ix), DE, HEADS, HIDDEN),), 0xFF,
                    dtype=torch.uint8, device=dev)
    enc = torch.randn(B, Nc, DE, generator=gen).to(dev)
    denc = torch.randn(B, Nc, DE, generator=gen).to(dev)                   # accumulated onto
    denc0 = denc.double()
    dout = torch.randn(B, n, DD, generator=gen).to(dev)
    h.out.fill_(float("nan"))
    L.check(lib.mmae_dechead_f32_forward(enc.data_ptr(), DE, ctypes.byref(h.ix), HEADS, HIDDEN, 1e-6, ctypes.byref(h.prm),
                                         h.out.data_ptr(), saved.data_ptr(), ws.data_ptr(), st), "dechead_f32 forward")
    ws.fill_(0xFF)
    L.check(lib.mmae_dechead_f32_backward(enc.data_ptr(), DE, ctypes.byref(h.ix), HEADS, HIDDEN, ctypes.byref(h.prm),
                                          ctypes.byref(h.grd), dout.data_ptr(), denc.data_ptr(), saved.data_ptr(),
                                          ws.data_ptr(), st), "dechead_f32 backward")
    torch.cuda.synchronize()

    leaves = {k: ([t.clone().requires_grad_(True) for t in v] if k == "task_emb" else v.clone().requires_grad_(k != "pos"))
              for k, v in prm.items()}
    s = enc.double().requires_grad_(True)
    c = s @ leaves["proj_context_w"].t() + leaves["proj_context_b"]
    x_out, _ = R.dechead_reference(c, ix, leaves, HEADS, 1e-6, False, dout.double(), round=False)
    errs = []
    for k in ["x_out", "denc"] + HEAD_W + HEAD_VEC + ["mask_token", "proj_context_w", "proj_context_b", "task_emb"]:
        if k == "x_out":
            pairs = [(k, h.out, x_out)]
        elif k == "denc":
            pairs = [(k, denc.double() - denc0, s.grad)]
        elif k == "task_emb":
            used = set(range(3)) | ({own} if own >= 0 else set())
            pairs = [("task_emb.%d" % t, h.g32[k][t].double() - prior[k][t], leaves[k][t].grad) for t in sorted(used)]
        else:
            pairs = [(k, h.g32[k].double() - prior[k], leaves[k].grad)]
        for label, g, r in pairs:
            whole, row = _rel_rows(g, r)
            b = HEAD32_FWD if k == "x_out" else HEAD32_GRAD
            errs.append((label, whole, b))
            if g.dim() >= 2:
                errs.append((label + " row", row, b))
    _assert_within("dechead_f32 %s" % case, errs)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("S,B", [(224, 128), (448, 32)])
def test_dectail_f32(dev, S, B, C):
    lib = L.lib()
    gen = torch.Generator().manual_seed(23)
    Dd, P = 256, 16
    nh = nw = S // 16
    x = _randn((B, nh * nw, Dd), gen, dev)
    w = _randn((C * P * P, Dd), gen, dev) / Dd ** 0.5
    w = w.float().double()
    b = (0.1 * _randn((C * P * P,), gen, dev)).float().double()
    dpred = _randn((B, C, nh * P, nw * P), gen, dev)
    prior_w, prior_b = _randn(w.shape, gen, dev), _randn(b.shape, gen, dev)
    x32, w32, b32, dp32 = (_f32(t) for t in (x, w, b, dpred))
    gw, gb = _f32(prior_w), _f32(prior_b)
    dims = (B, nh, nw, Dd, C, P)
    ws = torch.full((lib.mmae_dectail_f32_workspace_bytes(*dims),), 0xFF, dtype=torch.uint8, device=dev)
    pred = _nan((B, C, nh * P, nw * P), dev)
    dx = _nan((B, nh * nw, Dd), dev)
    st = L.current_stream()
    L.check(lib.mmae_dectail_f32_forward(x32.data_ptr(), *dims, w32.data_ptr(), b32.data_ptr(), pred.data_ptr(),
                                         ws.data_ptr(), st), "dectail_f32 forward")
    ws.fill_(0xFF)
    L.check(lib.mmae_dectail_f32_backward(x32.data_ptr(), dp32.data_ptr(), *dims, w32.data_ptr(), gw.data_ptr(),
                                          gb.data_ptr(), dx.data_ptr(), ws.data_ptr(), st), "dectail_f32 backward")
    torch.cuda.synchronize()
    y = x @ w.t() + b                                                   # per token: C * P * P outputs
    dy = R.patchify(dpred, P)
    pairs = [("pred", R.patchify(pred.double(), P), y), ("dx", dx, dy @ w),
             ("dW", gw.double() - prior_w, dy.flatten(0, 1).t() @ x.flatten(0, 1)),
             ("db", gb.double() - prior_b, dy.sum((0, 1)))]
    errs = []
    for label, g, r in pairs:
        whole, row = _rel_rows(g, r)
        errs.append((label, whole, TAIL32))
        if g.dim() >= 2:
            errs.append((label + " row", row, TAIL32))
    _assert_within("dectail_f32 S=%d C=%d" % (S, C), errs)
