"""GPU: the fine-tuning heads' entry points through the C ABI - the ConvNeXt head (mmae_convnext_proj / block / tail_*) and
the classification head (mmae_clshead_*) - against the float64 references of convnext_head_oracle and cls_head_oracle.

1. Exact tier (ConvNeXt).  Dyadic inputs (k / 8, k / 16) chosen as in test_cuda_pretrain_io: every bf16 cast is exact and,
   where the premise is asserted on the reference (terms multiples of 2^-q, sums of their magnitudes below 2^(23-q)),
   every fp32 sum the kernels form is exact, so the comparison is torch.equal - asserted for proj (x_out, denc, d_w, d_b),
   the dwconv forward and the tail (out, dx, d_w, d_b; inputs sparse enough that the weight-gradient sums over every
   pixel stay exact).  Every upsample ratio r = 16 / s is a power
   of two, so the bilinear weights are multiples of 1 / (2r) (asserted).  The dwconv is checked on its own: its forward
   output is the `d` the block saves, its transposed backward and its weight / bias gradients are checked against the
   LayerNorm gradient `dd` the kernels leave in the workspace.  `dd` is not dyadic and a weight-gradient sum runs over
   every pixel, so where the premise does not hold the result is held element by element to the bound of any fp32
   summation order, n 2^-24 times the sum of the n terms' magnitudes (one rounding per addition): a wrong tap, halo pixel
   or row is off by a whole term.  Those checks print their worst error as a fraction of the bound; the rounding tier
   holds the same gradients per row.
2. Rounding tier.  Random inputs against the round=True references: float64 with a bf16 rounding wherever the kernels
   store bf16.  What they do NOT mirror: fp32 accumulation order, the LayerNorm's fp32 statistics, GELU's fp32 erf and
   the fused epilogue's arithmetic (< 1e-6 relative each).  Such a difference ahead of a bf16 store can move the stored
   value to its neighbour, one ulp = 2u (u = 2^-8) relative on that element, so each store that can flip adds 2u to a
   row's budget:
     * ConvNeXt block: h, z, a flip in the forward -> the branch x_out - x_in per pixel row, 4u (3 stores, rounded up as
       test_cuda_block's FWD_ROW); backward adds dgrad(fc2), dz and dh -> dx_in - dx_out per pixel row and every
       parameter gradient (per output row for the matrices and the 7x7 kernel, as a whole for the vectors), 8u.
     * ConvNeXt tail forward and proj forward: the only bf16 stores are casts of the caller's fp32 values, the same in
       the reference, so nothing can flip: fp32 summation alone.  The longest such sum is the proj's, T*D + 1 <= 2048
       terms (C <= 1024 for the tail, D <= 1024 for the classification head): n 2^-24 <= 2^-13 of the terms' magnitude,
       with a factor 4 for the cancellation of random signs -> 2^-11 = u/8 per (b, k, Y) output row, per (b, k) plane and
       per pixel row of the proj output.  Tail backward: bf16(dcmap) can flip -> dx per pixel row and d_w per class row
       2u; d_b is a column sum of the fp32 dcmap, u/8.
     * Classification head: the LayerNorm output xn is stored bf16 for the head GEMM -> logits per sample and d_head_w
       per class row 2u; the input gradient, the bias and LayerNorm gradients do not go through a stored value that can
       flip (bf16(dlogits) is a cast of the caller's gradient) -> u/8 per token row / per element.
     * Segmenter tail: Xpc, the bf16 copies of P and C can flip (3 x 2u); the class LayerNorm's fp32 statistics and the
       fp32 row norms are below that -> cmap per patch row and the output per (b, k, Y) row 8u.  Backward adds what the
       reference does not mirror - the bf16 Gs = dM rp rc (u) and the normalise backward from the bf16 copies (u) - and
       the flips of dP / dC and dXpc (2 x 2u) -> dP per patch row, dC per class row, the tail's dx per patch row and per
       class row (held apart) and the weight gradients per row 16u; mask_norm and decoder_norm gradients per element
       (against the vector's RMS) 16u.  The Segmenter proj is the ConvNeXt proj GEMM plus copies: exact tier.
   Vector gradients (biases, LayerNorm weights) are held per element, each element's error against the vector's RMS, so a
   single wrong channel cannot hide in a whole-tensor norm.
3. Contracts, in every case: `saved`, `ws` and every output are NaN before each call; parameter gradients start at
   non-zero priors and the check is on grad - prior; guard bands around every output and the workspace stay untouched;
   proj's denc is exactly 0 on the global token and the tokens of tasks that are not main tasks.  Registered bf16 weight
   mirrors (mmae_weight_mirror_register): every entry point runs twice on the cast path and once with its weights in a
   mirror, on the same inputs and priors; every output and gradient of the mirror run must have the cast run's bits
   wherever the two cast runs agree bit for bit.  The weight-gradient GEMMs and the LayerNorm parameter gradients
   accumulate with atomics (include/multimae_b200.h), so where a split-K sum makes the two cast runs differ, the mirror
   run is held to fp32 reassociation (1e-6 per row) instead.
4. Sensitivity: deliberately wrong references (convnext_head_oracle.MUTATIONS, cls_head_oracle's "mean_short") must miss
   by >= 10x the budget at the level each one can show at: per pixel, border ring only, per output row, first output
   rows only, per plane, per row, per sample."""
import ctypes
import os

import pytest
import torch

import cls_head_oracle as CH
import convnext_head_oracle as CX
from multimae_b200 import _lib as L
import segmenter_head_oracle as SG
from test_cuda_pretrain_io import _dy, _report

pytestmark = pytest.mark.gpu

U = 2.0 ** -8
BLOCK_ROW = 4 * U                  # ConvNeXt block branch, per pixel row
GRAD_ROW = 8 * U                   # ConvNeXt block gradients
FP32_ROW = U / 8                   # outputs that no bf16 flip can reach
FLIP1 = 2 * U                      # one store that can flip
EPS = 1e-6
GUARD = 256                        # bytes of guard band on each side
SENTINEL_F = 7.25
SENTINEL_B = 0x5A
MIRROR_TOL = 1e-6                  # mirror against cast, per row, where the cast path itself does not repeat bit for bit


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


# ============================================================================================================ buffers
class _Guarded:
    """A device tensor of `shape` inside a larger allocation with GUARD bytes of sentinel on each side; the tensor itself
    is filled with NaN (0xFF bytes) or with `init`."""

    def __init__(self, shape, dtype, dev, init=None):
        es = torch.empty((), dtype=dtype).element_size()
        n, g = int(torch.Size(shape).numel()), GUARD // es
        if dtype == torch.uint8:
            self.full = torch.full((n + 2 * g,), SENTINEL_B, dtype=dtype, device=dev)
        else:
            self.full = torch.full((n + 2 * g,), SENTINEL_F, dtype=dtype, device=dev)
        self.g = g
        self.t = self.full[g:g + n].view(shape)
        self.fill(init)

    def fill(self, init=None):
        if init is None:
            self.t.view(torch.uint8).fill_(0xFF)
        else:
            self.t.copy_(init)

    def ptr(self):
        return self.t.data_ptr()

    def guards_ok(self):
        s = SENTINEL_B if self.full.dtype == torch.uint8 else SENTINEL_F
        return bool((self.full[:self.g] == s).all()) and bool((self.full[self.g + self.t.numel():] == s).all())


def _guards(what, bufs):
    bad = [k for k, b in bufs.items() if not b.guards_ok()]
    assert not bad, (what, "written outside the caller's tensors", bad)


def _f32(t):
    return t.float().contiguous()


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _grads(fn, inputs, dout):
    """(out, {name: grad}) of fn(**leaves) for the output gradient dout (float64 autograd on the inputs' device)"""
    lv = {k: v.detach().clone().requires_grad_(True) for k, v in inputs.items()}
    out = fn(**lv)
    out.backward(dout)
    return out.detach(), {k: v.grad for k, v in lv.items()}


def _check_exact(what, got, ref, absref, q, nterms):
    """torch.equal where the exactness premise holds on the reference, else within the fp32 summation bound
    nterms 2^-24 sum|terms| element by element.  Returns which of the two was checked."""
    got = got.double()
    exact = (torch.equal(ref, ref.float().double()) and torch.equal(absref * 2 ** q, torch.round(absref * 2 ** q))
             and float(absref.max()) < 2.0 ** (23 - q))
    if exact:
        assert torch.equal(got, ref), (what, float((got - ref).abs().max()))
        return "exact"
    err = (got - ref).abs()
    bound = nterms * 2.0 ** -24 * absref
    assert bool((err <= bound).all()), (what, int((err > bound).sum()), float((err - bound).max()))
    return "bound(%.2g)" % float((err / bound.clamp_min(1e-300)).max())


def _row_rel(got, ref):
    """per-row relative L2 error over the last dimension (rows of zero norm compare absolutely)"""
    got, ref = got.double().flatten(0, -2), ref.double().flatten(0, -2)
    return (got - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-30)


def _whole_rel(got, ref):
    return float((got.double() - ref).norm() / ref.norm().clamp_min(1e-30))


def _elem_rel(got, ref):
    """worst element error of a vector against its RMS"""
    ref = ref.double().flatten()
    return float((got.double().flatten() - ref).abs().max() / ref.pow(2).mean().sqrt().clamp_min(1e-30))


def _same_bits(what, cast1, cast2, mirror):
    """the mirror run has the cast run's bits where the cast path repeats bit for bit, else within MIRROR_TOL per row"""
    if torch.equal(cast1, cast2):
        assert torch.equal(mirror, cast1), (what, "mirror differs from cast")
        return "bits"
    rel = float(_row_rel(mirror.reshape(-1, mirror.shape[-1]), cast1.reshape(-1, cast1.shape[-1])).max())
    assert rel <= MIRROR_TOL, (what, rel)
    return "%.1e" % rel


# ========================================================================================================= ConvNeXt
# B, nh, nw, s, C, K, main tasks (E = s*s*C; the encoder has three tasks of n = nh*nw tokens and one global token)
CNX_CASES = {
    "ade512": (2, 32, 32, 4, 384, 150, 1),           # ADE20K 512^2, K = 150: ragged backward class chunks at W = 512
    "nyu640_rgb": (2, 40, 40, 4, 384, 40, 1),       # NYUv2 640^2: forward class chunks 37 + 3
    "nyu640_rgbd": (1, 40, 40, 4, 384, 40, 2),
    "depth256": (2, 16, 16, 8, 96, 1, 1),            # the depth head: C = 96 (the narrow LayerNorm), K = 1
    "ragged3x5": (3, 3, 5, 4, 384, 13, 2),           # Hf x Wf = 12 x 20: partial dwconv tiles both ways
    "s2_nonsquare": (2, 6, 4, 2, 256, 13, 1),
    "s1": (2, 5, 7, 1, 512, 9, 1),
    "nonsquare": (2, 3, 4, 4, 384, 21, 2),
}
D_ENC = 768


def _starts(case):
    B, nh, nw, s, C, K, T = CNX_CASES[case]
    n = nh * nw
    return n, ([n] if T == 1 else [2 * n, 0])       # other tasks' tokens and the global token between / after them


def _align(x, a=256):
    return (x + a - 1) // a * a


def _block_offsets(P, C):
    """byte offsets of `d` in the block's saved buffer and of `dd` in its workspace (blk_saved / blk_ws in
    convnext_head.cu: 256-byte aligned takes in that order)"""
    w = _align(4 * C * C * 2)
    d_off = _align(w + 4 * C * C * 2)
    dd_off = _align(_align(_align(P * C * 2) + P * 4 * C * 2) + P * C * 2)
    return d_off, dd_off


class _Mirror:
    """fp32 weights packed into one registered parameter buffer with its bf16 twin (8-element aligned slots)"""

    def __init__(self, tensors, dev):
        sizes = [_align(t.numel(), 8) for t in tensors]
        self.flat = torch.zeros(sum(sizes), device=dev)
        self.views, off = [], 0
        for t, n in zip(tensors, sizes):
            v = self.flat[off:off + t.numel()].view(t.shape)
            v.copy_(t)
            self.views.append(v)
            off += n
        self.twin = self.flat.to(torch.bfloat16)
        L.check(L.lib().mmae_weight_mirror_register(self.flat.data_ptr(), self.twin.data_ptr(), self.flat.numel()), "mirror")

    def close(self):
        L.lib().mmae_weight_mirror_register(self.flat.data_ptr(), None, 0)


def _proj_call(dev, case, enc, w, b, dx_out, prior_w, prior_b, mirror=None):
    """forward + backward of mmae_convnext_proj on fp32 copies; returns (x_out, denc, d_w - prior, d_b - prior)"""
    B, nh, nw, s, C, K, T = CNX_CASES[case]
    n, starts = _starts(case)
    lib, st = L.lib(), L.current_stream()
    E, N = s * s * C, enc.shape[1]
    st_arr = (ctypes.c_int * T)(*starts)
    w32 = mirror.views[0] if mirror else _f32(w)
    bufs = {"saved": _Guarded((lib.mmae_convnext_proj_saved_bytes(B, n, D_ENC * T, E),), torch.uint8, dev),
            "ws": _Guarded((lib.mmae_convnext_proj_workspace_bytes(B, n, D_ENC * T, E),), torch.uint8, dev),
            "x_out": _Guarded((B * n, E), torch.float32, dev), "denc": _Guarded((B, N, D_ENC), torch.float32, dev),
            "d_w": _Guarded(w.shape, torch.float32, dev, prior_w), "d_b": _Guarded(b.shape, torch.float32, dev, prior_b)}
    enc32, b32, dx32 = _f32(enc), _f32(b), _f32(dx_out)
    L.check(lib.mmae_convnext_proj_forward(enc32.data_ptr(), B, N, D_ENC, n, T, st_arr, E, w32.data_ptr(), b32.data_ptr(),
                                           bufs["x_out"].ptr(), bufs["saved"].ptr(), bufs["ws"].ptr(), st), "proj forward")
    bufs["ws"].fill()
    L.check(lib.mmae_convnext_proj_backward(dx32.data_ptr(), B, N, D_ENC, n, T, st_arr, E, w32.data_ptr(),
                                            bufs["d_w"].ptr(), bufs["d_b"].ptr(), bufs["denc"].ptr(), bufs["saved"].ptr(),
                                            bufs["ws"].ptr(), st), "proj backward")
    torch.cuda.synchronize()
    _guards("proj " + case, bufs)
    return (bufs["x_out"].t.double(), bufs["denc"].t.double(), bufs["d_w"].t.double() - prior_w,
            bufs["d_b"].t.double() - prior_b)


def _block_call(dev, case, x, prm, dx_out, priors, mirror=None):
    """forward + backward of mmae_convnext_block; returns (x_out, dx_in, {name: grad - prior}, saved d, workspace dd)"""
    B, nh, nw, s, C, K, T = CNX_CASES[case]
    lib, st = L.lib(), L.current_stream()
    P = B * nh * nw * s * s
    p32 = {k: _f32(v) for k, v in prm.items()}
    if mirror:
        p32["pw1_w"], p32["pw2_w"] = mirror.views[1], mirror.views[2]
    bufs = {"saved": _Guarded((lib.mmae_convnext_block_saved_bytes(B, nh, nw, s, C),), torch.uint8, dev),
            "ws": _Guarded((lib.mmae_convnext_block_workspace_bytes(B, nh, nw, s, C),), torch.uint8, dev),
            "x_out": _Guarded((P, C), torch.float32, dev), "dx_in": _Guarded((P, C), torch.float32, dev)}
    for k in CX.BLOCK_PARAMS:
        bufs["g_" + k] = _Guarded(prm[k].shape, torch.float32, dev, priors[k])
    x32, dx32 = _f32(x), _f32(dx_out)
    pa = _ptrs([p32[k] for k in CX.BLOCK_PARAMS])
    ga = _ptrs([bufs["g_" + k].t for k in CX.BLOCK_PARAMS])
    L.check(lib.mmae_convnext_block_forward(x32.data_ptr(), bufs["x_out"].ptr(), B, nh, nw, s, C, EPS, pa,
                                            bufs["saved"].ptr(), bufs["ws"].ptr(), st), "block forward")
    bufs["ws"].fill()
    L.check(lib.mmae_convnext_block_backward(x32.data_ptr(), dx32.data_ptr(), bufs["dx_in"].ptr(), B, nh, nw, s, C, pa, ga,
                                             bufs["saved"].ptr(), bufs["ws"].ptr(), st), "block backward")
    torch.cuda.synchronize()
    _guards("block " + case, bufs)
    d_off, dd_off = _block_offsets(P, C)
    d = bufs["saved"].t[d_off:d_off + 4 * P * C].view(torch.float32).view(P, C).double()
    dd = bufs["ws"].t[dd_off:dd_off + 4 * P * C].view(torch.float32).view(P, C).double()
    grads = {k: bufs["g_" + k].t.double() - priors[k] for k in CX.BLOCK_PARAMS}
    return bufs["x_out"].t.double(), bufs["dx_in"].t.double(), grads, d, dd


def _tail_call(dev, case, x, w, b, dout, prior_w, prior_b, mirror=None):
    B, nh, nw, s, C, K, T = CNX_CASES[case]
    lib, st = L.lib(), L.current_stream()
    H, W = nh * 16, nw * 16
    dims = (B, nh, nw, s, C, K)
    w32 = mirror.views[3] if mirror else _f32(w)
    bufs = {"saved": _Guarded((lib.mmae_convnext_tail_saved_bytes(*dims),), torch.uint8, dev),
            "ws": _Guarded((lib.mmae_convnext_tail_workspace_bytes(*dims),), torch.uint8, dev),
            "out": _Guarded((B, K, H, W), torch.float32, dev), "dx": _Guarded(x.shape, torch.float32, dev),
            "d_w": _Guarded(w.shape, torch.float32, dev, prior_w), "d_b": _Guarded(b.shape, torch.float32, dev, prior_b)}
    x32, b32, do32 = _f32(x), _f32(b), _f32(dout)
    L.check(lib.mmae_convnext_tail_forward(x32.data_ptr(), *dims, H, W, w32.data_ptr(), b32.data_ptr(), bufs["out"].ptr(),
                                           bufs["saved"].ptr(), bufs["ws"].ptr(), st), "tail forward")
    bufs["ws"].fill()
    L.check(lib.mmae_convnext_tail_backward(do32.data_ptr(), *dims, H, W, w32.data_ptr(), bufs["d_w"].ptr(),
                                            bufs["d_b"].ptr(), bufs["dx"].ptr(), bufs["saved"].ptr(), bufs["ws"].ptr(), st),
            "tail backward")
    torch.cuda.synchronize()
    _guards("tail " + case, bufs)
    return (bufs["out"].t.double(), bufs["dx"].t.double(), bufs["d_w"].t.double() - prior_w,
            bufs["d_b"].t.double() - prior_b)


def _sparse(shape, keep, gen, dev):
    return (torch.rand(shape, generator=gen) < keep).double().to(dev)


def _exact_inputs(case, dev, gen):
    B, nh, nw, s, C, K, T = CNX_CASES[case]
    n, _ = _starts(case)
    P, E = B * n * s * s, s * s * C
    r = lambda *shape, scale=1.0: (torch.randn(*shape, generator=gen, dtype=torch.float64) * scale).float().double().to(dev)
    z = {"enc": _dy((B, 3 * n + 1, D_ENC), 3, gen, dev), "proj_w": _dy((E, T * D_ENC), 4, gen, dev),
         "proj_b": _dy((E,), 4, gen, dev), "proj_dx": _dy((P, C), 4, gen, dev),
         "proj_pw": _dy((E, T * D_ENC), 4, gen, dev), "proj_pb": _dy((E,), 4, gen, dev),
         "x": _dy((P, C), 3, gen, dev), "blk_dx": _dy((P, C), 4, gen, dev),
         "prm": {"dw_w": _dy((C, 1, 7, 7), 4, gen, dev), "dw_b": _dy((C,), 4, gen, dev), "norm_w": 1 + _dy((C,), 4, gen, dev),
                 "norm_b": _dy((C,), 4, gen, dev), "pw1_w": r(4 * C, C, scale=C ** -0.5), "pw1_b": r(4 * C, scale=0.1),
                 "pw2_w": r(C, 4 * C, scale=(4 * C) ** -0.5), "pw2_b": r(C, scale=0.1)},
         # sparse {0, +-1/8} / {0, +-1/16}: the tail's weight- and bias-gradient sums over every pixel stay exact
         "tail_x": _dy((P, C), 3, gen, dev, kmax=1) * _sparse((P, C), 0.5, gen, dev),
         "tail_w": _dy((K, C), 4, gen, dev, kmax=4), "tail_b": _dy((K,), 4, gen, dev),
         "tail_dout": _dy((B, K, nh * 16, nw * 16), 4, gen, dev, kmax=1) * _sparse((B, K, nh * 16, nw * 16), 0.125, gen, dev),
         "tail_pw": _dy((K, C), 4, gen, dev), "tail_pb": _dy((K,), 4, gen, dev)}
    z["blk_prior"] = {k: _dy(v.shape, 4, gen, dev) for k, v in z["prm"].items()}
    return z


@pytest.mark.parametrize("case", list(CNX_CASES))
def test_convnext_exact(dev, case):
    B, nh, nw, s, C, K, T = CNX_CASES[case]
    n, starts = _starts(case)
    geo, H, W = (B, nh, nw, s), nh * 16, nw * 16
    P = B * n * s * s
    z = _exact_inputs(case, dev, torch.Generator().manual_seed(41))
    got_p = _proj_call(dev, case, z["enc"], z["proj_w"], z["proj_b"], z["proj_dx"], z["proj_pw"], z["proj_pb"])
    got_b = _block_call(dev, case, z["x"], z["prm"], z["blk_dx"], z["blk_prior"])
    got_t = _tail_call(dev, case, z["tail_x"], z["tail_w"], z["tail_b"], z["tail_dout"], z["tail_pw"], z["tail_pb"])
    kinds = []
    # ---- proj: gather + GEMM, and the scatter of the input gradient
    fn = lambda enc, w, b: CX.proj(enc, w, b, starts, n).reshape(P, C)
    ins = {"enc": z["enc"], "w": z["proj_w"], "b": z["proj_b"]}
    ref, rg = _grads(fn, ins, z["proj_dx"])
    aref, ag = _grads(fn, {k: v.abs() for k, v in ins.items()}, z["proj_dx"].abs())
    kinds.append(_check_exact("proj x_out", got_p[0].reshape(P, C), ref, aref, 7, T * D_ENC + 1))
    kinds.append(_check_exact("proj denc", got_p[1], rg["enc"], ag["enc"], 8, s * s * C))
    kinds.append(_check_exact("proj d_w", got_p[2], rg["w"], ag["w"] + z["proj_pw"].abs(), 7, B * n + 1))
    kinds.append(_check_exact("proj d_b", got_p[3], rg["b"], ag["b"] + z["proj_pb"].abs(), 4, B * n + 1))
    tok = torch.ones(3 * n + 1, dtype=torch.bool, device=dev)
    for s0 in starts:
        tok[s0:s0 + n] = False
    assert torch.equal(got_p[1][:, tok], torch.zeros_like(got_p[1][:, tok]))   # other tasks' tokens, the global token
    # ---- dwconv forward (the saved d), its transposed backward and parameter gradients against the kernels' dd
    x_out, dx_in, gb, d, dd = got_b
    conv = lambda x, w, b: CX.image_to_rows(CX.dwconv(CX.rows_to_image(x, geo), w, b), geo)
    ins = {"x": z["x"], "w": z["prm"]["dw_w"], "b": z["prm"]["dw_b"]}
    ref, rg = _grads(conv, ins, dd)
    aref, ag = _grads(conv, {k: v.abs() for k, v in ins.items()}, dd.abs())
    kinds.append(_check_exact("dwconv d", d, ref, aref, 7, 50))
    kinds.append(_check_exact("dwconv dx_in", dx_in, z["blk_dx"] + rg["x"], z["blk_dx"].abs() + ag["x"], 24, 50))
    kinds.append(_check_exact("dwconv d_w", gb["dw_w"], rg["w"], ag["w"] + z["blk_prior"]["dw_w"].abs(), 24,
                              B * nh * nw * s * s + 1))
    kinds.append(_check_exact("dwconv d_b", gb["dw_b"], rg["b"], ag["b"] + z["blk_prior"]["dw_b"].abs(), 24, P + 1))
    assert not bool(torch.isnan(x_out).any())
    # ---- tail: final_layer + upsample and its gather-form backward
    r = 16 // s
    m = CX.interp_matrix(H, nh * s)
    assert torch.equal(m * 2 * r, torch.round(m * 2 * r)), case
    fn = lambda x, w, b: CX.tail(x, w, b, geo, H, W)
    ins = {"x": z["tail_x"], "w": z["tail_w"], "b": z["tail_b"]}
    ref, rg = _grads(fn, ins, z["tail_dout"])
    aref, ag = _grads(fn, {k: v.abs() for k, v in ins.items()}, z["tail_dout"].abs())
    qb = 2 * (r.bit_length())                                   # two weights, each a multiple of 2^-log2(2r)
    kinds.append(_check_exact("tail out", got_t[0], ref, aref, 7 + qb, C + 5))
    kinds.append(_check_exact("tail dx", got_t[1], rg["x"], ag["x"], 4 + qb + 4, K + 4 * r * r))
    kinds.append(_check_exact("tail d_w", got_t[2], rg["w"], ag["w"] + z["tail_pw"].abs(), 4 + qb + 3, P + 4 * r * r))
    kinds.append(_check_exact("tail d_b", got_t[3], rg["b"], ag["b"] + z["tail_pb"].abs(), 4 + qb, P + 4 * r * r))
    names = ["proj x_out", "proj denc", "proj d_w", "proj d_b", "dwconv d", "dwconv dx_in", "dwconv d_w", "dwconv d_b",
             "tail out", "tail dx", "tail d_w", "tail d_b"]
    print("convnext exact %s: %s" % (case, ", ".join("%s %s" % nk for nk in zip(names, kinds))))
    bounded = ("dwconv dx_in", "dwconv d_w", "dwconv d_b")        # sums of the kernels' non-dyadic dd
    not_exact = [nm for nm, k in zip(names, kinds) if k != "exact" and nm not in bounded]
    assert not not_exact, not_exact


@pytest.mark.parametrize("case", ["ragged3x5", "depth256", "nyu640_rgbd"])
def test_convnext_weight_mirror(dev, case):
    """proj, block and tail with their weights in a registered bf16 mirror against the cast path, same inputs and priors"""
    z = _exact_inputs(case, dev, torch.Generator().manual_seed(42))

    def run(mir=None):
        p = _proj_call(dev, case, z["enc"], z["proj_w"], z["proj_b"], z["proj_dx"], z["proj_pw"], z["proj_pb"], mir)
        b = _block_call(dev, case, z["x"], z["prm"], z["blk_dx"], z["blk_prior"], mir)
        t = _tail_call(dev, case, z["tail_x"], z["tail_w"], z["tail_b"], z["tail_dout"], z["tail_pw"], z["tail_pb"], mir)
        out = dict(zip(["proj x_out", "proj denc", "proj d_w", "proj d_b"], p))
        out.update(zip(["block x_out", "block dx_in"], b[:2]))
        out.update({"block " + k: v for k, v in b[2].items()})
        out.update(zip(["tail out", "tail dx", "tail d_w", "tail d_b"], t))
        return out

    cast1, cast2 = run(), run()
    mir = _Mirror([_f32(z["proj_w"]), _f32(z["prm"]["pw1_w"]), _f32(z["prm"]["pw2_w"]), _f32(z["tail_w"])], dev)
    try:
        mirrored = run(mir)
    finally:
        mir.close()
    print("convnext %s mirror: %s" % (case, ", ".join("%s %s" % (k, _same_bits(k, cast1[k], cast2[k], mirrored[k]))
                                                      for k in cast1)))


# ------------------------------------------------------------------------------------------------------ rounding tier
def _regions(geo, dev):
    """masks over the [P] pixel rows: map-border ring (within 3 of an edge), dwconv tile boundaries (within 3 of the edge
    of an 8 x 16 tile, not on the ring) and the interior"""
    B, nh, nw, s = geo
    Hf, Wf = nh * s, nw * s
    yy = torch.arange(Hf, device=dev).view(1, 1, Hf, 1).expand(B, 1, Hf, Wf)
    xx = torch.arange(Wf, device=dev).view(1, 1, 1, Wf).expand(B, 1, Hf, Wf)
    y, x = CX.image_to_rows(yy, geo)[:, 0], CX.image_to_rows(xx, geo)[:, 0]
    ring = (y < 3) | (y >= Hf - 3) | (x < 3) | (x >= Wf - 3)
    tile = ~ring & ((y % 8 < 3) | (y % 8 >= 5) | (x % 16 < 3) | (x % 16 >= 13))
    return {"ring": ring, "tile": tile, "interior": ~ring & ~tile}


def _rnd(gen, dev, *shape, scale=1.0, offset=0.0):
    return (offset + scale * torch.randn(*shape, generator=gen, dtype=torch.float64)).float().double().to(dev)


def _cnx_round_run(dev, case, fuse, mutations=()):
    B, nh, nw, s, C, K, T = CNX_CASES[case]
    n, starts = _starts(case)
    geo, H, W = (B, nh, nw, s), nh * 16, nw * 16
    P, E = B * n * s * s, s * s * C
    gen = torch.Generator().manual_seed(43)
    r = lambda *shape, **kw: _rnd(gen, dev, *shape, **kw)
    enc, pw, pb = r(B, 3 * n + 1, D_ENC), r(E, T * D_ENC, scale=(T * D_ENC) ** -0.5), r(E, scale=0.1)
    prm = {"dw_w": r(C, 1, 7, 7, scale=0.2), "dw_b": r(C, scale=0.1), "norm_w": r(C, scale=0.1, offset=1.0),
           "norm_b": r(C, scale=0.1), "pw1_w": r(4 * C, C, scale=C ** -0.5), "pw1_b": r(4 * C, scale=0.1),
           "pw2_w": r(C, 4 * C, scale=(4 * C) ** -0.5), "pw2_b": r(C, scale=0.1)}
    priors = {k: r(*v.shape) for k, v in prm.items()}
    x, dx_out = r(P, C), r(P, C)
    tw, tb, dout = r(K, C, scale=C ** -0.5), r(K, scale=0.1), r(B, K, H, W)
    tpw, tpb = r(K, C), r(K)
    got_p = _proj_call(dev, case, enc, pw, pb, r(P, C), r(E, T * D_ENC), r(E))
    got_b = _block_call(dev, case, x, prm, dx_out, priors)
    got_t = _tail_call(dev, case, x, tw, tb, dout, tpw, tpb)
    reg = _regions(geo, dev)

    def checks(mutate):
        """[(label, error, budget)] plus the per-level maxima the mutations are judged at"""
        errs, lev = [], {}
        # proj forward, per pixel row
        pref = CX.proj(enc, pw, pb, starts, n, mutate=mutate if mutate == "tasks_reversed" else None).reshape(P, C)
        e = _row_rel(got_p[0].reshape(P, C), pref)
        errs.append(("proj x_out row", float(e.max()), FP32_ROW))
        lev["pixel"] = [float(e.max()) / FP32_ROW]
        # block
        bm = mutate if mutate in CX.MUTATIONS else None
        leaves = {k: v.clone().requires_grad_(True) for k, v in prm.items()}
        xi = x.clone().requires_grad_(True)
        xo = CX.block(xi, leaves, geo, EPS, True, bool(fuse), bm)
        xo.backward(dx_out)
        br = _row_rel(got_b[0] - x, (xo - xi).detach())
        dxr = _row_rel(got_b[1] - dx_out, xi.grad - dx_out)
        for nm, v, bud in (("branch", br, BLOCK_ROW), ("dx_in - dx_out", dxr, GRAD_ROW)):
            for rg_, msk in reg.items():
                if bool(msk.any()):
                    errs.append(("%s %s row" % (nm, rg_), float(v[msk].max()), bud))
            lev["pixel"].append(float(v.max()) / bud)
            lev.setdefault("ring", []).append(float(v[reg["ring"]].max()) / bud)
        for k in CX.BLOCK_PARAMS:
            g, rf_ = got_b[2][k], leaves[k].grad
            if k in ("dw_w", "pw1_w", "pw2_w"):
                errs.append((k + " row", float(_row_rel(g.flatten(1), rf_.flatten(1)).max()), GRAD_ROW))
            else:
                errs.append((k + " element", _elem_rel(g, rf_), GRAD_ROW))
        # tail
        lv = {"w": tw.clone().requires_grad_(True), "b": tb.clone().requires_grad_(True), "x": x.clone().requires_grad_(True)}
        out = CX.tail(lv["x"], lv["w"], lv["b"], geo, H, W, mutate=mutate if mutate in CX.MUTATIONS else None)
        out.backward(dout)
        out = out.detach()
        orow = _row_rel(got_t[0], out).view(B, K, H)
        oplane = _row_rel(got_t[0].flatten(2), out.flatten(2))
        errs += [("tail out row", float(orow.max()), FP32_ROW), ("tail out plane", float(oplane.max()), FP32_ROW),
                 ("tail dx row", float(_row_rel(got_t[1], lv["x"].grad).max()), FLIP1),
                 ("tail d_w row", float(_row_rel(got_t[2], lv["w"].grad).max()), FLIP1),
                 ("tail d_b element", _elem_rel(got_t[3], lv["b"].grad), FP32_ROW)]
        lev["out_row"] = [float(orow.max()) / FP32_ROW]
        lev["first_rows"] = [float(orow[:, :, :r_half].max()) / FP32_ROW]
        lev["plane"] = [float(oplane.max()) / FP32_ROW]
        return errs, lev

    r_half = max(1, (16 // s) // 2)
    errs, _ = checks(None)
    frac = _report("convnext %s fuse=%d" % (case, fuse), errs)
    assert frac <= 1.0, [e for e in errs if e[1] > e[2]]
    levels = {"tasks_reversed": "pixel", "pixel_transpose": "pixel", "flip_fwd": "pixel", "flip_bwd": "pixel",
              "neighbour_sample": "pixel", "replicate_pad": "ring", "align_corners": "out_row", "no_clamp": "first_rows",
              "class_shift": "plane"}
    for m in mutations:
        _, lev = checks(m)
        miss = max(lev[levels[m]])
        print("  wrong reference %s: %.1f x budget at the %s level" % (m, miss, levels[m]))
        assert miss >= 10.0, (m, miss)


@pytest.mark.parametrize("case", list(CNX_CASES))
def test_convnext_against_rounding_reference(dev, case):
    muts = ()
    if case == "ragged3x5":
        muts = CX.MUTATIONS
    elif case == "nyu640_rgb":
        muts = ("class_shift",)
    _cnx_round_run(dev, case, int(os.environ.get("MMAE_FUSE_GELU", "0")), muts)      # the library's default mode


def test_convnext_fused_gelu(dev, fuse_gelu):
    _cnx_round_run(dev, "nonsquare", fuse_gelu)


# ========================================================================================================= cls head
# B, N, D, C, mean_pool
CLS_CASES = {
    "in1k_mean": (128, 197, 768, 1000, 1),
    "in1k_last": (128, 197, 768, 1000, 0),
    "c101": (8, 197, 768, 101, 1),
    "c37_last": (8, 197, 768, 37, 0),
    "c1": (8, 197, 768, 1, 1),
    "c0": (8, 197, 768, 0, 1),
    "d1024": (16, 197, 1024, 1000, 1),
    "n1": (4, 1, 768, 37, 1),
}


def _cls_call(dev, case, x, nw_, nb_, hw, hb, dout, priors, mirror=None):
    B, N, D, C, mean = CLS_CASES[case]
    lib, st = L.lib(), L.current_stream()
    bufs = {"saved": _Guarded((lib.mmae_clshead_saved_bytes(B, N, D, C),), torch.uint8, dev),
            "ws": _Guarded((lib.mmae_clshead_workspace_bytes(B, N, D, C),), torch.uint8, dev),
            "out": _Guarded((B, C if C else D), torch.float32, dev), "dx": _Guarded((B, N, D), torch.float32, dev),
            "d_nw": _Guarded((D,), torch.float32, dev, priors["nw"]), "d_nb": _Guarded((D,), torch.float32, dev, priors["nb"])}
    if C:
        bufs["d_hw"] = _Guarded((C, D), torch.float32, dev, priors["hw"])
        bufs["d_hb"] = _Guarded((C,), torch.float32, dev, priors["hb"])
    x32, nw32, nb32, do32 = _f32(x), _f32(nw_), _f32(nb_), _f32(dout)
    hw32 = (mirror.views[0] if mirror else _f32(hw)) if C else None
    hb32 = _f32(hb) if C else None
    pp = lambda t: None if t is None else t.data_ptr()
    L.check(lib.mmae_clshead_forward(x32.data_ptr(), B, N, D, C, mean, EPS, nw32.data_ptr(), nb32.data_ptr(), pp(hw32),
                                     pp(hb32), bufs["out"].ptr(), bufs["saved"].ptr(), bufs["ws"].ptr(), st), "cls forward")
    bufs["ws"].fill()
    L.check(lib.mmae_clshead_backward(do32.data_ptr(), B, N, D, C, mean, nw32.data_ptr(), pp(hw32), bufs["d_nw"].ptr(),
                                      bufs["d_nb"].ptr(), bufs["d_hw"].ptr() if C else None,
                                      bufs["d_hb"].ptr() if C else None, bufs["dx"].ptr(), bufs["saved"].ptr(),
                                      bufs["ws"].ptr(), st), "cls backward")
    torch.cuda.synchronize()
    _guards("cls " + case, bufs)
    got = {"out": bufs["out"].t.double(), "dx": bufs["dx"].t.double(), "nw": bufs["d_nw"].t.double() - priors["nw"],
           "nb": bufs["d_nb"].t.double() - priors["nb"]}
    if C:
        got["hw"] = bufs["d_hw"].t.double() - priors["hw"]
        got["hb"] = bufs["d_hb"].t.double() - priors["hb"]
    return got


@pytest.mark.parametrize("case", list(CLS_CASES))
def test_cls_head_against_rounding_reference(dev, case):
    B, N, D, C, mean = CLS_CASES[case]
    gen = torch.Generator().manual_seed(47)
    r = lambda *shape, **kw: _rnd(gen, dev, *shape, **kw)
    x = r(B, N, D, offset=0.3)
    ins = {"enc": x, "nw": r(D, scale=0.1, offset=1.0), "nb": r(D, scale=0.1)}
    if C:
        ins.update(hw=r(C, D, scale=D ** -0.5), hb=r(C, scale=0.1))
    dout = r(B, C if C else D)
    priors = {"nw": r(D), "nb": r(D), "hw": r(C, D) if C else None, "hb": r(C) if C else None}
    got = _cls_call(dev, case, x, ins["nw"], ins["nb"], ins.get("hw"), ins.get("hb"), dout, priors)
    if C:
        again = _cls_call(dev, case, x, ins["nw"], ins["nb"], ins["hw"], ins["hb"], dout, priors)
        mir = _Mirror([_f32(ins["hw"])], dev)
        try:
            got_m = _cls_call(dev, case, x, ins["nw"], ins["nb"], ins["hw"], ins["hb"], dout, priors, mir)
        finally:
            mir.close()
        print("cls %s mirror: %s" % (case, ", ".join("%s %s" % (k, _same_bits(k, got[k], again[k], got_m[k]))
                                                     for k in got)))

    def checks(mutate):
        fn = lambda enc, nw, nb, hw=None, hb=None: CH.head(enc, nw, nb, hw, hb, bool(mean), EPS, True, mutate)
        ref, rg = _grads(fn, ins, dout)
        lev = [float(_row_rel(got["out"], ref).max()) / (FLIP1 if C else FP32_ROW)]
        errs = [("out per sample", float(_row_rel(got["out"], ref).max()), FLIP1 if C else FP32_ROW),
                ("dx per token row", float(_row_rel(got["dx"], rg["enc"]).max()), FP32_ROW),
                ("d_norm_w element", _elem_rel(got["nw"], rg["nw"]), FP32_ROW),
                ("d_norm_b element", _elem_rel(got["nb"], rg["nb"]), FP32_ROW)]
        lev.append(float(_row_rel(got["dx"].flatten(1), rg["enc"].flatten(1)).max()) / FP32_ROW)
        if C:
            errs += [("d_head_w per class row", float(_row_rel(got["hw"], rg["hw"]).max()), FLIP1),
                     ("d_head_b element", _elem_rel(got["hb"], rg["hb"]), FP32_ROW)]
        return errs, max(lev)

    errs, _ = checks(None)
    frac = _report("cls %s" % case, errs)
    assert frac <= 1.0, [e for e in errs if e[1] > e[2]]
    if mean:                                     # every token row of a sample gets the same gradient, bit for bit
        assert torch.equal(got["dx"], got["dx"][:, :1].expand(-1, N, -1))
    else:                                        # only the global token (the last row) gets one
        assert not bool(got["dx"][:, :-1].any()) and bool(got["dx"][:, -1].any())
    if case == "in1k_mean":
        _, miss = checks("mean_short")
        print("  wrong reference mean_short: %.1f x budget per sample" % miss)
        assert miss >= 10.0, miss


# ======================================================================================================== Segmenter
SEG_E = 768
SEG_FWD = 8 * U                    # cmap per patch row, output per row
SEG_BWD = 16 * U                   # dP / dC / dx per row, weight gradients per row, vectors per element
# B, nh, nw, K, one patch row all zero (the 1e-12 clamp of the row norms)
SEG_CASES = {
    "ade_n1024_k150": (2, 32, 32, 150, False),
    "nyu_n1280_k41": (2, 40, 32, 41, False),        # 640 x 512
    "k8": (2, 10, 10, 8, False),                    # K on both sides of the mask kernel's accumulator widths 64 / 160 / 256
    "k64": (2, 10, 10, 64, False),
    "k65": (2, 10, 10, 65, False),
    "k160": (2, 10, 10, 160, False),
    "k161": (2, 10, 10, 161, False),
    "k256": (2, 10, 10, 256, False),
    "n12": (3, 3, 4, 13, False),                    # n not a multiple of the 64-row CTA: 12, 77, 100
    "n77_zero_row": (2, 7, 11, 20, True),
}


def _seg_tail_offsets(B, n, K, E):
    """byte offsets of cmap / dPC in the tail's workspace (tl_ws in segmenter_head.cu: 256-byte aligned takes)"""
    rows = B * (n + K)
    dpc = _align(rows * E * 2)
    cmap = _align(_align(_align(dpc + rows * E * 2) + rows * E * 2) + rows * E * 4)
    return cmap, dpc


def _seg_tail_call(dev, case, x, prm, dout, priors, mirror=None):
    B, nh, nw, K, _ = SEG_CASES[case]
    n, E, Kp = nh * nw, SEG_E, _align(K, 8)
    lib, st = L.lib(), L.current_stream()
    H, W = nh * 16, nw * 16
    p32 = {k: _f32(v) for k, v in prm.items()}
    if mirror:
        p32["patch_w"], p32["classes_w"] = mirror.views
    bufs = {"saved": _Guarded((lib.mmae_segmenter_tail_saved_bytes(B, nh, nw, E, K),), torch.uint8, dev),
            "ws": _Guarded((lib.mmae_segmenter_tail_workspace_bytes(B, nh, nw, E, K),), torch.uint8, dev),
            "out": _Guarded((B, K, H, W), torch.float32, dev), "dx": _Guarded(x.shape, torch.float32, dev)}
    for k in SG.TAIL_PARAMS:
        bufs["g_" + k] = _Guarded(prm[k].shape, torch.float32, dev, priors[k])
    x32, do32 = _f32(x), _f32(dout)
    pa = _ptrs([p32[k] for k in SG.TAIL_PARAMS])
    ga = _ptrs([bufs["g_" + k].t for k in SG.TAIL_PARAMS])
    cm_off, dpc_off = _seg_tail_offsets(B, n, K, E)
    L.check(lib.mmae_segmenter_tail_forward(x32.data_ptr(), B, nh, nw, E, K, H, W, EPS, EPS, pa, bufs["out"].ptr(),
                                            bufs["saved"].ptr(), bufs["ws"].ptr(), st), "segmenter tail forward")
    cmap = bufs["ws"].t[cm_off:cm_off + 4 * B * n * Kp].view(torch.float32).view(B * n, Kp).double().clone()
    bufs["ws"].fill()
    L.check(lib.mmae_segmenter_tail_backward(x32.data_ptr(), do32.data_ptr(), bufs["dx"].ptr(), B, nh, nw, E, K, H, W, pa, ga,
                                             bufs["saved"].ptr(), bufs["ws"].ptr(), st), "segmenter tail backward")
    torch.cuda.synchronize()
    _guards("segmenter tail " + case, bufs)
    dpc = bufs["ws"].t[dpc_off:dpc_off + 2 * B * (n + K) * E].view(torch.bfloat16).view(B * (n + K), E).double()
    got = {"out": bufs["out"].t.double(), "dx": bufs["dx"].t.double(), "cmap": cmap, "dP": dpc[:B * n], "dC": dpc[B * n:]}
    got.update({k: bufs["g_" + k].t.double() - priors[k] for k in SG.TAIL_PARAMS})
    return got


def _seg_inputs(case, dev, seed):
    B, nh, nw, K, zero_row = SEG_CASES[case]
    n, E = nh * nw, SEG_E
    gen = torch.Generator().manual_seed(seed)
    r = lambda *shape, **kw: _rnd(gen, dev, *shape, **kw)
    x = r(B, n + K, E)
    prm = {"dec_w": r(E, scale=0.1, offset=1.0), "dec_b": r(E, scale=0.1), "patch_w": r(E, E, scale=E ** -0.5),
           "classes_w": r(E, E, scale=E ** -0.5), "mask_w": r(K, scale=0.1, offset=1.0), "mask_b": r(K, scale=0.1)}
    if zero_row:                  # a zero token normalises to 0 and, without a decoder_norm bias, projects to P = 0
        x[0, 5] = 0.0
        prm["dec_b"] = torch.zeros_like(prm["dec_b"])
    priors = {k: r(*v.shape) for k, v in prm.items()}
    return x, prm, r(B, K, nh * 16, nw * 16), priors


@pytest.mark.parametrize("case", list(SEG_CASES))
def test_segmenter_tail_against_rounding_reference(dev, case):
    B, nh, nw, K, zero_row = SEG_CASES[case]
    n = nh * nw
    x, prm, dout, priors = _seg_inputs(case, dev, 53)
    got = _seg_tail_call(dev, case, x, prm, dout, priors)
    assert not bool(got["cmap"][:, K:].any())                 # the class map's pad columns are zero

    def checks(mutate):
        keep = {}
        ref, rg = _grads(lambda x, **p: SG.tail(x, p, nh, nw, nh * 16, nw * 16, EPS, EPS, True, mutate, keep),
                         dict(prm, x=x), dout)
        cm = _row_rel(got["cmap"][:, :K], keep["m"].detach().reshape(B * n, K))
        errs = [("cmap per patch row", float(cm.max()), SEG_FWD),
                ("out per row", float(_row_rel(got["out"], ref).max()), SEG_FWD),
                ("dP per patch row", float(_row_rel(got["dP"], keep["P"].grad.reshape(B * n, -1)).max()), SEG_BWD),
                ("dC per class row", float(_row_rel(got["dC"], keep["C"].grad.reshape(B * K, -1)).max()), SEG_BWD),
                ("dx per patch row", float(_row_rel(got["dx"][:, :n], rg["x"][:, :n]).max()), SEG_BWD),
                ("dx per class row", float(_row_rel(got["dx"][:, n:], rg["x"][:, n:]).max()), SEG_BWD)]
        for k in SG.TAIL_PARAMS:
            if k in ("patch_w", "classes_w"):
                errs.append((k + " row", float(_row_rel(got[k], rg[k]).max()), SEG_BWD))
            else:
                errs.append((k + " element", _elem_rel(got[k], rg[k]), SEG_BWD))
        return errs, float(cm.max()) / SEG_FWD

    errs, _ = checks(None)
    frac = _report("segmenter tail %s" % case, errs)
    assert frac <= 1.0, [e for e in errs if e[1] > e[2]]
    if zero_row:
        assert float(got["dP"][5].abs().max()) > 1e6         # the clamped row norm 1e-12 scales its gradient up
    if case == "k65":
        _, miss = checks("ln_over_patches")
        print("  wrong reference ln_over_patches: %.1f x budget per patch row" % miss)
        assert miss >= 10.0, miss


def test_segmenter_tail_weight_mirror(dev):
    """patch_proj / classes_proj weights in a registered bf16 mirror against the cast path, same inputs and priors"""
    case = "k65"
    x, prm, dout, priors = _seg_inputs(case, dev, 54)
    cast1 = _seg_tail_call(dev, case, x, prm, dout, priors)
    cast2 = _seg_tail_call(dev, case, x, prm, dout, priors)
    mir = _Mirror([_f32(prm["patch_w"]), _f32(prm["classes_w"])], dev)
    try:
        mirrored = _seg_tail_call(dev, case, x, prm, dout, priors, mir)
    finally:
        mir.close()
    print("segmenter mirror: %s" % ", ".join("%s %s" % (k, _same_bits(k, cast1[k], cast2[k], mirrored[k])) for k in cast1))


@pytest.mark.parametrize("case", ["ade_n1024_k150", "nyu_n1280_k41", "n12"])
def test_segmenter_proj_exact(dev, case):
    """gather + proj_dec GEMM + class tokens, and the backward's scatter and d_cls column sums, on dyadic inputs"""
    B, nh, nw, K, _ = SEG_CASES[case]
    n, E = nh * nw, SEG_E
    T = 2 if case.startswith("nyu") else 1
    starts = [2 * n, 0] if T == 2 else [n]
    N = 3 * n + 1
    gen = torch.Generator().manual_seed(55)
    lib, st = L.lib(), L.current_stream()
    enc, w, b = _dy((B, N, D_ENC), 3, gen, dev), _dy((E, T * D_ENC), 4, gen, dev), _dy((E,), 4, gen, dev)
    cls, dseq = _dy((K, E), 4, gen, dev), _dy((B, n + K, E), 4, gen, dev)
    pw, pb, pc = _dy(w.shape, 4, gen, dev), _dy(b.shape, 4, gen, dev), _dy(cls.shape, 4, gen, dev)
    st_arr = (ctypes.c_int * T)(*starts)
    bufs = {"saved": _Guarded((lib.mmae_segmenter_proj_saved_bytes(B, n, T * D_ENC, E),), torch.uint8, dev),
            "ws": _Guarded((lib.mmae_segmenter_proj_workspace_bytes(B, n, T * D_ENC, E),), torch.uint8, dev),
            "seq": _Guarded((B, n + K, E), torch.float32, dev), "denc": _Guarded((B, N, D_ENC), torch.float32, dev),
            "d_w": _Guarded(w.shape, torch.float32, dev, pw), "d_b": _Guarded(b.shape, torch.float32, dev, pb),
            "d_cls": _Guarded(cls.shape, torch.float32, dev, pc)}
    enc32, w32, b32, c32, ds32 = _f32(enc), _f32(w), _f32(b), _f32(cls), _f32(dseq)
    L.check(lib.mmae_segmenter_proj_forward(enc32.data_ptr(), B, N, D_ENC, n, T, st_arr, E, K, w32.data_ptr(), b32.data_ptr(),
                                            c32.data_ptr(), bufs["seq"].ptr(), bufs["saved"].ptr(), bufs["ws"].ptr(), st),
            "segmenter proj forward")
    bufs["ws"].fill()
    L.check(lib.mmae_segmenter_proj_backward(ds32.data_ptr(), B, N, D_ENC, n, T, st_arr, E, K, w32.data_ptr(),
                                             bufs["d_w"].ptr(), bufs["d_b"].ptr(), bufs["d_cls"].ptr(), bufs["denc"].ptr(),
                                             bufs["saved"].ptr(), bufs["ws"].ptr(), st), "segmenter proj backward")
    torch.cuda.synchronize()
    _guards("segmenter proj " + case, bufs)
    fn = lambda enc, w, b, cls: SG.proj(enc, w, b, cls, starts, n)
    ins = {"enc": enc, "w": w, "b": b, "cls": cls}
    ref, rg = _grads(fn, ins, dseq)
    aref, ag = _grads(fn, {k: v.abs() for k, v in ins.items()}, dseq.abs())
    kinds = [_check_exact("seq", bufs["seq"].t, ref, aref, 7, T * D_ENC + 1),
             _check_exact("denc", bufs["denc"].t, rg["enc"], ag["enc"], 8, E),
             _check_exact("d_w", bufs["d_w"].t.double() - pw, rg["w"], ag["w"] + pw.abs(), 7, B * n + 1),
             _check_exact("d_b", bufs["d_b"].t.double() - pb, rg["b"], ag["b"] + pb.abs(), 4, B * n + 1),
             _check_exact("d_cls", bufs["d_cls"].t.double() - pc, rg["cls"], ag["cls"] + pc.abs(), 4, B + 1)]
    print("segmenter proj exact %s: %s" % (case, " ".join(kinds)))
    assert kinds == ["exact"] * 5, kinds
    tok = torch.ones(N, dtype=torch.bool, device=dev)
    for s0 in starts:
        tok[s0:s0 + n] = False
    assert not bool(bufs["denc"].t[:, tok].any())            # other tasks' tokens and the global token: exactly 0
