"""CPU: the float64 references of the fine-tuning heads' entry points (convnext_head_oracle.proj / block / tail,
segmenter_head_oracle.proj / tail, cls_head_oracle.head), which tests/test_cuda_heads.py holds the kernels to.

1. round=False: each part, and their composition, against autograd of the module's arithmetic restated with torch's own
   operators in the image layout (F.conv2d with padding, F.layer_norm, F.gelu, F.interpolate), value and every gradient,
   to 1e-12.
2. round=True differs from round=False, by O(u) (u = 2^-8, bf16's unit roundoff).
3. Every deliberately wrong variant (`mutate`) differs from the right one."""
import math

import pytest
import torch
import torch.nn.functional as F

import cls_head_oracle as CH
import convnext_head_oracle as CX
import segmenter_head_oracle as SG

U = 2.0 ** -8


def _leaves(d):
    return {k: v.detach().clone().requires_grad_(True) for k, v in d.items()}


def _run(fn, inputs, dout_seed=0):
    """fn(**leaves) -> out; returns (out, {name: grad}) for a seeded random output gradient"""
    lv = _leaves(inputs)
    out = fn(**lv)
    g = torch.Generator().manual_seed(dout_seed)
    out.backward(torch.randn(out.shape, generator=g, dtype=out.dtype))
    return out.detach(), {k: v.grad for k, v in lv.items()}


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _assert_close(got, ref, tol, what):
    (o1, g1), (o2, g2) = got, ref
    assert _rel(o1, o2) <= tol, (what, "out", _rel(o1, o2))
    for k in g2:
        if g2[k] is not None:
            assert _rel(g1[k], g2[k]) <= tol, (what, k, _rel(g1[k], g2[k]))


def _r(gen, *shape, scale=1.0):
    return scale * torch.randn(*shape, generator=gen, dtype=torch.float64)


# ------------------------------------------------------------------------------------------------------------- ConvNeXt
GEOS = {"square_s4": (2, 3, 3, 4), "ragged_3x5_s4": (3, 3, 5, 4), "s2": (2, 4, 3, 2), "s1": (2, 5, 4, 1),
        "s8": (2, 2, 2, 8)}


def _block_inputs(geo, C, gen):
    B, nh, nw, s = geo
    P = B * nh * nw * s * s
    prm = {"dw_w": _r(gen, C, 1, 7, 7, scale=0.2), "dw_b": _r(gen, C, scale=0.1), "norm_w": 1 + _r(gen, C, scale=0.1),
           "norm_b": _r(gen, C, scale=0.1), "pw1_w": _r(gen, 4 * C, C, scale=C ** -0.5), "pw1_b": _r(gen, 4 * C, scale=0.1),
           "pw2_w": _r(gen, C, 4 * C, scale=(4 * C) ** -0.5), "pw2_b": _r(gen, C, scale=0.1)}
    return dict(prm, x=_r(gen, P, C))


def _block_torch(x, dw_w, dw_b, norm_w, norm_b, pw1_w, pw1_b, pw2_w, pw2_b, geo, eps=1e-6):
    """ConvNeXtBlock in the image layout (output_adapter_utils.py:47-57) on the rows rearranged by einops' pattern"""
    B, nh, nw, s = geo
    C = x.shape[1]
    img = x.reshape(B, nh * nw, s * s * C).reshape(B, nh, nw, s, s, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, nh * s, nw * s)
    y = F.conv2d(img, dw_w, dw_b, padding=3, groups=C).permute(0, 2, 3, 1)
    y = F.layer_norm(y, (C,), norm_w, norm_b, eps)
    y = F.linear(F.gelu(F.linear(y, pw1_w, pw1_b)), pw2_w, pw2_b)
    out = img + y.permute(0, 3, 1, 2)
    return out.reshape(B, C, nh, s, nw, s).permute(0, 2, 4, 3, 5, 1).reshape(-1, C)


def _tail_torch(x, w, b, geo, H, W):
    B, nh, nw, s = geo
    K, C = w.shape
    img = x.reshape(B, nh, nw, s, s, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, nh * s, nw * s)
    return F.interpolate(F.conv2d(img, w[:, :, None, None], b), size=(H, W), mode="bilinear", align_corners=False)


@pytest.mark.parametrize("geo", list(GEOS))
def test_block_plain_matches_torch(geo):
    g = GEOS[geo]
    inp = _block_inputs(g, 32, torch.Generator().manual_seed(1))
    got = _run(lambda x, **p: CX.block(x, p, g, round=False), inp)
    ref = _run(lambda **a: _block_torch(geo=g, **a), inp)
    _assert_close(got, ref, 1e-12, geo)


@pytest.mark.parametrize("geo", list(GEOS))
def test_tail_plain_matches_torch(geo):
    g = GEOS[geo]
    B, nh, nw, s = g
    gen = torch.Generator().manual_seed(2)
    H, W = nh * 16, nw * 16
    inp = {"x": _r(gen, B * nh * nw * s * s, 32), "w": _r(gen, 13, 32), "b": _r(gen, 13)}
    got = _run(lambda x, w, b: CX.tail(x, w, b, g, H, W, round=False), inp)
    ref = _run(lambda x, w, b: _tail_torch(x, w, b, g, H, W), inp)
    _assert_close(got, ref, 1e-12, geo)


def test_proj_plain_matches_torch():
    gen = torch.Generator().manual_seed(3)
    B, N, D, n, E = 2, 2 * 12 + 1, 16, 12, 64
    inp = {"enc": _r(gen, B, N, D), "w": _r(gen, E, 2 * D), "b": _r(gen, E)}
    got = _run(lambda enc, w, b: CX.proj(enc, w, b, [0, n], n, round=False), inp)
    ref = _run(lambda enc, w, b: F.linear(torch.cat([enc[:, :n], enc[:, n:2 * n]], -1), w, b), inp)
    _assert_close(got, ref, 1e-12, "proj")
    assert not bool(got[1]["enc"][:, 2 * n:].any())            # the global token gets no gradient


def test_head_composition_matches_torch():
    """convnext_head (proj -> blocks -> tail) against the whole head in the image layout, on a non-square map"""
    gen = torch.Generator().manual_seed(4)
    B, nh, nw, s, C, K, D = 2, 2, 3, 4, 32, 5, 16
    n = nh * nw
    pre = "h."
    p = {pre + "proj_dec.weight": _r(gen, s * s * C, 2 * D, scale=0.2), pre + "proj_dec.bias": _r(gen, s * s * C, scale=0.1),
         pre + "final_layer.weight": _r(gen, K, C, 1, 1), pre + "final_layer.bias": _r(gen, K)}
    for i in range(2):
        bp = _block_inputs((B, nh, nw, s), C, gen)
        for k, nm in zip(CX.BLOCK_PARAMS, ["dwconv.weight", "dwconv.bias", "norm.weight", "norm.bias", "pwconv1.weight",
                                           "pwconv1.bias", "pwconv2.weight", "pwconv2.bias"]):
            p["%sblocks.%d.%s" % (pre, i, nm)] = bp[k]
    inp = dict(p, enc=_r(gen, B, 2 * n + 1, D))

    def torch_head(enc, **q):
        x = F.linear(torch.cat([enc[:, n:2 * n], enc[:, :n]], -1), q[pre + "proj_dec.weight"], q[pre + "proj_dec.bias"])
        x = x.reshape(-1, C)
        for i in range(2):
            bq = "%sblocks.%d." % (pre, i)
            x = _block_torch(x, *[q[bq + nm] for nm in ["dwconv.weight", "dwconv.bias", "norm.weight", "norm.bias",
                                                        "pwconv1.weight", "pwconv1.bias", "pwconv2.weight",
                                                        "pwconv2.bias"]], geo=(B, nh, nw, s))
        return _tail_torch(x, q[pre + "final_layer.weight"].flatten(1), q[pre + "final_layer.bias"], (B, nh, nw, s),
                           nh * 16, nw * 16)

    got = _run(lambda enc, **q: CX.convnext_head(enc, q, [n, 0], n, nh * 16, nw * 16, s * s, 2, prefix=pre), inp)
    ref = _run(torch_head, inp)
    _assert_close(got, ref, 1e-12, "composition")


def test_interp_weights_dyadic():
    """r = 16 / s a power of two: every bilinear weight is a multiple of 1 / (2r)"""
    for s in (1, 2, 4, 8):
        r = 16 // s
        m = CX.interp_matrix(7 * s * r, 7 * s)
        assert torch.equal(m * 2 * r, torch.round(m * 2 * r)), s
        assert torch.allclose(m.sum(1), torch.ones(m.shape[0], dtype=torch.float64), rtol=0, atol=0)


def _rounding_gap(fn, inp):
    """relative differences (out, then every gradient in input order) between round=True and round=False; a bias gradient
    that is a column sum of the fp32 output gradient has none"""
    a, b = _run(lambda **q: fn(True, **q), inp), _run(lambda **q: fn(False, **q), inp)
    return [_rel(a[0], b[0])] + [_rel(a[1][k], b[1][k]) for k in b[1]]


def test_convnext_rounding_is_order_u():
    gen = torch.Generator().manual_seed(5)
    g = GEOS["ragged_3x5_s4"]
    B, nh, nw, s = g
    binp = _block_inputs(g, 32, gen)
    for fuse in (False, True):
        gaps = _rounding_gap(lambda rnd, x, **p: CX.block(x, p, g, round=rnd, fuse_gelu=fuse), binp)
        assert gaps[0] > 0 and gaps[1] > 0 and max(gaps) < 8 * U, (fuse, gaps)
    tinp = {"x": binp["x"], "w": _r(gen, 13, 32), "b": _r(gen, 13)}
    gaps = _rounding_gap(lambda rnd, x, w, b: CX.tail(x, w, b, g, 48, 80, round=rnd), tinp)
    assert min(gaps[:3]) > 0 and max(gaps) < 8 * U, gaps
    pinp = {"enc": _r(gen, B, 2 * 15 + 1, 16), "w": _r(gen, 512, 32), "b": _r(gen, 512)}
    gaps = _rounding_gap(lambda rnd, enc, w, b: CX.proj(enc, w, b, [0, 15], 15, round=rnd), pinp)
    assert min(gaps[:3]) > 0 and max(gaps) < 8 * U, gaps


@pytest.mark.parametrize("mutate", CX.MUTATIONS)
def test_convnext_mutations_differ(mutate):
    gen = torch.Generator().manual_seed(6)
    g = GEOS["ragged_3x5_s4"]
    B, nh, nw, s = g
    binp = _block_inputs(g, 32, gen)
    if mutate == "tasks_reversed":
        inp = {"enc": _r(gen, B, 2 * 15 + 1, 16), "w": _r(gen, 512, 32), "b": _r(gen, 512)}
        fn = lambda m, enc, w, b: CX.proj(enc, w, b, [0, 15], 15, mutate=m)
    elif mutate in ("align_corners", "no_clamp", "class_shift"):
        inp = {"x": binp["x"], "w": _r(gen, 13, 32), "b": _r(gen, 13)}
        fn = lambda m, x, w, b: CX.tail(x, w, b, g, 48, 80, mutate=m)
    else:
        inp = binp
        fn = lambda m, x, **p: CX.block(x, p, g, mutate=m)
    right, wrong = _run(lambda **q: fn(None, **q), inp), _run(lambda **q: fn(mutate, **q), inp)
    if mutate == "flip_bwd":                       # the value is right, the input gradient is not
        assert torch.equal(right[0], wrong[0])
        assert _rel(wrong[1]["x"], right[1]["x"]) > 1e-2
    else:
        assert _rel(wrong[0], right[0]) > 1e-3, mutate


# ---------------------------------------------------------------------------------------------------------- cls head
@pytest.mark.parametrize("mean_pool", [True, False])
@pytest.mark.parametrize("C", [37, 0])
def test_cls_head_plain_matches_torch(mean_pool, C):
    gen = torch.Generator().manual_seed(7)
    B, N, D = 3, 9, 64
    inp = {"enc": _r(gen, B, N, D), "nw": 1 + _r(gen, D, scale=0.1), "nb": _r(gen, D, scale=0.1)}
    if C:
        inp.update(hw=_r(gen, C, D, scale=D ** -0.5), hb=_r(gen, C, scale=0.1))

    def torch_head(enc, nw, nb, hw=None, hb=None):
        x = F.layer_norm(enc.mean(1) if mean_pool else enc[:, -1], (D,), nw, nb, 1e-6)
        return x if hw is None else F.linear(x, hw, hb)

    got = _run(lambda enc, nw, nb, hw=None, hb=None: CH.head(enc, nw, nb, hw, hb, mean_pool), inp)
    ref = _run(torch_head, inp)
    _assert_close(got, ref, 1e-12, (mean_pool, C))
    if C:
        gaps = _rounding_gap(lambda rnd, enc, nw, nb, hw, hb: CH.head(enc, nw, nb, hw, hb, mean_pool, round=rnd), inp)
        assert gaps[0] > 0 and max(gaps) < 8 * U, gaps
    if mean_pool:
        wrong = _run(lambda enc, nw, nb, hw=None, hb=None: CH.head(enc, nw, nb, hw, hb, mean_pool, mutate="mean_short"), inp)
        assert _rel(wrong[0], ref[0]) > 1e-3
    else:
        assert not bool(got[1]["enc"][:, :-1].any())


def test_cls_head_composition():
    """cls_head (the state-dict form) is head()"""
    gen = torch.Generator().manual_seed(8)
    p = {"c.norm.weight": _r(gen, 32), "c.norm.bias": _r(gen, 32), "c.head.weight": _r(gen, 5, 32), "c.head.bias": _r(gen, 5)}
    enc = _r(gen, 2, 4, 32)
    assert torch.equal(CH.cls_head(enc, p, prefix="c."), CH.head(enc, *p.values()))
    assert math.isfinite(float(CH.cls_head(enc, {k: v for k, v in p.items() if "head" not in k}, prefix="c.").sum()))


# --------------------------------------------------------------------------------------------------------- Segmenter
def _seg_inputs(B, n, K, E, gen):
    return {"x": _r(gen, B, n + K, E), "dec_w": 1 + _r(gen, E, scale=0.1), "dec_b": _r(gen, E, scale=0.1),
            "patch_w": _r(gen, E, E, scale=E ** -0.5), "classes_w": _r(gen, E, E, scale=E ** -0.5),
            "mask_w": 1 + _r(gen, K, scale=0.1), "mask_b": _r(gen, K, scale=0.1)}


def _seg_tail_torch(x, dec_w, dec_b, patch_w, classes_w, mask_w, mask_b, nh, nw, eps=1e-6):
    """SegmenterMaskTransformerAdapter.forward after the blocks (output_adapters.py:463-476) with torch's operators"""
    n, E = nh * nw, x.shape[-1]
    y = F.layer_norm(x, (E,), dec_w, dec_b, eps)
    P, C = F.normalize(F.linear(y[:, :n], patch_w), dim=2), F.normalize(F.linear(y[:, n:], classes_w), dim=2)
    m = F.layer_norm(P @ C.transpose(1, 2), (mask_w.shape[0],), mask_w, mask_b, eps)
    return F.interpolate(m.transpose(1, 2).reshape(x.shape[0], -1, nh, nw), size=(nh * 16, nw * 16), mode="bilinear",
                         align_corners=False)


@pytest.mark.parametrize("nh,nw,K", [(3, 4, 9), (2, 5, 13)])
def test_segmenter_tail_plain_matches_torch(nh, nw, K):
    inp = _seg_inputs(2, nh * nw, K, 64, torch.Generator().manual_seed(9))
    got = _run(lambda x, **p: SG.tail(x, p, nh, nw, nh * 16, nw * 16, round=False), inp)
    ref = _run(lambda **a: _seg_tail_torch(nh=nh, nw=nw, **a), inp)
    _assert_close(got, ref, 1e-12, (nh, nw, K))


def test_segmenter_proj_plain_matches_torch():
    gen = torch.Generator().manual_seed(10)
    B, n, D, E, K = 2, 6, 16, 32, 9
    inp = {"enc": _r(gen, B, 2 * n + 1, D), "w": _r(gen, E, 2 * D), "b": _r(gen, E), "cls": _r(gen, K, E)}
    got = _run(lambda enc, w, b, cls: SG.proj(enc, w, b, cls, [n, 0], n, round=False), inp)
    ref = _run(lambda enc, w, b, cls: torch.cat([F.linear(torch.cat([enc[:, n:2 * n], enc[:, :n]], -1), w, b),
                                                 cls.expand(B, -1, -1)], 1), inp)
    _assert_close(got, ref, 1e-12, "segmenter proj")


def test_segmenter_rounding_and_mutation():
    nh, nw, K = 3, 4, 9
    inp = _seg_inputs(2, nh * nw, K, 64, torch.Generator().manual_seed(11))
    gaps = _rounding_gap(lambda rnd, x, **p: SG.tail(x, p, nh, nw, 48, 64, round=rnd), inp)
    assert gaps[0] > 0 and gaps[1] > 0 and max(gaps) < 8 * U, gaps
    right = _run(lambda x, **p: SG.tail(x, p, nh, nw, 48, 64), inp)
    wrong = _run(lambda x, **p: SG.tail(x, p, nh, nw, 48, 64, mutate="ln_over_patches"), inp)
    assert _rel(wrong[0], right[0]) > 1e-2
