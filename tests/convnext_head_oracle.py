"""Restatement of the semantic-segmentation head of fine-tuning for the tests: ConvNeXtAdapter.forward
(multimae/output_adapters.py:545-573) with ConvNeXtBlock (multimae/output_adapter_utils.py:47-57), on top of the oracle
encoder of cls_head_oracle.encoder_tokens, as a composition of one function per C entry point (proj, block, tail).  Also
the model and values of the convnext_head.pt fixture."""
import math
from functools import partial

import torch
import torch.nn.functional as F

from helpers import formula_fill_
from pretrain_io_oracle import _ln, gelu, rf, roundings

# convnext_head.pt: MultiViT (dim 128, depth 2, 2 heads) on rgb + depth at 48 x 64 (3 x 4 patches), B = 2, with two heads:
# 16 predictions per patch over both tasks' tokens (C = 128, upsample x4) and 4 per patch over rgb (C = 512, upsample x8)
CONFIG = dict(in_domains=["rgb", "depth"], B=2, H=48, W=64, dim=128, depth=2, heads=2,
              adapters={"semseg": dict(num_classes=5, embed_dim=2048, preds_per_patch=16, depth=2, main_tasks=["rgb", "depth"]),
                        "aux": dict(num_classes=8, embed_dim=2048, preds_per_patch=4, depth=1, main_tasks=["rgb"])})


def build(MultiViT, Patched, ConvNeXtAdapter, c=CONFIG):
    """The fixture's model from the given classes (the reference's, or this package's)."""
    ins = {"rgb": Patched(num_channels=3, stride_level=1, patch_size_full=16, image_size=(c["H"], c["W"])),
           "depth": Patched(num_channels=1, stride_level=1, patch_size_full=16, image_size=(c["H"], c["W"]))}
    outs = {k: ConvNeXtAdapter(**v) for k, v in c["adapters"].items()}
    return MultiViT(ins, outs, num_global_tokens=1, dim_tokens=c["dim"], depth=c["depth"], num_heads=c["heads"], mlp_ratio=4,
                    qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def fill_(named_params):
    """formula_fill_ values (non-zero biases), with the ConvNeXt blocks' LayerNorm weights moved to around 1."""
    named_params = list(named_params)
    formula_fill_(named_params)
    with torch.no_grad():
        for n, p in named_params:
            if ".blocks." in n and n.endswith(".norm.weight"):
                p.add_(1.0)


def inputs(c=CONFIG, seed=5):
    """Images and labels [B, H, W] (class ids, with about 10 % ignored pixels = 255) of each head."""
    g = torch.Generator().manual_seed(seed)
    x = {"rgb": torch.randn(c["B"], 3, c["H"], c["W"], generator=g), "depth": torch.randn(c["B"], 1, c["H"], c["W"], generator=g)}
    labels = {}
    for k, a in c["adapters"].items():
        lab = torch.randint(0, a["num_classes"], (c["B"], c["H"], c["W"]), generator=g)
        lab[torch.rand(lab.shape, generator=g) < 0.1] = 255
        labels[k] = lab
    return x, labels


def seg_loss(outs, labels):
    """Sum over the heads of CrossEntropyLoss(ignore_index=255) (the criterion of run_finetuning_semseg.py)."""
    return sum(F.cross_entropy(outs[k], labels[k].to(outs[k].device), ignore_index=255) for k in labels)


# ----------------------------------------------------------------------------------------------- entry-point parts
# One function per entry point of convnext_head.cu (tests/test_cuda_heads.py), in the kernels' layout: the feature map is the
# [P, C] view of the proj_dec output, row (b*n + t)*s*s + a*s + c' = pixel ((t / nw)*s + a, (t % nw)*s + c') of sample b;
# geo = (B, nh, nw, s).  round=True: float64 with a bf16 rounding wherever the kernels store bf16 (pretrain_io_oracle's rf on
# values, rb on gradient operands), round=False: plain float64.  Bias gradients are column sums of the fp32 gradient, taken
# before its bf16 cast (mmae_cast_colsum_f32), except pwconv1's: mmae_dgelu_colsum_bf16 sums the stored bf16 dz.  The
# dwconv, LayerNorm statistics, upsample, gather / scatter and the residual stream are fp32 in the kernels, unrounded here.
#
# `mutate` names a deliberately wrong variant for the sensitivity checks:
#   "tasks_reversed"   proj: the main tasks' tokens concatenated in reverse order;
#   "pixel_transpose"  block: pixel (a, c') of each patch taken for (c', a), i.e. "(pw ph c)" instead of "(ph pw c)";
#   "flip_fwd"         block: the 7x7 kernel flipped in the forward dwconv;
#   "flip_bwd"         block: the 7x7 kernel flipped in the input gradient's transposed dwconv only;
#   "replicate_pad"    block: replicate instead of zero padding at the map borders;
#   "neighbour_sample" block: the dwconv of every sample reads the previous sample's map;
#   "align_corners"    tail: bilinear with align_corners=True;
#   "no_clamp"         tail: negative source coordinates not clamped to 0 (truncated toward 0, weights outside [0, 1]);
#   "class_shift"      tail: output plane k is upsampled from class k + 1 of the class map.
MUTATIONS = ("tasks_reversed", "pixel_transpose", "flip_fwd", "flip_bwd", "replicate_pad", "neighbour_sample",
             "align_corners", "no_clamp", "class_shift")
BLOCK_PARAMS = ["dw_w", "dw_b", "norm_w", "norm_b", "pw1_w", "pw1_b", "pw2_w", "pw2_b"]   # the C ABI's pointer order


def rows_to_image(x, geo, mutate=None):
    """[P, C] rows -> [B, C, nh*s, nw*s]"""
    B, nh, nw, s = geo
    x = x.reshape(B, nh, nw, s, s, x.shape[-1])
    if mutate == "pixel_transpose":
        x = x.transpose(3, 4)
    return x.permute(0, 5, 1, 3, 2, 4).reshape(B, -1, nh * s, nw * s)


def image_to_rows(img, geo, mutate=None):
    """[B, C, nh*s, nw*s] -> [P, C] rows (the inverse of rows_to_image)"""
    B, nh, nw, s = geo
    x = img.reshape(B, -1, nh, s, nw, s).permute(0, 2, 4, 3, 5, 1)
    if mutate == "pixel_transpose":
        x = x.transpose(3, 4)
    return x.reshape(-1, img.shape[1])


def proj(enc, w, b, starts, n, round=True, mutate=None):
    """mmae_convnext_proj_*: enc [B, N, D] -> [B, n, E] (the [P, C] rows, reshaped)"""
    rf_, rb_ = roundings(round)
    order = starts[::-1] if mutate == "tasks_reversed" else starts
    a = torch.cat([enc[:, s0:s0 + n] for s0 in order], dim=-1)
    return rb_(rf_(a) @ rf_(w).t()) + b


def dwconv(img, w, b, mutate=None):
    """nn.Conv2d(C, C, 7, padding=3, groups=C) on [B, C, Hf, Wf]"""
    C = img.shape[1]
    if mutate == "neighbour_sample":
        img = torch.roll(img, 1, 0)
    if mutate == "replicate_pad":
        return F.conv2d(F.pad(img, (3, 3, 3, 3), mode="replicate"), w, b, groups=C)
    if mutate == "flip_fwd":
        return F.conv2d(img, w.flip(-1, -2), b, padding=3, groups=C)
    if mutate == "flip_bwd":                  # the value of the true conv; the input gradient through the flipped kernel
        d1 = F.conv2d(img, w.detach().flip(-1, -2), None, padding=3, groups=C)
        return F.conv2d(img.detach(), w, b, padding=3, groups=C) + d1 - d1.detach()
    return F.conv2d(img, w, b, padding=3, groups=C)


def block(x, prm, geo, eps=1e-6, round=True, fuse_gelu=False, mutate=None):
    """mmae_convnext_block_*: x [P, C] -> x + pwconv2(GELU(pwconv1(LN(dwconv7x7(x))))).  prm: BLOCK_PARAMS names, dw_w
    [C, 1, 7, 7].  GELU as block_oracle: the streaming kernel on the stored bf16 z, or (fuse_gelu) in the fc1 epilogue."""
    rf_, rb_ = roundings(round)
    d = image_to_rows(dwconv(rows_to_image(x, geo, mutate), prm["dw_w"], prm["dw_b"], mutate), geo, mutate)
    h = rb_(rf_(_ln(d, prm["norm_w"], prm["norm_b"], eps)))
    zp = h @ rf_(prm["pw1_w"]).t() + prm["pw1_b"]
    z = rb_(rf_(zp))
    if fuse_gelu and round:
        gz = gelu(z)
        a = rf(gelu(zp).detach() + gz - gz.detach())
    else:
        a = rb_(rf_(gelu(z)))
    return x + (rb_(a @ rf_(prm["pw2_w"]).t()) + prm["pw2_b"])


def interp_matrix(out, inp, mutate=None, dtype=torch.float64, device=None):
    """[out, inp] weights of F.interpolate(mode="bilinear") along one axis, as ATen forms them: src = max(0, (dst + 0.5)
    in / out - 0.5), i0 = int(src), i1 = i0 + (i0 < in - 1), lambda = src - i0."""
    dst = torch.arange(out, dtype=torch.float64)
    if mutate == "align_corners":
        src = dst * ((inp - 1) / (out - 1) if out > 1 else 0.0)
    else:
        src = (dst + 0.5) * (inp / out) - 0.5
        if mutate != "no_clamp":
            src = src.clamp_min(0.0)
    i0 = src.trunc().long()
    i1 = torch.where(i0 < inp - 1, i0 + 1, i0)
    l1 = src - i0
    m = torch.zeros(out, inp, dtype=torch.float64)
    rows = torch.arange(out)
    m.index_put_((rows, i0), 1.0 - l1, accumulate=True)
    m.index_put_((rows, i1), l1, accumulate=True)
    return m.to(dtype=dtype, device=device)


def upsample(img, H, W, mutate=None):
    """F.interpolate(img, (H, W), mode="bilinear", align_corners=False) of [B, K, h, w]"""
    my = interp_matrix(H, img.shape[2], mutate, img.dtype, img.device)
    mx = interp_matrix(W, img.shape[3], mutate, img.dtype, img.device)
    return torch.einsum("yi,bkij,xj->bkyx", my, img, mx)


def tail(x, w, b, geo, H, W, round=True, mutate=None):
    """mmae_convnext_tail_*: x [P, C], w [K, C] -> [B, K, H, W] (final_layer, then the upsample)"""
    rf_, rb_ = roundings(round)
    cmap = rows_to_image(rb_(rf_(x) @ rf_(w).t()) + b, geo)
    if mutate == "class_shift":
        cmap = torch.roll(cmap, -1, 1)
    return upsample(cmap, H, W, mutate)


def block_params(p, q):
    """BLOCK_PARAMS of the ConvNeXtBlock with state-dict prefix q"""
    names = ["dwconv.weight", "dwconv.bias", "norm.weight", "norm.bias", "pwconv1.weight", "pwconv1.bias", "pwconv2.weight",
             "pwconv2.bias"]
    return {k: p[q + nm] for k, nm in zip(BLOCK_PARAMS, names)}


def convnext_head(enc, p, starts, n, H, W, preds_per_patch, depth, patch=16, eps=1e-6, prefix="output_adapters.semseg.",
                  round=False):
    """enc [B, N, D] -> [B, K, H, W]; `starts`: first token of each main task, `n` tokens per task.  proj -> block x depth
    -> tail ("b n (p c) -> b (n p) c" then "b (nh nw ph pw) c -> b c (nh ph) (nw pw)" is the rows layout)."""
    geo = (enc.shape[0], H // patch, W // patch, int(math.isqrt(preds_per_patch)))
    x = proj(enc, p[prefix + "proj_dec.weight"], p[prefix + "proj_dec.bias"], starts, n, round)
    x = x.reshape(-1, x.shape[-1] // preds_per_patch)
    for i in range(depth):
        x = block(x, block_params(p, "%sblocks.%d." % (prefix, i)), geo, eps, round)
    return tail(x, p[prefix + "final_layer.weight"].flatten(1), p[prefix + "final_layer.bias"], geo, H, W, round)
