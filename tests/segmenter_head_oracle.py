"""fp32 restatement of the Segmenter head of semantic-segmentation fine-tuning for the tests:
SegmenterMaskTransformerAdapter.forward (multimae/output_adapters.py:450-478), on top of the oracle encoder of
cls_head_oracle.encoder_tokens.  Also the model and values of the segmenter_head.pt fixture."""
from functools import partial

import torch
import torch.nn.functional as F

import convnext_head_oracle as CX
from convnext_head_oracle import inputs as _inputs
from convnext_head_oracle import seg_loss  # noqa: F401  (re-exported: the criterion of run_finetuning_semseg.py)
from helpers import formula_fill_
from pretrain_io_oracle import _ln, roundings

# segmenter_head.pt: MultiViT (dim 128, depth 2, 2 heads) on rgb + depth at 48 x 64 (3 x 4 patches), B = 2, with two heads
# of width 128: 9 classes over both tasks' tokens (depth 2, 4 heads of 32) and 13 classes over rgb (depth 1, 2 heads of 64)
CONFIG = dict(in_domains=["rgb", "depth"], B=2, H=48, W=64, dim=128, depth=2, heads=2,
              adapters={"semseg": dict(num_classes=9, embed_dim=128, depth=2, num_heads=4, drop_path_rate=0.0,
                                       main_tasks=["rgb", "depth"]),
                        "aux": dict(num_classes=13, embed_dim=128, depth=1, num_heads=2, drop_path_rate=0.0,
                                    main_tasks=["rgb"])})


def build(MultiViT, Patched, Adapter, c=CONFIG):
    """The fixture's model from the given classes (the reference's, or this package's)."""
    ins = {"rgb": Patched(num_channels=3, stride_level=1, patch_size_full=16, image_size=(c["H"], c["W"])),
           "depth": Patched(num_channels=1, stride_level=1, patch_size_full=16, image_size=(c["H"], c["W"]))}
    outs = {k: Adapter(**v) for k, v in c["adapters"].items()}
    return MultiViT(ins, outs, num_global_tokens=1, dim_tokens=c["dim"], depth=c["depth"], num_heads=c["heads"], mlp_ratio=4,
                    qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def fill_(named_params):
    """formula_fill_ values (non-zero biases) with the heads' LayerNorm weights moved to around 1; the heads' matrices and
    class tokens are seeded normal draws instead (fan-in scaling; class tokens at 0.5).  formula_fill_'s smooth patterns make
    the heads' matrices nearly low-rank, and the cosine + class LayerNorm then turns the 1e-2 that bf16 blocks differ by into
    tens of percent - in any half-precision arithmetic, the reference's own under autocast included - so such a fixture
    could only be checked in fp32.  Class tokens that differ from each other, as trained ones do, keep the class map's
    spread over the classes (what mask_norm divides by) well above the rounding noise."""
    named_params = list(named_params)
    formula_fill_(named_params)
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for n, p in named_params:
            if not n.startswith("output_adapters."):
                continue
            if "norm" in n and n.endswith(".weight"):
                p.add_(1.0)
            elif n.endswith("cls_emb"):
                p.copy_(0.5 * torch.randn(p.shape, generator=g))
            elif n.endswith(".weight") and p.dim() == 2:
                p.copy_(torch.randn(p.shape, generator=g) / p.shape[1] ** 0.5)


def inputs(c=CONFIG, seed=5):
    return _inputs(c, seed)


def block(x, p, q, heads, eps=1e-6, s_attn=None, s_mlp=None):
    """Pre-LN transformer block with parameters p[q + ...]; s_attn / s_mlp: per-sample factors of stochastic depth."""
    B, T, E = x.shape
    h = F.layer_norm(x, (E,), p[q + "norm1.weight"], p[q + "norm1.bias"], eps)
    qkv = (h @ p[q + "attn.qkv.weight"].t() + p[q + "attn.qkv.bias"]).reshape(B, T, 3, heads, E // heads).permute(2, 0, 3, 1, 4)
    a = ((qkv[0] * (E // heads) ** -0.5) @ qkv[1].transpose(-2, -1)).softmax(-1)
    y = (a @ qkv[2]).transpose(1, 2).reshape(B, T, E) @ p[q + "attn.proj.weight"].t() + p[q + "attn.proj.bias"]
    x = x + (y if s_attn is None else y * s_attn.view(B, 1, 1))
    h = F.layer_norm(x, (E,), p[q + "norm2.weight"], p[q + "norm2.bias"], eps)
    y = F.gelu(h @ p[q + "mlp.fc1.weight"].t() + p[q + "mlp.fc1.bias"]) @ p[q + "mlp.fc2.weight"].t() + p[q + "mlp.fc2.bias"]
    return x + (y if s_mlp is None else y * s_mlp.view(B, 1, 1))


# ----------------------------------------------------------------------------------------------- entry-point parts
# One function per entry point of segmenter_head.cu (tests/test_cuda_heads.py).  round=True: float64 with a bf16 rounding
# wherever the kernels store bf16 (pretrain_io_oracle's rf on values, rb on gradient operands): the decoder_norm output
# Xpc (and its gradient dXpc), patch_proj / classes_proj weights, the projections' bf16 copies the mask kernel multiplies
# (seg_rownorm_kernel; the row norms come from the fp32 projections) and their gradients dP / dC.  Not mirrored: the mask
# backward's bf16 Gs = dM rp rc, and its normalise backward formed from the bf16 copies.  The proj GEMM is the ConvNeXt
# head's (convnext_head_oracle.proj); cls_emb, the class LayerNorm and the upsample are fp32.  round=False: plain float64.
# mutate="ln_over_patches": the class LayerNorm taken over the patches instead of the classes (the sensitivity checks).
TAIL_PARAMS = ["dec_w", "dec_b", "patch_w", "classes_w", "mask_w", "mask_b"]     # the C ABI's pointer order


def cosine_mask(P, C, gamma, beta, eps=1e-6, round=False, mutate=None):
    """LayerNorm over the classes of the cosine of every (patch, class) pair: P [B, n, E], C [B, K, E] -> [B, n, K]."""
    rf_, _ = roundings(round)
    m = (rf_(P) @ rf_(C).transpose(1, 2)) / P.norm(dim=2, keepdim=True).clamp_min(1e-12)
    m = m / C.norm(dim=2).clamp_min(1e-12).unsqueeze(1)
    if mutate == "ln_over_patches":
        return _ln(m.transpose(1, 2), 1.0, 0.0, eps).transpose(1, 2) * gamma + beta
    return _ln(m, gamma, beta, eps)


def proj(enc, w, b, cls_emb, starts, n, round=True):
    """mmae_segmenter_proj_*: enc [B, N, D] -> seq [B, n + K, E] (patch rows, then cls_emb)"""
    x = CX.proj(enc, w, b, starts, n, round)
    return torch.cat([x, cls_emb.expand(x.shape[0], -1, -1)], dim=1)


def tail(x, prm, nh, nw, H, W, eps_dec=1e-6, eps_mask=1e-6, round=True, mutate=None, keep=None):
    """mmae_segmenter_tail_*: x [B, n + K, E] -> [B, K, H, W].  prm: TAIL_PARAMS names.  keep: a dict that receives the
    projections P, C (retaining their gradients) and the class map m [B, n, K]."""
    rf_, rb_ = roundings(round)
    B, n = x.shape[0], nh * nw
    y = rb_(rf_(_ln(x, prm["dec_w"], prm["dec_b"], eps_dec)))
    P = rb_(y[:, :n] @ rf_(prm["patch_w"]).t())
    C = rb_(y[:, n:] @ rf_(prm["classes_w"]).t())
    m = cosine_mask(P, C, prm["mask_w"], prm["mask_b"], eps_mask, round, mutate)
    if keep is not None:
        P.retain_grad()
        C.retain_grad()
        keep.update(P=P, C=C, m=m)
    return CX.upsample(m.transpose(1, 2).reshape(B, -1, nh, nw), H, W)


def segmenter_head(enc, p, starts, n, H, W, depth, heads, patch=16, eps=1e-6, prefix="output_adapters.semseg.", scales=None):
    """enc [B, N, D] -> [B, K, H, W]; `starts`: first token of each main task, `n` tokens per task; `scales`: per block
    (s_attn, s_mlp) or None.  proj -> transformer blocks -> tail."""
    x = proj(enc, p[prefix + "proj_dec.weight"], p[prefix + "proj_dec.bias"], p[prefix + "cls_emb"][0], starts, n, round=False)
    for i in range(depth):
        sc = scales[i] if scales is not None and scales[i] is not None else (None, None)
        x = block(x, p, "%sblocks.%d." % (prefix, i), heads, eps, *sc)
    names = ["decoder_norm.weight", "decoder_norm.bias", "patch_proj.weight", "classes_proj.weight", "mask_norm.weight",
             "mask_norm.bias"]
    prm = {k: p[prefix + nm] for k, nm in zip(TAIL_PARAMS, names)}
    return tail(x, prm, H // patch, W // patch, H, W, eps, eps, round=False)
