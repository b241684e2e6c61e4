"""fp32 restatement of the Segmenter head of semantic-segmentation fine-tuning for the tests:
SegmenterMaskTransformerAdapter.forward (multimae/output_adapters.py:450-478), on top of the oracle encoder of
cls_head_oracle.encoder_tokens.  Also the model and values of the segmenter_head.pt fixture."""
from functools import partial

import torch
import torch.nn.functional as F

from convnext_head_oracle import inputs as _inputs
from convnext_head_oracle import seg_loss  # noqa: F401  (re-exported: the criterion of run_finetuning_semseg.py)
from helpers import formula_fill_

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


def cosine_mask(P, C, gamma, beta, eps=1e-6):
    """LayerNorm over the classes of the cosine of every (patch, class) pair: P [B, n, E], C [B, K, E] -> [B, n, K]."""
    Pn = P / P.norm(dim=2, keepdim=True).clamp_min(1e-12)
    Cn = C / C.norm(dim=2, keepdim=True).clamp_min(1e-12)
    return F.layer_norm(Pn @ Cn.transpose(1, 2), (C.shape[1],), gamma, beta, eps)


def segmenter_head(enc, p, starts, n, H, W, depth, heads, patch=16, eps=1e-6, prefix="output_adapters.semseg.", scales=None):
    """enc [B, N, D] -> [B, K, H, W]; `starts`: first token of each main task, `n` tokens per task; `scales`: per block
    (s_attn, s_mlp) or None."""
    x = torch.cat([enc[:, s0:s0 + n] for s0 in starts], dim=-1)
    x = x @ p[prefix + "proj_dec.weight"].t() + p[prefix + "proj_dec.bias"]
    B, K = x.shape[0], p[prefix + "cls_emb"].shape[1]
    x = torch.cat([x, p[prefix + "cls_emb"].expand(B, -1, -1)], dim=1)
    for i in range(depth):
        sc = scales[i] if scales is not None and scales[i] is not None else (None, None)
        x = block(x, p, "%sblocks.%d." % (prefix, i), heads, eps, *sc)
    x = F.layer_norm(x, (x.shape[-1],), p[prefix + "decoder_norm.weight"], p[prefix + "decoder_norm.bias"], eps)
    m = cosine_mask(x[:, :n] @ p[prefix + "patch_proj.weight"].t(), x[:, n:] @ p[prefix + "classes_proj.weight"].t(),
                    p[prefix + "mask_norm.weight"], p[prefix + "mask_norm.bias"], eps)
    m = m.transpose(1, 2).reshape(B, K, H // patch, W // patch)
    return F.interpolate(m, size=(H, W), mode="bilinear", align_corners=False)
