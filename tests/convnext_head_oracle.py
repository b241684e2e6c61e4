"""fp32 restatement of the semantic-segmentation head of fine-tuning for the tests: ConvNeXtAdapter.forward
(multimae/output_adapters.py:545-573) with ConvNeXtBlock (multimae/output_adapter_utils.py:47-57), on top of the oracle
encoder of cls_head_oracle.encoder_tokens.  Also the model and values of the convnext_head.pt fixture."""
import math
from functools import partial

import torch
import torch.nn.functional as F

from helpers import formula_fill_

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


def convnext_head(enc, p, starts, n, H, W, preds_per_patch, depth, patch=16, eps=1e-6, prefix="output_adapters.semseg."):
    """enc [B, N, D] -> [B, K, H, W]; `starts`: first token of each main task, `n` tokens per task."""
    x = torch.cat([enc[:, s0:s0 + n] for s0 in starts], dim=-1)
    x = x @ p[prefix + "proj_dec.weight"].t() + p[prefix + "proj_dec.bias"]
    B, s = x.shape[0], int(math.isqrt(preds_per_patch))
    nh, nw = H // patch, W // patch
    C = x.shape[-1] // preds_per_patch
    # "b n (p c) -> b (n p) c" then "b (nh nw ph pw) c -> b c (nh ph) (nw pw)"
    x = x.reshape(B, nh, nw, s, s, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, nh * s, nw * s)
    for i in range(depth):
        q = "%sblocks.%d." % (prefix, i)
        y = F.conv2d(x, p[q + "dwconv.weight"], p[q + "dwconv.bias"], padding=3, groups=C).permute(0, 2, 3, 1)
        y = F.layer_norm(y, (C,), p[q + "norm.weight"], p[q + "norm.bias"], eps)
        y = F.gelu(y @ p[q + "pwconv1.weight"].t() + p[q + "pwconv1.bias"])
        y = y @ p[q + "pwconv2.weight"].t() + p[q + "pwconv2.bias"]
        x = x + y.permute(0, 3, 1, 2)
    x = F.conv2d(x, p[prefix + "final_layer.weight"], p[prefix + "final_layer.bias"])
    return F.interpolate(x, size=(H, W), mode="bilinear", align_corners=False)
