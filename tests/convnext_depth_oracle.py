"""Depth fine-tuning with the ConvNeXt head (run_finetuning_depth.py --output_adapter convnext) for the tests: the model and
values of the convnext_depth.pt fixture and an fp32 restatement of the script's masked losses.  The head itself is
convnext_head_oracle.convnext_head."""
from functools import partial

import torch

from convnext_head_oracle import fill_  # noqa: F401  (re-exported: the fixture's parameter values)

# convnext_depth.pt: MultiViT (dim 128, depth 2, 2 heads) on rgb + depth at 48 x 64 (3 x 4 patches), B = 2, with two
# one-channel heads: 64 predictions per patch over both tasks' tokens (C = 2048 / 64 = 32, s = 8, upsample x2) and 16 per
# patch over rgb (C = 1536 / 16 = 96, s = 4, upsample x4)
CONFIG = dict(in_domains=["rgb", "depth"], B=2, H=48, W=64, dim=128, depth=2, heads=2,
              adapters={"depth": dict(num_classes=1, embed_dim=2048, preds_per_patch=64, depth=2, main_tasks=["rgb", "depth"]),
                        "aux": dict(num_classes=1, embed_dim=1536, preds_per_patch=16, depth=1, main_tasks=["rgb"])})


def build(MultiViT, Patched, ConvNeXtAdapter, c=CONFIG):
    """The fixture's model from the given classes (the reference's, or this package's)."""
    ins = {"rgb": Patched(num_channels=3, stride_level=1, patch_size_full=16, image_size=(c["H"], c["W"])),
           "depth": Patched(num_channels=1, stride_level=1, patch_size_full=16, image_size=(c["H"], c["W"]))}
    outs = {k: ConvNeXtAdapter(**v) for k, v in c["adapters"].items()}
    return MultiViT(ins, outs, num_global_tokens=1, dim_tokens=c["dim"], depth=c["depth"], num_heads=c["heads"], mlp_ratio=4,
                    qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def inputs(c=CONFIG, seed=11):
    """rgb, the depth target (positive), and mask_valid [B, 1, H, W] (bool, about 15 % invalid pixels).  The depth input is
    the target with the invalid pixels set to 0, as the script's train_one_epoch does before the forward."""
    g = torch.Generator().manual_seed(seed)
    B, H, W = c["B"], c["H"], c["W"]
    rgb = torch.randn(B, 3, H, W, generator=g)
    target = 0.5 + 4.0 * torch.rand(B, 1, H, W, generator=g)
    mask_valid = torch.rand(B, 1, H, W, generator=g) >= 0.15
    depth_in = torch.where(mask_valid, target, torch.zeros(()))
    return {"rgb": rgb, "depth": depth_in}, target, mask_valid


def masked_berhu_loss(preds, target, mask_valid):
    """run_finetuning_depth.py masked_berhu_loss: reverse Huber on the valid pixels, threshold c = 0.2 max |diff| (at least
    1e-5, no gradient through c), summed and divided by the number of valid pixels."""
    if preds.shape[1] != mask_valid.shape[1]:
        mask_valid = mask_valid.repeat_interleave(preds.shape[1], 1)
    diff = torch.where(mask_valid, preds - target, torch.zeros((), device=preds.device))
    with torch.no_grad():
        c = torch.clamp_min(diff.abs().max() * 0.2, 1e-5)
    ad = diff.abs()
    l2 = (diff * diff + c * c) / 2.0 / c
    return torch.where(ad < c, ad, l2).sum() / mask_valid.sum()


def masked_l1_loss(preds, target, mask_valid):
    """run_finetuning_depth.py masked_l1_loss: |preds - target| on the valid pixels over the number of valid pixels."""
    if preds.shape[1] != mask_valid.shape[1]:
        mask_valid = mask_valid.repeat_interleave(preds.shape[1], 1)
    return torch.where(mask_valid, (preds - target).abs(), torch.zeros((), device=preds.device)).sum() / mask_valid.sum()


def depth_loss(outs, target, mask_valid):
    """The fixture's training loss: berhu on the 'depth' head plus L1 on the 'aux' head, both against the same target."""
    t, m = target.to(outs["depth"].device), mask_valid.to(outs["depth"].device)
    return masked_berhu_loss(outs["depth"], t, m) + masked_l1_loss(outs["aux"], t, m)
