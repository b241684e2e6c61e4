"""Record learnable_pos.pt from the LIVE reference: trainable position tables of the input adapters.

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_learnable_pos.py

Two models, one training step each (nothing random in the step), weights from formula_fill_ (not stored):
  mae : MultiMAE with rgb + depth + semseg inputs and outputs (+ norm_rgb), dim 128, B = 2, 64 x 64, every input table
        trainable.  The depth and semseg tables are the sin-cos tables with learnable_pos_emb=True; the rgb one is random,
        as sincos_pos_emb=False makes it.  Fixed task masks keep 10 of 48 patches per sample, so that some patches of
        every task are masked in both samples.  The reference takes ONE visible count from the whole batch for
        caller-supplied masks (multimae/multimae.py:338), so the masks reach it as the triple generate_random_masks
        returns, computed with the stable sort the CUDA path's fixed-mask branch uses.  Tables at the 4 x 4 grid of the
        input: the resize is the identity.  Losses as in record_model of make_golden.py.
  vit : MultiViT with rgb + semseg inputs, no output adapter, dim 128, B = 2.  The tables are built for 48 x 64 images
        (3 x 4 patches) and the inputs are 80 x 96 (5 x 6 patches): the rgb table is resized bicubic, the semseg table
        bilinear, both ways.  The rgb table is random (sincos_pos_emb=False), the semseg one sin-cos with
        learnable_pos_emb=True.  Loss: sum(encoder_tokens * weights) with fixed random weights.

Stored per model: config, initial tables, inputs, masks / index triple (mae), outputs, losses, the pos_emb gradients in
full and every other parameter gradient as a digest (norm + strided samples)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as MG  # noqa: E402
from helpers import digest, formula_fill_, save_fixture  # noqa: E402

MAE = dict(in_domains=["rgb", "depth", "semseg"], B=2, size=64, dim=128, depth=1, heads=2, dec_dim=128, dec_depth=1,
           dec_heads=4, image_size=64, n_visible=10)
VIT = dict(in_domains=["rgb", "semseg"], B=2, table_size=(48, 64), input_size=(80, 96), dim=128, depth=1, heads=2)


def mae_task_masks(c):
    """1 = masked: per sample a random choice of n_visible of the 3 x 16 patches stays visible."""
    g = torch.Generator().manual_seed(61)
    n = (c["size"] // 16) ** 2
    total = n * len(c["in_domains"])
    mask = torch.ones(c["B"], total, dtype=torch.long)
    for b in range(c["B"]):
        mask[b, torch.randperm(total, generator=g)[:c["n_visible"]]] = 0
    return {d: mask[:, i * n:(i + 1) * n].clone() for i, d in enumerate(c["in_domains"])}


def mae_inputs(c):
    g = torch.Generator().manual_seed(62)
    s = c["size"]
    return {"rgb": torch.randn(c["B"], 3, s, s, generator=g), "depth": torch.randn(c["B"], 1, s, s, generator=g),
            "semseg": torch.randint(0, 133, (c["B"], s // 4, s // 4), generator=g)}


def vit_inputs(c):
    g = torch.Generator().manual_seed(63)
    H, W = c["input_size"]
    x = {"rgb": torch.randn(c["B"], 3, H, W, generator=g), "semseg": torch.randint(0, 133, (c["B"], H // 4, W // 4), generator=g)}
    n = (H // 16) * (W // 16) * len(c["in_domains"]) + 1
    return x, torch.randn(c["B"], n, c["dim"], generator=g)


def random_table(shape, seed):
    """The values sincos_pos_emb=False starts from (trunc_normal_(std=0.02)), drawn here from a fixed generator."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * 0.02).clamp(-0.04, 0.04)


def stable_triple(task_masks, domains):
    mask_all = torch.cat([task_masks[d] for d in domains], dim=1)
    ids_shuffle = torch.argsort(mask_all, dim=1, stable=True)
    ids_restore = torch.argsort(ids_shuffle, dim=1, stable=True)
    n_vis = int((mask_all[0] == 0).sum())
    return task_masks, ids_shuffle[:, :n_vis], ids_restore


def _grads(model):
    pos = {n: p.grad.clone() for n, p in model.named_parameters() if n.endswith("pos_emb") and p.grad is not None}
    rest = {n: digest(p.grad) for n, p in model.named_parameters() if not n.endswith("pos_emb") and p.grad is not None}
    return pos, rest


def record_mae(R):
    c = MAE
    torch.manual_seed(60)
    model = MG.build_model(R, tuple(c["in_domains"]), dim=c["dim"], depth=c["depth"], heads=c["heads"], dec_dim=c["dec_dim"],
                           dec_depth=c["dec_depth"], dec_heads=c["dec_heads"], image_size=c["image_size"])
    formula_fill_(list(model.named_parameters()))
    with torch.no_grad():
        model.input_adapters["rgb"].pos_emb.copy_(random_table(model.input_adapters["rgb"].pos_emb.shape, 64))
    for ad in model.input_adapters.values():
        ad.pos_emb.requires_grad_(True)
    tables = {"input_adapters.%s.pos_emb" % d: ad.pos_emb.detach().clone() for d, ad in model.input_adapters.items()}
    x = mae_inputs(c)
    tm = mae_task_masks(c)
    triple = stable_triple(tm, c["in_domains"])
    model.generate_random_masks = lambda *a, **k: triple
    preds, masks = model(x, num_encoded_tokens=c["n_visible"], alphas=1.0)
    loss_fns = {"rgb": R.MSE(16, 1), "depth": R.L1(16, 1), "semseg": R.CE(16, 4), "norm_rgb": R.MSE(16, 1, norm_pix=True)}
    losses = {}
    for task in preds:
        src = "rgb" if task == "norm_rgb" else task
        losses[task] = loss_fns[task](preds[task].float(), x[src], mask=masks.get(src))
    sum(losses.values()).backward()
    pos, rest = _grads(model)
    return {"config": c, "tables": tables, "inputs": x, "task_masks": tm, "ids_keep": triple[1], "ids_restore": triple[2],
            "preds": {k: v.detach().clone() for k, v in preds.items()},
            "losses": {k: v.detach().clone() for k, v in losses.items()}, "pos_grads": pos, "grads": rest}


def record_vit(R):
    c = VIT
    torch.manual_seed(65)
    inputs = {"rgb": R.Patched(num_channels=3, stride_level=1, patch_size_full=16, image_size=c["table_size"],
                               sincos_pos_emb=False),
              "semseg": R.SemSeg(num_classes=133, dim_class_emb=64, interpolate_class_emb=False, stride_level=4,
                                 patch_size_full=16, image_size=c["table_size"], learnable_pos_emb=True)}
    model = R.mm.MultiViT(input_adapters=inputs, output_adapters=None, num_global_tokens=1, dim_tokens=c["dim"],
                          depth=c["depth"], num_heads=c["heads"], mlp_ratio=4, qkv_bias=True).float().train()
    formula_fill_(list(model.named_parameters()))
    with torch.no_grad():
        model.input_adapters["rgb"].pos_emb.copy_(random_table(model.input_adapters["rgb"].pos_emb.shape, 66))
    assert all(ad.pos_emb.requires_grad for ad in model.input_adapters.values())
    tables = {"input_adapters.%s.pos_emb" % d: ad.pos_emb.detach().clone() for d, ad in model.input_adapters.items()}
    x, weights = vit_inputs(c)
    tokens = model(x)
    loss = (tokens * weights).sum()
    loss.backward()
    pos, rest = _grads(model)
    return {"config": c, "tables": tables, "inputs": x, "weights": weights, "tokens": tokens.detach().clone(),
            "loss": loss.detach().clone(), "pos_grads": pos, "grads": rest}


if __name__ == "__main__":
    R = MG.import_reference()
    out = {"mae": record_mae(R), "vit": record_vit(R)}
    save_fixture(out, os.path.join(HERE, "learnable_pos.pt"))
    print("wrote learnable_pos.pt", {k: round(float(v), 6) for k, v in out["mae"]["losses"].items()},
          round(float(out["vit"]["loss"]), 6))
