"""Record convnext_head.pt from the LIVE reference: MultiViT + ConvNeXtAdapter, the model of run_finetuning_semseg.py.

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_convnext.py

The model and inputs are tests/convnext_head_oracle.py's CONFIG / build / fill_ / inputs: a small MultiViT on non-square
48 x 64 rgb + depth inputs, B = 2, with ConvNeXtAdapter(5, embed_dim=2048, preds_per_patch=16, depth=2,
main_tasks=['rgb', 'depth']) and ConvNeXtAdapter(8, embed_dim=2048, preds_per_patch=4, depth=1) (512 channels, x8
upsample).  Weights come from formula_fill_ (non-zero biases, block LayerNorm weights around 1) and are not stored.  One
training step (eval mode: nothing random) with the loss sum_heads CrossEntropyLoss(ignore_index=255) against fixed labels
that include ignored pixels.

Stored: config, the state_dict schema (keys and shapes, in order), inputs, labels, both outputs, the loss, and every
parameter gradient as a digest (norm + strided samples)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as MG  # noqa: E402
from convnext_head_oracle import CONFIG, build, fill_, inputs, seg_loss  # noqa: E402
from helpers import digest, save_fixture  # noqa: E402


def record(R, name):
    from multimae.output_adapters import ConvNeXtAdapter
    model = build(R.mm.MultiViT, R.Patched, ConvNeXtAdapter)
    fill_(model.named_parameters())
    model = model.float().eval()
    x, labels = inputs()
    outs = model(x)
    loss = seg_loss(outs, labels)
    loss.backward()
    out = {"config": CONFIG, "schema": [(k, tuple(v.shape)) for k, v in model.state_dict().items()], "inputs": x,
           "labels": labels, "outputs": {k: v.detach().clone() for k, v in outs.items()}, "loss": loss.detach().clone(),
           "grads": {n: digest(p.grad) for n, p in model.named_parameters() if p.grad is not None}}
    save_fixture(out, os.path.join(HERE, name))
    print("wrote", name, round(float(loss), 6))


if __name__ == "__main__":
    record(MG.import_reference(), "convnext_head.pt")
