"""Record segmenter_head.pt from the LIVE reference: MultiViT + SegmenterMaskTransformerAdapter, the model of
run_finetuning_semseg.py --output_adapter segmenter.

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_segmenter.py

The model and inputs are tests/segmenter_head_oracle.py's CONFIG / build / fill_ / inputs: a small MultiViT on non-square
48 x 64 rgb + depth inputs, B = 2, with a 9-class head of depth 2 over both tasks' tokens and a 13-class head of depth 1
over rgb.  Weights come from segmenter_head_oracle.fill_ (formula_fill_ with seeded normal head matrices and class tokens) and are not
stored.
One training step (eval mode: nothing random) with the loss sum_heads CrossEntropyLoss(ignore_index=255) against fixed
labels that include ignored pixels.

Stored: config, the state_dict schema (keys and shapes, in order), inputs, labels, both outputs, the loss, and every
parameter gradient as a digest (norm + strided samples)."""
import os
import sys

import torch  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as MG  # noqa: E402
from helpers import digest, save_fixture  # noqa: E402
from segmenter_head_oracle import CONFIG, build, fill_, inputs, seg_loss  # noqa: E402


def record(R, name):
    from multimae.output_adapters import SegmenterMaskTransformerAdapter
    model = build(R.mm.MultiViT, R.Patched, SegmenterMaskTransformerAdapter)
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
    record(MG.import_reference(), "segmenter_head.pt")
