"""Record convnext_depth.pt from the LIVE reference: MultiViT + ConvNeXtAdapter, the model of run_finetuning_depth.py
--output_adapter convnext.

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_convnext_depth.py

The model and inputs are tests/convnext_depth_oracle.py's CONFIG / build / fill_ / inputs: a small MultiViT on non-square
48 x 64 rgb + depth inputs, B = 2, with ConvNeXtAdapter(1, embed_dim=2048, preds_per_patch=64, depth=2,
main_tasks=['rgb', 'depth']) (32 channels, x2 upsample) and ConvNeXtAdapter(1, embed_dim=1536, preds_per_patch=16, depth=1)
(96 channels, x4 upsample).  Weights come from fill_ and are not stored.  One training step (eval mode: nothing random)
with the script's masked berhu loss on the first head plus its masked L1 loss on the second, against a fixed depth target
and a mask_valid with invalid pixels.  The losses are tests/convnext_depth_oracle.py's restatement; the maker checks it
against the script's own masked_berhu_loss / masked_l1_loss before it writes anything.

Stored: config, the state_dict schema (keys and shapes, in order), inputs, target, mask_valid, both outputs, the loss, and
every parameter gradient as a digest (norm + strided samples)."""
import importlib.util
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as MG  # noqa: E402
from convnext_depth_oracle import CONFIG, build, depth_loss, fill_, inputs  # noqa: E402
from helpers import digest, save_fixture  # noqa: E402


def _script_losses():
    """run_finetuning_depth.py as a module (its main() is not run): the loss functions the script trains with."""
    spec = importlib.util.spec_from_file_location("run_finetuning_depth", os.path.join(MG.REF, "run_finetuning_depth.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def record(R, name):
    from multimae.output_adapters import ConvNeXtAdapter
    model = build(R.mm.MultiViT, R.Patched, ConvNeXtAdapter)
    fill_(model.named_parameters())
    model = model.float().eval()
    x, target, mask_valid = inputs()
    outs = model(x)
    loss = depth_loss(outs, target, mask_valid)
    script = _script_losses()
    own = script.masked_berhu_loss(outs["depth"], target, mask_valid) + script.masked_l1_loss(outs["aux"], target, mask_valid)
    assert torch.allclose(loss, own, rtol=1e-6, atol=0), (float(loss), float(own))
    loss.backward()
    out = {"config": CONFIG, "schema": [(k, tuple(v.shape)) for k, v in model.state_dict().items()], "inputs": x,
           "target": target, "mask_valid": mask_valid, "outputs": {k: v.detach().clone() for k, v in outs.items()},
           "loss": loss.detach().clone(),
           "grads": {n: digest(p.grad) for n, p in model.named_parameters() if p.grad is not None}}
    save_fixture(out, os.path.join(HERE, name))
    print("wrote", name, round(float(loss.detach()), 6))


if __name__ == "__main__":
    record(MG.import_reference(), "convnext_depth.pt")
