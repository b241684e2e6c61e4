"""Record dropout.pt from the LIVE reference: a MultiViT training step with all three dropout sites live.

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_dropout.py

A small MultiViT (dim 128, 2 heads of 64, depth 2) on 64 x 64 rgb + depth inputs, B = 3, built with drop_rate = 0.25 and
attn_drop_rate = 0.4 (run_finetuning_cls.py's --drop / --attn_drop_rate), so every Block has Attention.attn_drop,
Attention.proj_drop and Mlp.drop live (multimae/multimae_utils.py:154,177,181).  The biases and the global token are
perturbed.  One training step: the encoder tokens times a fixed weight, summed, backward.

For the duration of the run nn.Dropout.forward is replaced by a wrapper that calls the original and recovers its keep
mask as (output != 0), checked against the original's output bit for bit (input * mask / (1 - p)); the inputs of every
recorded site are checked to have no zeros, so the mask is unambiguous.  The reference source is not modified.

Stored: config, state_dict, inputs, weight, the keep masks per block and site with their rates, the encoder tokens and
every parameter gradient."""
import os
import sys
from functools import partial

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as MG  # noqa: E402
from helpers import save_fixture  # noqa: E402

CONFIG = dict(in_domains=["rgb", "depth"], B=3, size=64, dim=128, depth=2, heads=2, drop_rate=0.25, attn_drop_rate=0.4)


def record(R, name, seed=71):
    c = CONFIG
    torch.manual_seed(seed)
    inputs = {"rgb": R.Patched(num_channels=3, stride_level=1, patch_size_full=16, image_size=c["size"]),
              "depth": R.Patched(num_channels=1, stride_level=1, patch_size_full=16, image_size=c["size"])}
    model = R.mm.MultiViT(input_adapters=inputs, output_adapters=None, num_global_tokens=1, dim_tokens=c["dim"],
                          depth=c["depth"], num_heads=c["heads"], mlp_ratio=4, qkv_bias=True,
                          drop_rate=c["drop_rate"], attn_drop_rate=c["attn_drop_rate"],
                          norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith(".bias") or n == "global_tokens":
                p.add_(torch.randn(p.shape, generator=g) * 0.05)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = {"rgb": torch.randn(c["B"], 3, c["size"], c["size"], generator=g),
         "depth": torch.randn(c["B"], 1, c["size"], c["size"], generator=g)}
    names = {}
    for i, blk in enumerate(model.encoder):
        names[id(blk.attn.attn_drop)] = ("encoder.%d" % i, "attn")
        names[id(blk.attn.proj_drop)] = ("encoder.%d" % i, "proj")
        names[id(blk.mlp.drop)] = ("encoder.%d" % i, "mlp")
    masks = {}
    original = torch.nn.Dropout.forward

    def recording_forward(self, t):
        out = original(self, t)
        if self.training and self.p > 0 and id(self) in names:
            assert bool((t != 0).all()), "a zero input makes the mask ambiguous"
            keep = out != 0
            assert torch.equal(out, t * keep.to(t.dtype) * (1.0 / (1.0 - self.p))), "mask recovery diverged"
            prefix, site = names[id(self)]
            assert site not in masks.setdefault(prefix, {})
            masks[prefix][site] = (keep.clone(), float(self.p))
        return out

    torch.nn.Dropout.forward = recording_forward
    try:
        model.train()
        tokens = model(x)
    finally:
        torch.nn.Dropout.forward = original
    w = torch.randn(tokens.shape, generator=g)
    (tokens * w).sum().backward()
    assert sorted(masks) == ["encoder.%d" % i for i in range(c["depth"])]
    assert all(sorted(m) == ["attn", "mlp", "proj"] for m in masks.values())
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    save_fixture({"config": dict(c), "state_dict": state, "inputs": x, "weight": w, "masks": masks,
                  "tokens": tokens.detach().clone(), "grads": grads}, os.path.join(HERE, name))
    print("wrote", name, {k: {s: round(float(m.float().mean()), 3) for s, (m, _) in v.items()} for k, v in masks.items()})


if __name__ == "__main__":
    record(MG.import_reference(), "dropout.pt")
