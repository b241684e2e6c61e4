"""Record cls_head.pt from the LIVE reference: MultiViT + LinearOutputAdapter, the model of run_finetuning_cls.py.

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_cls.py

A small MultiViT (dim 128 so that the LayerNorm kernels apply, 2 heads of 64, depth 2) on 64 x 64 rgb + depth inputs,
B = 3, with output_adapters={'cls': LinearOutputAdapter(num_classes=10)}, run once with use_mean_pooling=True (the mean
over all tokens, the global token included) and once with use_mean_pooling=False (the global token), both from the same
state_dict.  The biases, the head LayerNorm weight and the global token are perturbed so that every term is exercised.
One training step per pooling mode (eval mode: drop_path_rate is 0, so both modes give the same values), with a fixed
loss: soft-target cross-entropy (utils/cross_entropy.py SoftTargetCrossEntropy) against a fixed soft target.

Stored: config, state_dict, inputs, target, logits and loss per mode, every parameter gradient per mode."""
import os
import sys
from functools import partial

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402
from make_golden import save_fixture  # noqa: E402

CONFIG = dict(in_domains=["rgb", "depth"], B=3, size=64, dim=128, depth=2, heads=2, num_classes=10)


def build(R, LinearOutputAdapter, mean_pool):
    c = CONFIG
    inputs = {"rgb": R.Patched(num_channels=3, stride_level=1, patch_size_full=16, image_size=c["size"]),
              "depth": R.Patched(num_channels=1, stride_level=1, patch_size_full=16, image_size=c["size"])}
    outputs = {"cls": LinearOutputAdapter(num_classes=c["num_classes"], use_mean_pooling=mean_pool)}
    return R.mm.MultiViT(input_adapters=inputs, output_adapters=outputs, num_global_tokens=1, dim_tokens=c["dim"],
                         depth=c["depth"], num_heads=c["heads"], mlp_ratio=4, qkv_bias=True,
                         norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def soft_target_ce(logits, target):
    return torch.sum(-target * torch.nn.functional.log_softmax(logits, dim=-1), dim=-1).mean()


def record(R, name, seed=61):
    from multimae.output_adapters import LinearOutputAdapter
    c = CONFIG
    torch.manual_seed(seed)
    model = build(R, LinearOutputAdapter, True)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith(".bias") or n == "global_tokens":
                p.add_(torch.randn(p.shape, generator=g) * 0.05)
            elif n == "output_adapters.cls.norm.weight":
                p.add_(torch.randn(p.shape, generator=g) * 0.1)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x = {"rgb": torch.randn(c["B"], 3, c["size"], c["size"], generator=g),
         "depth": torch.randn(c["B"], 1, c["size"], c["size"], generator=g)}
    target = torch.softmax(2.0 * torch.randn(c["B"], c["num_classes"], generator=g), dim=-1)
    out = {"config": dict(c), "state_dict": state, "inputs": x, "target": target, "logits": {}, "loss": {}}
    for mode, mean_pool in (("mean", True), ("last", False)):
        m = build(R, LinearOutputAdapter, mean_pool)
        m.load_state_dict(state)
        m = m.float().eval()
        logits = m(x)["cls"]
        loss = soft_target_ce(logits, target)
        loss.backward()
        out["logits"][mode] = logits.detach().clone()
        out["loss"][mode] = loss.detach().clone()
        out["grads_" + mode] = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    assert not torch.allclose(out["logits"]["mean"], out["logits"]["last"])
    save_fixture(out, os.path.join(HERE, name))
    print("wrote", name, {k: round(float(v), 6) for k, v in out["loss"].items()})


if __name__ == "__main__":
    record(MG.import_reference(), "cls_head.pt")
