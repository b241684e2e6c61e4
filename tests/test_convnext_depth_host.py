"""CPU: depth fine-tuning with the ConvNeXt head (run_finetuning_depth.py --output_adapter convnext) without a GPU.

1. The fp32 restatement (tests/convnext_head_oracle.py + the script's masked losses in tests/convnext_depth_oracle.py) on the
   oracle encoder reproduces the reference's outputs, loss and every parameter gradient, recorded by
   tests/golden/make_golden_convnext_depth.py: heads of 32 and 96 channels per pixel, one output channel.
2. The host layer against a stub of the C library at C = 32 and 96, K = 1 and 3, s = 8: entry points and their order, sizes and
   gradient-arena pointers; the library's saved / workspace sizes at those shapes.
3. Widths that are not a multiple of 32, or above 1024, raise in the adapter and in the C ABI, and so do other multiples
   of 32 for heads of more than 8 output channels; the LayerNorm entry points refuse the fused forms at narrow widths.
4. The depth script's model, optimizer and scaler set-up with its default arguments through the overlay."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

from cls_head_oracle import encoder_tokens, vit_config
from convnext_depth_oracle import CONFIG, build, depth_loss, fill_, inputs, masked_berhu_loss, masked_l1_loss
from convnext_head_oracle import convnext_head
from helpers import load_fixture
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from test_convnext_head_host import assert_digest_close
from test_drop_path_host import _Rec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STANDIN = os.path.join(ROOT, "tests", "adamw_standin")


@pytest.fixture(scope="module")
def fx(golden_dir):
    return load_fixture(golden_dir, "convnext_depth.pt")


def _model():
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import ConvNeXtAdapter
    return build(MultiViT, PatchedInputAdapter, ConvNeXtAdapter)


def oracle_outputs(p, x, c=CONFIG):
    cfg = vit_config(c["in_domains"], c["dim"], c["depth"], c["heads"], 64)
    enc = encoder_tokens(p, x, cfg)
    n = (c["H"] // 16) * (c["W"] // 16)
    start = {"rgb": 0, "depth": n}
    return {k: convnext_head(enc, p, [start[t] for t in a["main_tasks"]], n, c["H"], c["W"], a["preds_per_patch"], a["depth"],
                             prefix="output_adapters.%s." % k) for k, a in c["adapters"].items()}


def test_oracle_head_against_reference(fx):
    from oracle import multimae_oracle as O
    model = _model()
    fill_(model.named_parameters())
    p = {k: v.detach().clone() for k, v in model.state_dict().items()}
    train = O.trainable(p)
    for v in train.values():
        v.requires_grad_(True)
    outs = oracle_outputs(p, fx["inputs"])
    for k, ref in fx["outputs"].items():
        assert outs[k].shape == ref.shape == (2, 1, 48, 64)
        torch.testing.assert_close(outs[k], ref, rtol=1e-4, atol=1e-5, msg=lambda m, k=k: "%s: %s" % (k, m))
    loss = depth_loss(outs, fx["target"], fx["mask_valid"])
    torch.testing.assert_close(loss, fx["loss"], rtol=1e-5, atol=1e-6)
    loss.backward()
    assert set(fx["grads"]) == {k for k, v in train.items() if v.grad is not None}
    for k, ref in fx["grads"].items():
        assert_digest_close(train[k].grad, ref, 2e-4, k)


def test_fixture_inputs_and_schema(fx):
    x, target, mask_valid = inputs()
    assert all(torch.equal(x[k], fx["inputs"][k]) for k in x)
    assert torch.equal(target, fx["target"]) and torch.equal(mask_valid, fx["mask_valid"])
    assert 0.1 < float((~mask_valid).float().mean()) < 0.2 and not x["depth"][~mask_valid].any()
    sd = _model().state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [(k, tuple(s)) for k, s in fx["schema"]]
    assert tuple(sd["output_adapters.depth.blocks.1.dwconv.weight"].shape) == (32, 1, 7, 7)
    assert tuple(sd["output_adapters.aux.blocks.0.norm.weight"].shape) == (96,)
    assert tuple(sd["output_adapters.depth.final_layer.weight"].shape) == (1, 32, 1, 1)


def test_masked_losses_by_hand():
    """The berhu / L1 restatement on a few hand-checked values: invalid pixels count neither in the sum nor the divisor."""
    preds = torch.tensor([[[[1.0, 2.0], [3.0, 10.0]]]])
    target = torch.tensor([[[[1.5, 2.0], [0.0, 0.0]]]])
    mask = torch.tensor([[[[True, True], [True, False]]]])
    # valid diffs 0.5, 0, 3 -> c = 0.6: 0.5 and 0 are L1, 3 is (9 + 0.36) / 1.2
    assert math.isclose(float(masked_berhu_loss(preds, target, mask)), (0.5 + 0.0 + 9.36 / 1.2) / 3, rel_tol=1e-6)
    assert math.isclose(float(masked_l1_loss(preds, target, mask)), 3.5 / 3, rel_tol=1e-6)


@pytest.fixture()
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(L, "lib", lambda: r)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    return r


def _info(H, W, tasks=("rgb",), patch=16):
    n = (H // patch) * (W // patch)
    return {"image_size": (H, W), "num_task_tokens": n * len(tasks), "num_global_tokens": 1,
            "tasks": {t: {"num_tokens": n, "start_idx": i * n, "end_idx": (i + 1) * n} for i, t in enumerate(tasks)}}


CALLS = ["mmae_convnext_proj_forward", "mmae_convnext_block_forward", "mmae_convnext_block_forward",
         "mmae_convnext_tail_forward", "mmae_convnext_tail_backward", "mmae_convnext_block_backward",
         "mmae_convnext_block_backward", "mmae_convnext_proj_backward"]


@pytest.mark.parametrize("C,K", [(32, 1), (96, 1), (96, 3)])
def test_entry_points_at_narrow_widths(rec, C, K):
    from multimae_b200.output_adapters import ConvNeXtAdapter
    ad = ConvNeXtAdapter(K, embed_dim=64 * C, preds_per_patch=64, depth=2, main_tasks=["rgb", "depth"])
    ad.init(dim_tokens_enc=128)
    ad.train()
    x = torch.randn(3, 2 * 12 + 1, 128, requires_grad=True)
    out = ad(x, _info(48, 64, tasks=("rgb", "depth")))
    assert out.shape == (3, K, 48, 64) and out.dtype == torch.float32
    out.sum().backward()
    assert [n for n in rec.names() if n.startswith("mmae_convnext") and not n.endswith("_bytes")] == CALLS
    calls = [a for n, a in rec.calls if n.startswith("mmae_convnext") and not n.endswith("_bytes")]
    pf, bf0, bf1, tf, tb, bb1, bb0, pb = calls
    arena = ad._bound["arena"]
    v = lambda k: arena.views[k].data_ptr()                                     # noqa: E731
    assert list(pf[1:6]) == [3, 25, 128, 12, 2] and list(pf[6][:2]) == [0, 12] and pf[7] == 64 * C
    assert pb[9] == v("proj_dec.weight") and pb[10] == v("proj_dec.bias") and pf[11] == pb[12]
    for i, (f, b) in enumerate(((bf0, bb0), (bf1, bb1))):
        assert list(f[2:7]) == [3, 3, 4, 8, C] and list(b[3:8]) == [3, 3, 4, 8, C] and b[10] == f[9]
        for j, name in enumerate(Fn.CONVNEXT_BLOCK_PARAM_NAMES):
            assert f[8][j] == dict(ad.named_parameters())["blocks.%d.%s" % (i, name)].data_ptr()
            assert b[9][j] == v("blocks.%d.%s" % (i, name)), (i, name)
    assert bf1[0] == bf0[1] and bb1[2] == bb0[1] and pf[10] == bf0[0] and tf[0] == bf1[1]
    # the proj output is the [B * n * s * s, C] view: 3 * 12 * 64 rows
    assert list(tf[1:9]) == [3, 3, 4, 8, C, K, 48, 64] and list(tb[1:9]) == list(tf[1:9])
    assert tf[11] == out.data_ptr() and tb[10] == v("final_layer.weight") and tb[11] == v("final_layer.bias")
    assert ("mmae_convnext_tail_saved_bytes", (3, 3, 4, 8, C, K)) in rec.calls
    assert ("mmae_convnext_block_workspace_bytes", (3, 3, 4, 8, C)) in rec.calls
    for n, p in ad.named_parameters():
        assert torch.equal(p.grad, arena.views[n]), n
    assert x.grad.shape == x.shape


def _carve(sizes):
    off = 0
    for n in sizes:
        off = (off + 255) // 256 * 256 + n
    return (off + 255) // 256 * 256


@pytest.mark.parametrize("B,nh,nw,C", [(4, 16, 16, 96), (3, 3, 4, 32), (1, 30, 40, 96)])
def test_saved_and_workspace_bytes(B, nh, nw, C):
    """The library's size queries at s = 8, K = 1 (padded to Kp = 8) against the layouts they describe."""
    lib, s, K, Kp = L.lib(), 8, 1, 8
    P = B * nh * nw * s * s
    tiles_x = -(-nw * s // 16)
    assert lib.mmae_convnext_block_saved_bytes(B, nh, nw, s, C) == _carve(
        [2 * 4 * C * C, 2 * 4 * C * C, 4 * P * C, 4 * P, 4 * P, 2 * P * C, 2 * P * 4 * C, 2 * P * 4 * C])
    assert lib.mmae_convnext_block_workspace_bytes(B, nh, nw, s, C) == _carve(
        [2 * P * C, 2 * P * 4 * C, 2 * P * C, 4 * P * C, 4 * B * tiles_x * C * 49])
    assert lib.mmae_convnext_tail_saved_bytes(B, nh, nw, s, C, K) == _carve([2 * P * C, 2 * Kp * C])
    assert lib.mmae_convnext_tail_workspace_bytes(B, nh, nw, s, C, K) == _carve([4 * P * Kp, 4 * Kp, 4 * Kp, 4 * Kp * C, 2 * P * Kp])


def test_width_errors():
    """Channel widths: multiples of 128 up to 1024 for any head; other multiples of 32 up to 1024 for heads of at most
    NARROW_HEAD_MAX_OUTPUTS output channels (the depth head); everything else raises with the rule in the message."""
    from multimae_b200.output_adapters import NARROW_HEAD_MAX_OUTPUTS, ConvNeXtAdapter
    assert NARROW_HEAD_MAX_OUTPUTS == 8
    for K, embed_dim, ppp in ((1, 6144, 64), (1, 1536, 16), (8, 2048, 64), (3, 16384, 16), (41, 6144, 16), (41, 2048, 4)):
        assert ConvNeXtAdapter(K, embed_dim=embed_dim, preds_per_patch=ppp).class_dim == embed_dim // ppp
    for K, embed_dim, ppp in ((1, 3072, 64), (1, 1600, 16), (1, 2048 * 16, 16), (1, 1056 * 16, 16), (41, 1536, 16),
                              (9, 6144, 64), (150, 6144, 64)):           # C = 48, 100, 2048, 1056; 96 for 41 / 9 / 150
        with pytest.raises(NotImplementedError, match="multiple of 128, at most 1024"):
            ConvNeXtAdapter(K, embed_dim=embed_dim, preds_per_patch=ppp)


def test_c_abi_width_errors():
    """The C checks fire before any CUDA call: ConvNeXt entry points and the LayerNorm forms at unsupported widths."""
    lib = L.lib()
    UNSUPPORTED = 3
    prm = (ctypes.c_void_p * 8)(*([16] * 8))
    for C in (48, 100, 1056):
        assert lib.mmae_convnext_block_forward(16, 16, 1, 2, 2, 8, C, 1e-6, prm, 16, 16, None) == UNSUPPORTED
        assert b"must be a multiple of 32, at most 1024" in lib.mmae_last_error()
        assert lib.mmae_convnext_tail_forward(16, 1, 2, 2, 8, C, 1, 32, 32, 16, 16, 16, 16, 16, None) == UNSUPPORTED
        assert b"multiple of 32" in lib.mmae_last_error()
        assert lib.mmae_layernorm_forward(16, C, 16, 16, 16, C, None, 0, 16, 16, 4, C, 1e-6, None) == UNSUPPORTED
        assert b"multiple of 128 (of 32 for the plain form)" in lib.mmae_last_error()
        assert lib.mmae_layernorm_backward(16, 1, C, 16, C, 16, 16, 16, None, 0, 16, C, 16, 16, 4, C, None) == UNSUPPORTED
    # the fused add / the bf16 copy of dx exist only for multiples of 128
    assert lib.mmae_add_layernorm_forward(16, 96, 16, 96, None, 0, 16, 16, 16, 96, 16, 16, 4, 96, 1e-6, None) == UNSUPPORTED
    assert b"fused add" in lib.mmae_last_error()
    assert lib.mmae_layernorm_backward_ex(16, 1, 96, 16, 96, 16, 16, 16, None, 0, 16, 96, 16, 16, 16, 96, None, 4, 96,
                                          None) == UNSUPPORTED
    assert b"bf16 copy" in lib.mmae_last_error()


# one process: the overlay rewires sys.modules; the library is a recording stub (no GPU here)
_SETUP = r"""
import argparse, os, sys
from functools import partial
import torch
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, "tests"))
sys.path.insert(0, %(standin)r)
from multimae_b200 import _lib as L, functional as Fn, optim as O, overlay
from test_drop_path_host import _Rec
L.lib = lambda: _Rec()
L.current_stream = lambda: 0
Fn._require_cuda = lambda t, what: None
O._on_device = lambda p: True
overlay.install()
from multimae import multimae as mm
from multimae.input_adapters import PatchedInputAdapter
from multimae.output_adapters import ConvNeXtAdapter, DPTOutputAdapter
from utils import NativeScalerWithGradNormCount as NativeScaler
from utils.optim_factory import LayerDecayValueAssigner, create_optimizer
import multimae_b200.output_adapters, multimae_b200.native_scaler
assert ConvNeXtAdapter is multimae_b200.output_adapters.ConvNeXtAdapter
assert NativeScaler is multimae_b200.native_scaler.NativeScalerWithGradNormCount
# run_finetuning_depth.py's defaults, with --output_adapter convnext and the given --in_domains / --decoder_main_tasks
args = argparse.Namespace(in_domains=%(in_domains)r.split("-"), decoder_main_tasks=%(main)r.split("-"), patch_size=16,
                          input_size=256, model="multivit_base", output_adapter="convnext", drop_path_encoder=%(dpe)r,
                          opt="adamw", opt_eps=1e-8, opt_betas=[0.9, 0.999], momentum=0.9, weight_decay=1e-4, lr=1e-4,
                          layer_decay=0.75, scale_input_lr=True)
DOMAIN_CONF = {"rgb": {"channels": 3, "stride_level": 1, "input_adapter": partial(PatchedInputAdapter, num_channels=3)},
               "depth": {"channels": 1, "stride_level": 1, "input_adapter": partial(PatchedInputAdapter, num_channels=1)}}
input_adapters = {d: DOMAIN_CONF[d]["input_adapter"](stride_level=DOMAIN_CONF[d]["stride_level"],
                                                     patch_size_full=args.patch_size, image_size=args.input_size)
                  for d in args.in_domains}
adapters_dict = {"dpt": DPTOutputAdapter, "convnext": partial(ConvNeXtAdapter, preds_per_patch=64)}
output_adapters = {d: adapters_dict[args.output_adapter](num_classes=DOMAIN_CONF[d]["channels"],
                                                          stride_level=DOMAIN_CONF[d]["stride_level"],
                                                          patch_size=args.patch_size, main_tasks=args.decoder_main_tasks)
                   for d in ["depth"]}
model = mm.__dict__[args.model](input_adapters=input_adapters, output_adapters=output_adapters,
                                drop_path_rate=args.drop_path_encoder)
sd = model.state_dict()
assert tuple(sd["output_adapters.depth.proj_dec.weight"].shape) == (6144, 768 * len(args.decoder_main_tasks))
assert tuple(sd["output_adapters.depth.blocks.3.dwconv.weight"].shape) == (96, 1, 7, 7)
assert "output_adapters.depth.blocks.4.dwconv.weight" not in sd          # the script does not pass --decoder_depth
assert tuple(sd["output_adapters.depth.final_layer.weight"].shape) == (1, 96, 1, 1)
num_layers = model.get_num_layers()
values = list(args.layer_decay ** (num_layers + 1 - i) for i in range(num_layers + 2))
assigner = LayerDecayValueAssigner(values)
optimizer = create_optimizer(args, model, skip_list=model.no_weight_decay(), get_num_layer=assigner.get_layer_id,
                             get_layer_scale=assigner.get_scale)
loss_scaler = NativeScaler(enabled=False)
scales = sorted({round(g["lr_scale"], 6) for g in optimizer.param_groups})
print("optimizer", type(optimizer).__module__ + "." + type(optimizer).__name__, len(optimizer.param_groups), len(scales))
print("params", sum(p.numel() for p in model.parameters()), "scaler", loss_scaler.state_dict())
print("ok")
"""


@pytest.mark.parametrize("in_domains,main,dpe,flat", [("rgb", "rgb", 0.0, "0"), ("rgb-depth", "rgb-depth", 0.1, "1")])
def test_depth_script_model_setup(in_domains, main, dpe, flat):
    """run_finetuning_depth.py:415-532 through the overlay: the input adapters of --in_domains, the convnext head as the
    script builds it (preds_per_patch 64 on the adapter's default embed_dim 6144 and depth 4: 96 channels per pixel), the
    registered multivit_base with --drop_path_encoder, the layer-decay parameter groups (stock AdamW, or GroupedFlatAdamW
    under MMAE_FLAT_ADAMW=1) and NativeScaler(enabled=False)."""
    env = dict(os.environ, MMAE_FLAT_ADAMW=flat)
    code = _SETUP % dict(root=ROOT, standin=STANDIN, in_domains=in_domains, main=main, dpe=dpe)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=env)
    assert res.returncode == 0 and res.stdout.endswith("ok\n"), res.stdout + res.stderr[-3000:]
    lines = res.stdout.splitlines()
    name = "multimae_b200.optim.GroupedFlatAdamW" if flat == "1" else "torch.optim.adamw.AdamW"
    opt = [ln for ln in lines if ln.startswith("optimizer ")]
    assert opt and opt[0].startswith("optimizer %s " % name) and opt[0].endswith(" 14"), lines     # 14 layer scales
