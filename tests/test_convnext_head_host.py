"""CPU: the semantic-segmentation head of fine-tuning (ConvNeXtAdapter, run_finetuning_semseg.py) without a GPU.

1. The fp32 restatement (tests/convnext_head_oracle.py) on the oracle encoder reproduces the reference's outputs, loss and
   every parameter gradient, recorded by tests/golden/make_golden_convnext.py.
2. A model built by our factory has the reference's state_dict schema and initialisation.
3. The host layer against a stub of the C library: entry points and their order, sizes, gradient-arena pointers,
   on_grads_ready, no-grad, and the errors raised for what the CUDA head does not cover.
4. The overlay resolves the three adapters of run_finetuning_semseg.py; its model set-up runs with the ADE config."""
import math
import os
import subprocess
import sys
from functools import partial

import pytest
import torch

from cls_head_oracle import encoder_tokens, vit_config
from convnext_head_oracle import CONFIG, build, convnext_head, fill_, inputs, seg_loss
from helpers import digest, load_fixture
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from test_drop_path_host import _Rec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx(golden_dir):
    return load_fixture(golden_dir, "convnext_head.pt")


def _model():
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import ConvNeXtAdapter
    return build(MultiViT, PatchedInputAdapter, ConvNeXtAdapter)


def _filled_state():
    model = _model()
    fill_(model.named_parameters())
    return model, {k: v.detach().clone() for k, v in model.state_dict().items()}


def oracle_outputs(p, x, c=CONFIG):
    """Both heads of the fixture model through the oracle encoder + the fp32 restatement."""
    cfg = vit_config(c["in_domains"], c["dim"], c["depth"], c["heads"], 64)
    enc = encoder_tokens(p, x, cfg)
    n = (c["H"] // 16) * (c["W"] // 16)
    start = {"rgb": 0, "depth": n}
    return {k: convnext_head(enc, p, [start[t] for t in a["main_tasks"]], n, c["H"], c["W"], a["preds_per_patch"], a["depth"],
                             prefix="output_adapters.%s." % k) for k, a in c["adapters"].items()}


def assert_digest_close(got, ref, rtol, what):
    d = digest(got)
    assert d["step"] == ref["step"], what
    assert abs(float(d["norm"]) - float(ref["norm"])) <= rtol * float(ref["norm"]) + 1e-12, (what, d["norm"], ref["norm"])
    err = float((d["samples"] - ref["samples"]).norm() / (ref["samples"].norm() + 1e-12))
    assert err <= rtol, (what, err)


def test_oracle_head_against_reference(fx):
    from oracle import multimae_oracle as O
    _, p = _filled_state()
    train = O.trainable(p)
    for v in train.values():
        v.requires_grad_(True)
    outs = oracle_outputs(p, fx["inputs"])
    for k, ref in fx["outputs"].items():
        torch.testing.assert_close(outs[k], ref, rtol=1e-4, atol=1e-5, msg=lambda m, k=k: "%s: %s" % (k, m))
    loss = seg_loss(outs, fx["labels"])
    torch.testing.assert_close(loss, fx["loss"], rtol=1e-5, atol=1e-6)
    loss.backward()
    assert set(fx["grads"]) == {k for k, v in train.items() if v.grad is not None}
    for k, ref in fx["grads"].items():
        assert_digest_close(train[k].grad, ref, 2e-4, k)


def test_fixture_inputs_are_the_recorded_ones(fx):
    x, labels = inputs()
    assert all(torch.equal(x[k], fx["inputs"][k]) for k in x)
    assert all(torch.equal(labels[k], fx["labels"][k]) for k in labels)
    assert any(bool((v == 255).any()) for v in labels.values())


def test_factory_model_schema_and_init(fx):
    """Keys, order and shapes of the reference's state_dict; the model's re-initialisation (xavier-uniform Linears with zero
    bias, LayerNorm 1 / 0) over proj_dec / pwconv1 / pwconv2, PyTorch's default Conv2d initialisation for dwconv and
    final_layer (the reference initialises neither)."""
    torch.manual_seed(0)
    sd = _model().state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [(k, tuple(s)) for k, s in fx["schema"]]
    pre = "output_adapters.semseg."
    keys = [k[len(pre):] for k in sd if k.startswith(pre)]
    assert keys[:8] == ["blocks.0." + n for n in Fn.CONVNEXT_BLOCK_PARAM_NAMES]
    assert keys[-4:] == ["final_layer.weight", "final_layer.bias", "proj_dec.weight", "proj_dec.bias"]
    for name, (fo, fi) in (("proj_dec", (2048, 256)), ("blocks.0.pwconv1", (512, 128)), ("blocks.1.pwconv2", (128, 512))):
        w = sd[pre + name + ".weight"]
        bound = math.sqrt(6.0 / (fo + fi))
        assert float(w.abs().max()) <= bound and float(w.abs().max()) > 0.9 * bound, name
        assert not sd[pre + name + ".bias"].any()
    assert torch.equal(sd[pre + "blocks.0.norm.weight"], torch.ones(128))
    assert not sd[pre + "blocks.0.norm.bias"].any()
    for name, fan_in in (("blocks.0.dwconv", 49), ("final_layer", 128)):
        bound = 1.0 / math.sqrt(fan_in)                                  # kaiming_uniform(a=sqrt(5)) and its bias rule
        w, b = sd[pre + name + ".weight"], sd[pre + name + ".bias"]
        assert float(w.abs().max()) <= bound and float(w.abs().max()) > 0.8 * bound, name
        assert float(b.abs().max()) <= bound and b.any(), name


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


def _adapter(num_classes=5, **kw):
    from multimae_b200.output_adapters import ConvNeXtAdapter
    kw = dict(dict(embed_dim=2048, preds_per_patch=16, depth=2), **kw)
    ad = ConvNeXtAdapter(num_classes, **kw)
    ad.init(dim_tokens_enc=128)
    return ad


CALLS = ["mmae_convnext_proj_forward", "mmae_convnext_block_forward", "mmae_convnext_block_forward",
         "mmae_convnext_tail_forward", "mmae_convnext_tail_backward", "mmae_convnext_block_backward",
         "mmae_convnext_block_backward", "mmae_convnext_proj_backward"]


@pytest.mark.parametrize("num_classes,preds_per_patch", [(5, 16), (150, 16), (8, 4)])
def test_entry_points_order_sizes_and_arena_pointers(rec, num_classes, preds_per_patch):
    ad = _adapter(num_classes, preds_per_patch=preds_per_patch, main_tasks=["depth", "rgb"]).train()
    s, C = int(math.isqrt(preds_per_patch)), 2048 // preds_per_patch
    x = torch.randn(3, 2 * 12 + 1, 128, requires_grad=True)
    out = ad(x, _info(48, 64, tasks=("rgb", "depth")))
    assert out.shape == (3, num_classes, 48, 64) and out.dtype == torch.float32
    out.sum().backward()
    names = [n for n in rec.names() if n.startswith("mmae_convnext") and not n.endswith("_bytes")]
    assert names == CALLS
    calls = [a for n, a in rec.calls if n.startswith("mmae_convnext") and not n.endswith("_bytes")]
    pf, bf0, bf1, tf, tb, bb1, bb0, pb = calls
    arena = ad._bound["arena"]
    v = lambda k: arena.views[k].data_ptr()                                     # noqa: E731
    # proj: B, N, D, n, tasks, starts (depth first: its tokens start at 12), E, weight
    assert list(pf[1:6]) == [3, 25, 128, 12, 2] and list(pf[6][:2]) == [12, 0] and pf[7] == 2048
    assert pf[0] == x.data_ptr() and pf[8] == ad.proj_dec.weight.data_ptr()
    assert list(pb[1:6]) == [3, 25, 128, 12, 2] and pb[9] == v("proj_dec.weight") and pb[10] == v("proj_dec.bias")
    assert pf[11] == pb[12]                                                     # the saved buffer travels to backward
    # blocks: B, nh, nw, s, C; parameter and gradient structs point at the block's own tensors / arena slots
    for i, (f, b) in enumerate(((bf0, bb0), (bf1, bb1))):
        assert list(f[2:7]) == [3, 3, 4, s, C] and f[7] == 1e-6 and list(b[3:8]) == [3, 3, 4, s, C]
        prm, grd = f[8], b[9]
        for j, name in enumerate(Fn.CONVNEXT_BLOCK_PARAM_NAMES):
            assert prm[j] == dict(ad.named_parameters())["blocks.%d.%s" % (i, name)].data_ptr()
            assert grd[j] == v("blocks.%d.%s" % (i, name)), (i, name)
        assert b[10] == f[9]
    assert bf1[0] == bf0[1] and bb1[2] == bb0[1]                                # x_out of block 0 feeds block 1, and back
    assert pf[10] == bf0[0] and tf[0] == bf1[1]
    # tail: the class count itself crosses the ABI (the library pads it to a multiple of 8 internally)
    assert list(tf[1:9]) == [3, 3, 4, s, C, num_classes, 48, 64] and list(tb[1:9]) == list(tf[1:9])
    assert tf[11] == out.data_ptr() and tb[10] == v("final_layer.weight") and tb[11] == v("final_layer.bias")
    assert ("mmae_convnext_tail_saved_bytes", (3, 3, 4, s, C, num_classes)) in rec.calls
    assert ("mmae_convnext_block_saved_bytes", (3, 3, 4, s, C)) in rec.calls
    for n, p in ad.named_parameters():
        assert torch.equal(p.grad, arena.views[n]), n
    assert x.grad is not None and x.grad.shape == x.shape


def test_model_reports_every_piece(rec):
    model = _model().train()
    seen = []
    model.set_grad_callback(lambda names: seen.append(list(names)))
    x, labels = inputs()
    outs = model(x)
    assert {k: tuple(v.shape) for k, v in outs.items()} == {"semseg": (2, 5, 48, 64), "aux": (2, 8, 48, 64)}
    (outs["semseg"].sum() + outs["aux"].sum()).backward()
    pre = "output_adapters.semseg."
    assert [pre + "final_layer.weight", pre + "final_layer.bias"] in seen
    assert [pre + "blocks.1." + n for n in Fn.CONVNEXT_BLOCK_PARAM_NAMES] in seen
    assert [pre + "blocks.0." + n for n in Fn.CONVNEXT_BLOCK_PARAM_NAMES] in seen
    assert [pre + "proj_dec.weight", pre + "proj_dec.bias"] in seen
    reported = [n for names in seen for n in names]
    assert sorted(reported) == sorted(n for n, p in model.named_parameters() if p.requires_grad)
    (pb,) = [a for n, a in rec.calls if n == "mmae_convnext_proj_backward" and a[5] == 2]
    assert pb[9] == model.grad_arena().views[pre + "proj_dec.weight"].data_ptr()


def test_no_grad_eval_saves_nothing(rec):
    model = _model().eval()
    x, _ = inputs()
    with torch.no_grad():
        outs = model(x)
    assert all(v.grad_fn is None for v in outs.values())
    buf = Fn.Workspace.get(0, torch.device("cpu"))
    lo, hi = buf.data_ptr(), buf.data_ptr() + buf.numel()
    pos = {"mmae_convnext_proj_forward": (11, 12), "mmae_convnext_block_forward": (9, 10),
           "mmae_convnext_tail_forward": (12, 13)}
    fwd = [(n, a) for n, a in rec.calls if n in pos]
    assert len(fwd) == 2 * 2 + 3
    for n, a in fwd:                                                    # saved and ws both in the stream's scratch buffer
        assert all(lo <= a[i] < hi for i in pos[n]), n
    assert not any("backward" in n for n in rec.names())


def test_errors():
    from multimae_b200.output_adapters import ConvNeXtAdapter
    with pytest.raises(NotImplementedError, match="multiple of 128"):
        ConvNeXtAdapter(41, embed_dim=1536, preds_per_patch=16)                  # the depth script's convnext: C = 96
    with pytest.raises(NotImplementedError, match="multiple of 128"):
        ConvNeXtAdapter(41, embed_dim=2048 * 16, preds_per_patch=16)             # C = 2048
    with pytest.raises(ValueError, match="perfect square"):
        ConvNeXtAdapter(41, embed_dim=6144, preds_per_patch=12)
    with pytest.raises(NotImplementedError, match="bilinear"):
        ConvNeXtAdapter(41, interpolate_mode="nearest")
    ad = _adapter(5, main_tasks=["rgb", "depth"])
    info = _info(48, 64, tasks=("rgb", "depth"))
    info["tasks"]["depth"]["end_idx"] -= 1
    with pytest.raises(ValueError, match="tokens"):
        ad(torch.zeros(1, 24, 128), info)
    with pytest.raises(NotImplementedError, match="return_all_layers"):
        ad([torch.zeros(1, 13, 128)], _info(48, 64))


def test_placeholder_adapters_raise():
    from multimae_b200.output_adapters import DPTOutputAdapter, SegmenterMaskTransformerAdapter
    with pytest.raises(NotImplementedError, match="SegmenterMaskTransformerAdapter"):
        SegmenterMaskTransformerAdapter(num_classes=150, depth=2, drop_path_rate=0.1, embed_dim=6144, patch_size=16)
    with pytest.raises(NotImplementedError, match="DPTOutputAdapter"):
        DPTOutputAdapter(stride_level=1, main_tasks=["rgb"], head_type="semseg", num_classes=150)


def test_overlay_resolves_the_semseg_adapters():
    code = ("import sys; sys.path.insert(0, %r); from multimae_b200 import overlay; overlay.install(); "
            "from multimae.output_adapters import ConvNeXtAdapter, DPTOutputAdapter, SegmenterMaskTransformerAdapter; "
            "import multimae_b200.output_adapters as O; assert ConvNeXtAdapter is O.ConvNeXtAdapter\n"
            "for cls in (DPTOutputAdapter, SegmenterMaskTransformerAdapter):\n"
            "    try:\n        cls(num_classes=3)\n    except NotImplementedError:\n        pass\n"
            "    else:\n        raise SystemExit(cls.__name__)\n"
            "print('ok')" % ROOT)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout + res.stderr


def test_semseg_script_model_setup_ade(rec):
    """run_finetuning_semseg.py:374-407 with the ADE config's values (cfgs/finetune/semseg/ade/ft_ade_64e_*.yaml):
    in_domains rgb, patch 16, 512 x 512, output_adapter convnext, decoder_dim 6144, decoder_preds_per_patch 16,
    decoder_depth 4, decoder_main_tasks rgb, 150 classes + void, drop_path_encoder 0.1 - through the overlay's
    `multimae.output_adapters` and the registered `multivit_base` factory."""
    code = r'''
import sys, types
from functools import partial
sys.path.insert(0, %r)
from multimae_b200 import overlay
overlay.install()
from multimae.input_adapters import PatchedInputAdapter
from multimae.output_adapters import ConvNeXtAdapter, DPTOutputAdapter, SegmenterMaskTransformerAdapter
from multimae import multimae as mm
args = types.SimpleNamespace(in_domains=["rgb"], patch_size=16, input_size=512, learnable_pos_emb=False,
                             model="multivit_base", output_adapter="convnext", decoder_depth=4, drop_path_decoder=0.0,
                             decoder_preds_per_patch=16, decoder_interpolate_mode="bilinear", decoder_main_tasks="rgb",
                             num_classes_with_void=151, decoder_dim=6144, drop_path_encoder=0.1)
DOMAIN_CONF = {"rgb": {"input_adapter": partial(PatchedInputAdapter, num_channels=3), "stride_level": 1}}
input_adapters = {
    domain: DOMAIN_CONF[domain]['input_adapter'](
        stride_level=DOMAIN_CONF[domain]['stride_level'],
        patch_size_full=args.patch_size,
        image_size=args.input_size,
        learnable_pos_emb=args.learnable_pos_emb,
    )
    for domain in args.in_domains
}
adapters_dict = {
    'segmenter': partial(SegmenterMaskTransformerAdapter, depth=args.decoder_depth, drop_path_rate=args.drop_path_decoder),
    'convnext': partial(ConvNeXtAdapter, preds_per_patch=args.decoder_preds_per_patch, depth=args.decoder_depth,
                        interpolate_mode=args.decoder_interpolate_mode, main_tasks=args.decoder_main_tasks.split('-')),
    'dpt': partial(DPTOutputAdapter, stride_level=1, main_tasks=args.decoder_main_tasks.split('-'), head_type='semseg'),
}
output_adapters = {
    'semseg': adapters_dict[args.output_adapter](
        num_classes=args.num_classes_with_void,
        embed_dim=args.decoder_dim, patch_size=args.patch_size,
    ),
}
model = mm.__dict__[args.model](input_adapters=input_adapters, output_adapters=output_adapters,
                                drop_path_rate=args.drop_path_encoder)
assert model.get_num_layers() == 12
assert "global_tokens" in model.no_weight_decay()
sd = model.state_dict()
assert tuple(sd["output_adapters.semseg.proj_dec.weight"].shape) == (6144, 768)
assert tuple(sd["output_adapters.semseg.blocks.3.dwconv.weight"].shape) == (384, 1, 7, 7)
assert tuple(sd["output_adapters.semseg.final_layer.weight"].shape) == (151, 384, 1, 1)
print("ok", sum(p.numel() for p in model.parameters()))
''' % ROOT
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout + res.stderr
