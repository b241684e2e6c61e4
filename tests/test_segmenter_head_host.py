"""CPU: the Segmenter head of semantic-segmentation fine-tuning (SegmenterMaskTransformerAdapter,
run_finetuning_semseg.py --output_adapter segmenter) without a GPU.

1. The fp32 restatement (tests/segmenter_head_oracle.py) on the oracle encoder reproduces the reference's outputs, loss and
   every parameter gradient, recorded by tests/golden/make_golden_segmenter.py.
2. A model built by our factory has the reference's state_dict schema; the adapter has its constructor signature.
3. The host layer against a stub of the C library: entry points and their order, sizes, gradient-arena pointers,
   on_grads_ready, no-grad, drop-path rates, and the errors raised for what the CUDA head does not cover."""
import inspect

import pytest
import torch

from cls_head_oracle import encoder_tokens, vit_config
from helpers import load_fixture
from multimae_b200 import functional as Fn
from segmenter_head_oracle import CONFIG, build, fill_, inputs, seg_loss, segmenter_head
from test_convnext_head_host import _info, assert_digest_close, rec  # noqa: F401  (rec: the library stub fixture)


@pytest.fixture(scope="module")
def fx(golden_dir):
    return load_fixture(golden_dir, "segmenter_head.pt")


def _model():
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import SegmenterMaskTransformerAdapter
    return build(MultiViT, PatchedInputAdapter, SegmenterMaskTransformerAdapter)


def oracle_outputs(p, x, c=CONFIG):
    """Both heads of the fixture model through the oracle encoder + the fp32 restatement."""
    enc = encoder_tokens(p, x, vit_config(c["in_domains"], c["dim"], c["depth"], c["heads"], 64))
    n = (c["H"] // 16) * (c["W"] // 16)
    start = {"rgb": 0, "depth": n}
    return {k: segmenter_head(enc, p, [start[t] for t in a["main_tasks"]], n, c["H"], c["W"], a["depth"], a["num_heads"],
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
        torch.testing.assert_close(outs[k], ref, rtol=1e-4, atol=2e-5, msg=lambda m, k=k: "%s: %s" % (k, m))
    loss = seg_loss(outs, fx["labels"])
    torch.testing.assert_close(loss, fx["loss"], rtol=1e-5, atol=1e-6)
    loss.backward()
    assert set(fx["grads"]) == {k for k, v in train.items() if v.grad is not None}
    for k, ref in fx["grads"].items():
        assert_digest_close(train[k].grad, ref, 5e-4, k)


def test_fixture_inputs_are_the_recorded_ones(fx):
    x, labels = inputs()
    assert all(torch.equal(x[k], fx["inputs"][k]) for k in x)
    assert all(torch.equal(labels[k], fx["labels"][k]) for k in labels)


def test_schema_signature_and_state_dict_round_trip(fx):
    from multimae_b200.output_adapters import SegmenterMaskTransformerAdapter as A
    sd = _model().state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [(k, tuple(s)) for k, s in fx["schema"]]
    pre = "output_adapters.semseg."
    keys = [k[len(pre):] for k in sd if k.startswith(pre)]
    assert keys[:3] == ["cls_emb", "patch_proj.weight", "classes_proj.weight"]
    assert keys[-6:] == ["decoder_norm.weight", "decoder_norm.bias", "mask_norm.weight", "mask_norm.bias", "proj_dec.weight",
                         "proj_dec.bias"]
    assert tuple(sd[pre + "cls_emb"].shape) == (1, 9, 128) and tuple(sd[pre + "mask_norm.weight"].shape) == (9,)
    other = _model()
    other.load_state_dict(sd, strict=True)
    sig = inspect.signature(A.__init__)
    assert list(sig.parameters)[1:] == ["num_classes", "depth", "num_heads", "embed_dim", "mlp_ratio", "drop_path_rate",
                                        "drop_rate", "attn_drop_rate", "qkv_bias", "main_tasks", "patch_size", "norm_layer",
                                        "kwargs"]
    d = {k: v.default for k, v in sig.parameters.items()}
    assert (d["depth"], d["num_heads"], d["embed_dim"], d["mlp_ratio"], d["drop_path_rate"], d["patch_size"]) == \
        (2, 12, 768, 4, 0.1, 16)
    # stand-alone initialisation: trunc_normal(0.02) for cls_emb and the Linear weights, zero biases, LayerNorm 1 / 0
    torch.manual_seed(0)
    ad = A(41)
    ad.init(768)
    for w in (ad.cls_emb, ad.patch_proj.weight, ad.proj_dec.weight, ad.blocks[1].mlp.fc1.weight):
        assert 0.015 < float(w.std()) < 0.025 and float(w.abs().max()) <= 2.0
    assert ad.patch_proj.bias is None and ad.classes_proj.bias is None and not ad.proj_dec.bias.any()
    assert torch.equal(ad.mask_norm.weight, torch.ones(41)) and not ad.decoder_norm.bias.any()


def _adapter(num_classes=13, **kw):
    from multimae_b200.output_adapters import SegmenterMaskTransformerAdapter
    kw = dict(dict(embed_dim=128, num_heads=4, depth=2, drop_path_rate=0.0), **kw)
    ad = SegmenterMaskTransformerAdapter(num_classes, **kw)
    ad.init(dim_tokens_enc=128)
    return ad


@pytest.mark.parametrize("num_classes", [8, 13, 151])
def test_entry_points_order_sizes_and_arena_pointers(rec, num_classes):  # noqa: F811
    ad = _adapter(num_classes, main_tasks=["depth", "rgb"]).train()
    x = torch.randn(3, 2 * 12 + 1, 128, requires_grad=True)
    out = ad(x, _info(48, 64, tasks=("rgb", "depth")))
    assert out.shape == (3, num_classes, 48, 64) and out.dtype == torch.float32
    out.sum().backward()
    names = [n for n in rec.names() if n.startswith(("mmae_segmenter", "mmae_block")) and not n.endswith("_bytes")
             and "saved_x_mid" not in n]
    assert names[0] == "mmae_segmenter_proj_forward" and names[-1] == "mmae_segmenter_proj_backward"
    mid = names[1:-1]
    k = mid.index("mmae_segmenter_tail_forward")
    assert mid[k + 1] == "mmae_segmenter_tail_backward"
    assert all(n.startswith("mmae_block") and "forward" in n for n in mid[:k]) and len(mid[:k]) >= 1
    assert all(n.startswith("mmae_block") and "backward" in n for n in mid[k + 2:]) and len(mid[k + 2:]) == len(mid[:k])
    calls = dict((n, a) for n, a in rec.calls if n.startswith("mmae_segmenter") and not n.endswith("_bytes"))
    pf, pb = calls["mmae_segmenter_proj_forward"], calls["mmae_segmenter_proj_backward"]
    tf, tb = calls["mmae_segmenter_tail_forward"], calls["mmae_segmenter_tail_backward"]
    arena = ad._bound["arena"]
    v = lambda k: arena.views[k].data_ptr()                                     # noqa: E731
    # proj: B, N, D, n, tasks, starts (depth first: its tokens start at 12), E, K, weight, bias, cls_emb
    assert list(pf[1:6]) == [3, 25, 128, 12, 2] and list(pf[6][:2]) == [12, 0] and list(pf[7:9]) == [128, num_classes]
    assert pf[0] == x.data_ptr() and pf[9] == ad.proj_dec.weight.data_ptr() and pf[11] == ad.cls_emb.data_ptr()
    assert list(pb[1:6]) == [3, 25, 128, 12, 2] and list(pb[7:9]) == [128, num_classes]
    assert [pb[10], pb[11], pb[12]] == [v("proj_dec.weight"), v("proj_dec.bias"), v("cls_emb")]
    assert pf[13] == pb[14]                                                     # the saved buffer travels to backward
    # tail: B, nh, nw, E, K, H, W, the two eps; parameter and gradient arrays in SEGMENTER_TAIL_PARAM_NAMES order
    assert list(tf[1:8]) == [3, 3, 4, 128, num_classes, 48, 64] and tf[8] == 1e-6 and tf[9] == 1e-6
    assert list(tb[3:10]) == [3, 3, 4, 128, num_classes, 48, 64] and tb[0] == tf[0] and tf[11] == out.data_ptr()
    params = dict(ad.named_parameters())
    for j, name in enumerate(Fn.SEGMENTER_TAIL_PARAM_NAMES):
        assert tf[10][j] == params[name].data_ptr() and tb[10][j] == params[name].data_ptr() and tb[11][j] == v(name), name
    assert tb[12] == tf[12]
    assert ("mmae_segmenter_tail_saved_bytes", (3, 3, 4, 128, num_classes)) in rec.calls
    for n, p in ad.named_parameters():
        assert torch.equal(p.grad, arena.views[n]), n
    assert x.grad is not None and x.grad.shape == x.shape


def test_model_reports_every_piece(rec):  # noqa: F811
    model = _model().train()
    seen = []
    model.set_grad_callback(lambda names: seen.append(list(names)))
    x, _ = inputs()
    outs = model(x)
    assert {k: tuple(v.shape) for k, v in outs.items()} == {"semseg": (2, 9, 48, 64), "aux": (2, 13, 48, 64)}
    (outs["semseg"].sum() + outs["aux"].sum()).backward()
    pre = "output_adapters.semseg."
    assert [pre + n for n in Fn.SEGMENTER_TAIL_PARAM_NAMES] in seen
    assert [pre + "proj_dec.weight", pre + "proj_dec.bias", pre + "cls_emb"] in seen
    reported = [n for names in seen for n in names]
    assert sorted(reported) == sorted(n for n, p in model.named_parameters() if p.requires_grad)
    (pb,) = [a for n, a in rec.calls if n == "mmae_segmenter_proj_backward" and a[5] == 2]
    assert pb[12] == model.grad_arena().views[pre + "cls_emb"].data_ptr()


def test_no_grad_eval_saves_nothing(rec):  # noqa: F811
    model = _model().eval()
    x, _ = inputs()
    with torch.no_grad():
        outs = model(x)
    assert all(v.grad_fn is None for v in outs.values())
    buf = Fn.Workspace.get(0, torch.device("cpu"))
    lo, hi = buf.data_ptr(), buf.data_ptr() + buf.numel()
    pos = {"mmae_segmenter_proj_forward": (13, 14), "mmae_segmenter_tail_forward": (12, 13)}
    fwd = [(n, a) for n, a in rec.calls if n in pos]
    assert len(fwd) == 4
    for n, a in fwd:                                                    # saved and ws both in the stream's scratch buffer
        assert all(lo <= a[i] < hi for i in pos[n]), n
    assert not any("backward" in n for n in rec.names())


def test_drop_path_and_dropout_rates_reach_the_blocks():
    ad = _adapter(13, depth=3, drop_path_rate=0.2, drop_rate=0.1, attn_drop_rate=0.05).train()
    assert [round(Fn.drop_path_prob(b), 6) for b in ad.blocks] == [0.0, 0.1, 0.2]
    assert all(b.attn.attn_drop.p == 0.05 and b.attn.proj_drop.p == 0.1 and b.mlp.drop.p == 0.1 for b in ad.blocks)
    assert [Fn.drop_path_prob(b) for b in ad.eval().blocks] == [0.0, 0.0, 0.0]


def test_errors():
    from multimae_b200.output_adapters import DPTOutputAdapter
    from multimae_b200.output_adapters import SegmenterMaskTransformerAdapter as A
    name = "SegmenterMaskTransformerAdapter"
    with pytest.raises(NotImplementedError, match=name + ".*--decoder_dim 768"):
        A(151, embed_dim=6144)                                          # the script's default --decoder_dim: heads of 512
    with pytest.raises(NotImplementedError, match=name):
        A(151, embed_dim=1536, num_heads=24)                            # above 1024
    with pytest.raises(NotImplementedError, match=name):
        A(151, embed_dim=192, num_heads=6)                              # not a multiple of 128
    with pytest.raises(NotImplementedError, match=name):
        A(151, embed_dim=768, num_heads=6)                              # heads of 128
    for k in (3, 7, 257):
        with pytest.raises(NotImplementedError, match=name + ".*8 to 256"):
            A(k)
    with pytest.raises(NotImplementedError, match="DPTOutputAdapter"):
        DPTOutputAdapter(num_classes=41)
    ad = _adapter(13, main_tasks=["rgb", "depth"])
    info = _info(48, 64, tasks=("rgb", "depth"))
    info["tasks"]["depth"]["end_idx"] -= 1
    with pytest.raises(ValueError, match="tokens"):
        ad(torch.zeros(1, 24, 128), info)
    with pytest.raises(NotImplementedError, match="return_all_layers"):
        ad([torch.zeros(1, 13, 128)], _info(48, 64))
