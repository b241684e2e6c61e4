"""CPU: the classification head of fine-tuning (LinearOutputAdapter, run_finetuning_cls.py) without a GPU.

1. The fp32 restatement (tests/cls_head_oracle.py) on the oracle encoder reproduces the reference's logits, loss and every
   parameter gradient, recorded by tests/golden/make_golden_cls.py, in both pooling modes.
2. A model built by our factory has the reference's state_dict schema and initialisation.
3. The host layer against a stub of the C library: entry points, sizes, gradient-arena pointers, on_grads_ready, no-grad.
4. The overlay resolves `multimae.output_adapters.LinearOutputAdapter`; MultiViT under AUTO_OWN_GRADIENTS."""
import math
import os
import subprocess
import sys
from functools import partial

import pytest
import torch

from cls_head_oracle import cls_head, encoder_tokens, soft_target_ce, vit_config
from helpers import load_fixture
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from oracle import multimae_oracle as O
from test_drop_path_host import _Rec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx(golden_dir):
    return load_fixture(golden_dir, "cls_head.pt")


def _build(num_classes=10, mean_pool=True, init_scale=1.0, dim=128, depth=2, heads=2, size=64, drop_path_rate=0.0):
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import LinearOutputAdapter
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=size),
           "depth": PatchedInputAdapter(num_channels=1, stride_level=1, patch_size_full=16, image_size=size)}
    outs = {"cls": LinearOutputAdapter(num_classes=num_classes, use_mean_pooling=mean_pool, init_scale=init_scale)}
    return MultiViT(ins, outs, num_global_tokens=1, dim_tokens=dim, depth=depth, num_heads=heads, mlp_ratio=4,
                    qkv_bias=True, drop_path_rate=drop_path_rate, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


@pytest.mark.parametrize("mode", ["mean", "last"])
def test_oracle_head_against_reference(fx, mode):
    c = fx["config"]
    cfg = vit_config(c["in_domains"], c["dim"], c["depth"], c["heads"], c["size"])
    p = {k: v.clone() for k, v in fx["state_dict"].items()}
    train = O.trainable(p)
    for v in train.values():
        v.requires_grad_(True)
    logits = cls_head(encoder_tokens(p, fx["inputs"], cfg), p, mean_pool=(mode == "mean"))
    torch.testing.assert_close(logits, fx["logits"][mode], rtol=1e-4, atol=1e-5)
    loss = soft_target_ce(logits, fx["target"])
    torch.testing.assert_close(loss, fx["loss"][mode], rtol=1e-5, atol=1e-6)
    loss.backward()
    ref = fx["grads_" + mode]
    assert set(ref) == {k for k, v in train.items() if v.grad is not None}
    for k, g in ref.items():
        torch.testing.assert_close(train[k].grad, g, rtol=2e-4, atol=2e-6, msg=lambda m, k=k: "%s: %s" % (k, m))


def test_factory_model_schema_and_init(fx):
    """Keys, order and shapes of the reference's state_dict; the head is re-initialised by the model (xavier-uniform, zero
    bias, LayerNorm 1 / 0) after LinearOutputAdapter.init, so init_scale changes nothing under the same seed."""
    torch.manual_seed(0)
    model = _build()
    sd = model.state_dict()
    assert list(sd) == list(fx["state_dict"])
    assert all(sd[k].shape == v.shape for k, v in fx["state_dict"].items())
    w, b = sd["output_adapters.cls.head.weight"], sd["output_adapters.cls.head.bias"]
    bound = math.sqrt(6.0 / (10 + 128))
    assert float(w.abs().max()) <= bound and float(w.abs().max()) > 0.9 * bound
    assert abs(float(w.std()) - bound / math.sqrt(3)) < 0.1 * bound
    assert torch.equal(b, torch.zeros(10))
    assert torch.equal(sd["output_adapters.cls.norm.weight"], torch.ones(128))
    assert torch.equal(sd["output_adapters.cls.norm.bias"], torch.zeros(128))
    torch.manual_seed(0)
    other = _build(init_scale=1e-3).state_dict()
    assert all(torch.equal(other[k], v) for k, v in sd.items())
    # stand-alone, the adapter keeps the reference's own initialisation: trunc_normal(0.02) x init_scale
    from multimae_b200.output_adapters import LinearOutputAdapter
    torch.manual_seed(0)
    ad = LinearOutputAdapter(10, dim_tokens_enc=128, init_scale=0.5)
    assert 0.008 < float(ad.head.weight.detach().std()) < 0.012 and not ad.head.bias.detach().any()
    assert ad.get_classifier() is ad.head
    ident = LinearOutputAdapter(0, dim_tokens_enc=128)
    assert isinstance(ident.head, torch.nn.Identity) and list(ident.state_dict()) == ["norm.weight", "norm.bias"]


@pytest.fixture()
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(L, "lib", lambda: r)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    return r


# argument positions of mmae_clshead_forward / _backward (include/multimae_b200.h)
FWD = dict(x=0, B=1, N=2, D=3, C=4, mean_pool=5, eps=6, norm_w=7, norm_b=8, head_w=9, head_b=10, out=11, saved=12, ws=13)
BWD = dict(dout=0, B=1, N=2, D=3, C=4, mean_pool=5, norm_w=6, head_w=7, d_norm_w=8, d_norm_b=9, d_head_w=10, d_head_b=11,
           dx=12, saved=13, ws=14)


@pytest.mark.parametrize("num_classes,mean_pool", [(10, True), (101, False), (0, True)])
def test_entry_points_sizes_and_arena_pointers(rec, num_classes, mean_pool):
    from multimae_b200.output_adapters import LinearOutputAdapter
    ad = LinearOutputAdapter(num_classes, dim_tokens_enc=128, use_mean_pooling=mean_pool).train()
    x = torch.randn(3, 9, 128, requires_grad=True)
    out = ad(x)
    assert out.shape == (3, num_classes if num_classes else 128) and out.dtype == torch.float32
    out.sum().backward()
    (f,) = [a for n, a in rec.calls if n == "mmae_clshead_forward"]
    (g,) = [a for n, a in rec.calls if n == "mmae_clshead_backward"]
    for args, pos in ((f, FWD), (g, BWD)):
        assert [args[pos[k]] for k in ("B", "N", "D", "C", "mean_pool")] == [3, 9, 128, num_classes, int(mean_pool)]
        assert args[pos["norm_w"]] == ad.norm.weight.data_ptr()
        assert args[pos["head_w"]] == (ad.head.weight.data_ptr() if num_classes else None)
    assert f[FWD["eps"]] == 1e-6 and f[FWD["x"]] == x.data_ptr() and f[FWD["out"]] == out.data_ptr()
    assert f[FWD["saved"]] == g[BWD["saved"]]
    assert ("mmae_clshead_saved_bytes", (3, 9, 128, num_classes)) in rec.calls
    arena = ad._bound["arena"]
    for k in ("norm.weight", "norm.bias") + (("head.weight", "head.bias") if num_classes else ()):
        assert g[BWD["d_" + k.replace(".weight", "_w").replace(".bias", "_b")]] == arena.views[k].data_ptr(), k
        assert torch.equal(dict(ad.named_parameters())[k].grad, arena.views[k])
    if not num_classes:
        assert g[BWD["d_head_w"]] is None and g[BWD["d_head_b"]] is None
    assert x.grad is not None and x.grad.shape == x.shape


def test_model_reports_the_four_head_gradients(rec):
    model = _build().train()
    seen = []
    model.set_grad_callback(lambda names: seen.append(list(names)))
    x = {"rgb": torch.randn(2, 3, 64, 64), "depth": torch.randn(2, 1, 64, 64)}
    model(x)["cls"].sum().backward()
    head = ["output_adapters.cls.%s" % n for n in Fn.CLS_PARAM_NAMES]
    assert head in seen
    reported = [n for names in seen for n in names]
    assert sorted(reported) == sorted(n for n, p in model.named_parameters() if p.requires_grad)
    (g,) = [a for n, a in rec.calls if n == "mmae_clshead_backward"]
    arena = model.grad_arena()
    assert g[BWD["d_head_w"]] == arena.views["output_adapters.cls.head.weight"].data_ptr()


def test_no_grad_eval_saves_nothing(rec):
    model = _build().eval()
    x = {"rgb": torch.randn(5, 3, 64, 64), "depth": torch.randn(5, 1, 64, 64)}
    with torch.no_grad():
        out = model(x)["cls"]
    assert out.grad_fn is None and out.shape == (5, 10)
    (f,) = [a for n, a in rec.calls if n == "mmae_clshead_forward"]
    buf = Fn.Workspace.get(0, torch.device("cpu"))
    lo, hi = buf.data_ptr(), buf.data_ptr() + buf.numel()
    assert lo <= f[FWD["saved"]] < hi and lo <= f[FWD["ws"]] < hi          # scratch, not a tensor kept for backward
    assert "mmae_clshead_backward" not in rec.names()
    with pytest.raises(NotImplementedError, match="return_all_layers"):
        model.output_adapters["cls"]([torch.zeros(1, 3, 128)])


def test_reset_classifier(rec):
    """Stand-alone: a new head for the new class count.  Inside a model whose gradient arena exists: a clear error, and
    the adapter is left as it was (no stale gradient slots)."""
    from multimae_b200.output_adapters import LinearOutputAdapter
    ad = LinearOutputAdapter(10, dim_tokens_enc=128)
    ad(torch.randn(2, 4, 128, requires_grad=True)).sum().backward()
    ad.reset_classifier(37)
    assert ad.num_classes == 37 and ad.head.weight.shape == (37, 128)
    rec.calls.clear()
    ad(torch.randn(2, 4, 128, requires_grad=True)).sum().backward()
    (g,) = [a for n, a in rec.calls if n == "mmae_clshead_backward"]
    assert g[BWD["C"]] == 37 and g[BWD["d_head_w"]] == ad._bound["arena"].views["head.weight"].data_ptr()
    assert ad._bound["arena"].views["head.weight"].shape == (37, 128)
    model = _build()
    model.output_adapters["cls"].reset_classifier(5)                   # before the first forward: fine
    assert model.output_adapters["cls"].head.weight.shape == (5, 128)
    model.grad_arena()
    with pytest.raises(RuntimeError, match="gradient arena"):
        model.output_adapters["cls"].reset_classifier(7)
    assert model.output_adapters["cls"].num_classes == 5
    assert model.output_adapters["cls"].head.weight.shape == (5, 128)


def test_multivit_auto_own_gradients(rec, monkeypatch):
    from multimae_b200 import multimae as mm
    monkeypatch.setattr(mm, "AUTO_OWN_GRADIENTS", True)
    model = _build(drop_path_rate=0.1).train()
    x = {"rgb": torch.randn(2, 3, 64, 64), "depth": torch.randn(2, 1, 64, 64)}
    model(x)["cls"].sum().backward()
    arena = model.grad_arena()
    assert arena.owned
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and p.grad.data_ptr() == arena.views[n].data_ptr(), n
    assert Fn.find_arena_for(list(model.parameters())) is arena
    # gradient accumulation: the next training forward keeps the arena while `accumulating` is set, else zeroes it
    arena.flat.fill_(1.0)
    arena.accumulating = True
    model(x)
    assert float(arena.flat[0]) == 1.0
    arena.accumulating = False
    model(x)
    assert float(arena.flat.abs().sum()) == 0.0


def test_overlay_resolves_linear_output_adapter():
    code = ("import sys; sys.path.insert(0, %r); from multimae_b200 import overlay; overlay.install(); "
            "from multimae.output_adapters import LinearOutputAdapter; from multimae import multimae as mm; "
            "import multimae_b200.output_adapters as O; assert LinearOutputAdapter is O.LinearOutputAdapter; "
            "assert mm.AUTO_OWN_GRADIENTS and 'multivit_base' in mm.__all__; print('ok')" % ROOT)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout + res.stderr
