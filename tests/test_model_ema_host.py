"""CPU: the model EMA of classification fine-tuning (run_finetuning_cls.py --model_ema, multimae_b200/model_ema.py) without
a GPU.

1. Through the overlay, utils.ModelEma / utils.model_ema.ModelEma / utils.model.ModelEma are the package's class, and
   utils.save_model then auto_load_model with --model_ema print and restore what they do with the reference's class
   (the reference's utils package is played by the stand-in under tests/ema_standin).
2. The host layer against a stub of the C library: one mmae_ema_update per update() carrying every state_dict pair of a
   multivit_base + 1000-class model in order, the ctypes arrays reused while the pointers hold; the stand-in for
   DistributedDataParallel is unwrapped (the reference's ModelEma raises KeyError on it); device='cpu' calls nothing.
3. The EMA copy shares nothing with the live model's training machinery.
4. The C entry point refuses bad arguments before any launch."""
import ctypes
import importlib.util
import os
import subprocess
import sys

import pytest
import torch

from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from test_drop_path_host import _Rec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STANDIN = os.path.join(ROOT, "tests", "ema_standin")


def _reference_model_ema():
    """The reference's ModelEma (stand-in restatement), loaded without putting a `utils` package on sys.path."""
    spec = importlib.util.spec_from_file_location("_ref_model_ema", os.path.join(STANDIN, "utils", "model_ema.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.ModelEma


def _cls_model(base=False, num_classes=37):
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    from multimae_b200.output_adapters import LinearOutputAdapter
    if base:
        return multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16,
                                                         image_size=224)}, {"cls": LinearOutputAdapter(1000)})
    from test_cls_head_host import _build
    return _build(num_classes=num_classes)


@pytest.fixture()
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(L, "lib", lambda: r)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    return r


def _ema_calls(rec):
    return [a for n, a in rec.calls if n == "mmae_ema_update"]


def test_one_call_per_update_with_every_pair_in_state_dict_order(rec):
    from multimae_b200.model_ema import ModelEma
    torch.manual_seed(0)
    model = _cls_model(base=True)
    ema = ModelEma(model)                                  # the script's default decay
    msd, esd = model.state_dict(), ema.ema.state_dict()
    assert len(esd) == 152 and sum(v.numel() for v in esd.values()) == 86_566_888
    assert sum(p.numel() for p in model.parameters() if p.requires_grad) == 86_416_360
    assert list(esd) == list(msd) and all(esd[k].shape == msd[k].shape for k in msd)
    ema.update(model)
    (args,) = _ema_calls(rec)
    dst, src, sizes, count, d, omd, stream = args
    assert count == 152 and stream == 0
    assert list(dst) == [v.data_ptr() for v in esd.values()]
    assert list(src) == [v.data_ptr() for v in msd.values()]
    assert list(sizes) == [v.numel() for v in msd.values()]
    assert d == 0.9999 and omd == 1.0 - 0.9999                     # the double subtraction; ctypes rounds both to fp32
    assert not set(dst) & set(src)                                 # the copy owns its storage
    # the arrays are reused while every pointer holds ...
    ema.update(model)
    assert [a[:3] for a in _ema_calls(rec)][1] == args[:3] and all(x is y for x, y in zip(_ema_calls(rec)[1], args[:3]))
    # ... and rebuilt after one changes
    head = model.output_adapters["cls"].head
    head.weight.data = head.weight.data.clone()
    ema.update(model)
    third = _ema_calls(rec)[2]
    assert third[1] is not args[1]
    i = list(msd).index("output_adapters.cls.head.weight")
    assert third[1][i] == head.weight.data_ptr() and list(third[1])[:i] == list(src)[:i]
    assert [n for n, _ in rec.calls] == ["mmae_ema_update"] * 3


def test_identity_ddp_is_unwrapped(rec):
    """run_finetuning_cls.py wraps the model in DistributedDataParallel after building the EMA; the overlay's stand-in
    forwards state_dict() without the 'module.' prefix the reference's ModelEma then looks for."""
    from multimae_b200 import overlay
    from multimae_b200.model_ema import ModelEma
    torch.manual_seed(0)
    model = _cls_model()
    ema, ref = ModelEma(model, decay=0.5), _reference_model_ema()(model, decay=0.5)
    wrapped = overlay._IdentityDDP(model, device_ids=[0])
    assert isinstance(wrapped, overlay._Wrapped) and wrapped.module is model
    with pytest.raises(KeyError, match="module."):
        ref.update(wrapped)
    ema.update(wrapped)
    (args,) = _ema_calls(rec)
    assert list(args[1]) == [v.data_ptr() for v in model.state_dict().values()]


def test_cpu_device_runs_the_host_loop(rec):
    """--model_ema_force_cpu: the reference's torch loop on the host, no library call; equal to the reference class."""
    from multimae_b200.model_ema import ModelEma
    torch.manual_seed(0)
    model = _cls_model()
    ema, ref = ModelEma(model, decay=0.9, device="cpu"), _reference_model_ema()(model, decay=0.9, device="cpu")
    g = torch.Generator().manual_seed(1)
    for _ in range(3):
        with torch.no_grad():
            for p in model.parameters():
                p.add_(torch.randn(p.shape, generator=g))
        ema.update(model)
        ref.update(model)
    assert rec.calls == []
    e, r = ema.ema.state_dict(), ref.ema.state_dict()
    assert list(e) == list(r) and all(torch.equal(e[k], r[k]) for k in e)
    assert not torch.equal(e["global_tokens"], model.global_tokens)


def test_copy_shares_nothing_with_the_training_machinery(rec, monkeypatch):
    """An EMA built from a model that has already trained (gradient arena owned by p.grad, bound blocks and heads, a
    data-parallel reducer, a cached position table) gets none of it, and the live model keeps all of it."""
    from multimae_b200 import multimae as mm
    from multimae_b200.model_ema import ModelEma
    monkeypatch.setattr(mm, "AUTO_OWN_GRADIENTS", True)
    model = _cls_model().train()
    x = {"rgb": torch.randn(2, 3, 64, 64), "depth": torch.randn(2, 1, 64, 64)}
    model(x)["cls"].sum().backward()
    arena = model.grad_arena()
    reducer = object()
    model._mmae_reducer = reducer
    model.input_adapters["rgb"]._resized_pos(4, 4, "bicubic")
    model.set_grad_callback(lambda names: None)
    ema = ModelEma(model)
    copy = ema.ema
    assert copy.training is False and all(not p.requires_grad for p in copy.parameters())
    assert all(p.grad is None for p in copy.parameters())
    assert copy._arena is None and copy._grad_callback is None and not hasattr(copy, "_mmae_reducer")
    assert all(blk._meta is None for blk in copy.encoder)
    assert copy.output_adapters["cls"]._bound is None and copy.output_adapters["cls"]._own_arena is False
    assert not any("_pos_cache" in m.__dict__ for m in copy.modules())
    live = {p.data_ptr() for p in model.parameters()} | {arena.flat.data_ptr()}
    assert not live & {v.data_ptr() for v in copy.state_dict().values()}
    msd, esd = model.state_dict(), copy.state_dict()
    assert list(esd) == list(msd) and all(torch.equal(esd[k], msd[k]) for k in msd)
    # the live model is untouched
    assert model._arena is arena and model._mmae_reducer is reducer and model._grad_callback is not None
    assert all(blk._meta is not None and blk._meta["arena"] is arena for blk in model.encoder)
    assert "_pos_cache" in model.input_adapters["rgb"].__dict__
    assert all(p.grad is not None and p.grad.data_ptr() == arena.views[n].data_ptr()
               for n, p in model.named_parameters() if p.requires_grad)
    # the copy runs on its own: a no-grad eval forward binds a private arena, not the live one
    with torch.no_grad():
        copy(x)
    assert copy._arena is not None and copy._arena is not arena


def test_refuses_non_fp32_entries(rec):
    from multimae_b200.model_ema import ModelEma
    model = torch.nn.Linear(4, 4).to(torch.float64)
    with pytest.raises(TypeError, match="fp32"):
        ModelEma(model).update(model)
    assert rec.calls == []


def test_entry_point_validates_before_any_launch():
    lib = L.lib()
    P, N = ctypes.c_void_p * 2, ctypes.c_int64 * 2
    before = lib.mmae_launch_count()
    cases = [
        (lambda: lib.mmae_ema_update(P(16, 32), P(48, 64), N(4, -1), 2, 0.5, 0.5, None), b"segment 1: negative size"),
        (lambda: lib.mmae_ema_update(P(16, None), P(48, 64), N(4, 4), 2, 0.5, 0.5, None), b"segment 1: null pointer"),
        (lambda: lib.mmae_ema_update(P(16, 32), P(48, None), N(4, 4), 2, 0.5, 0.5, None), b"segment 1: null pointer"),
        (lambda: lib.mmae_ema_update(P(16, 32), P(48, 64), N(4, 4), 2, float("nan"), 0.5, None), b"non-finite decay"),
        (lambda: lib.mmae_ema_update(P(16, 32), P(48, 64), N(4, 4), 2, 0.5, float("inf"), None), b"non-finite decay"),
        (lambda: lib.mmae_ema_update(None, None, None, 3, 0.5, 0.5, None), b"bad args"),
        (lambda: lib.mmae_ema_update(P(16, 32), P(48, 64), N(4, 4), -1, 0.5, 0.5, None), b"bad args"),
    ]
    for call, msg in cases:
        assert call() == 1
        assert msg in lib.mmae_last_error(), (msg, lib.mmae_last_error())
    # nothing to do: no launch, no error (an empty list, or only empty tensors, whose pointers may be null)
    assert lib.mmae_ema_update(None, None, None, 0, 0.5, 0.5, None) == 0
    assert lib.mmae_ema_update(P(None, None), P(None, None), N(0, 0), 2, 0.5, 0.5, None) == 0
    assert lib.mmae_launch_count() == before
    with pytest.raises(L.MmaeError, match="non-finite decay"):
        L.check(lib.mmae_ema_update(P(16, 32), P(48, 64), N(4, 4), 2, float("nan"), 0.5, None), "mmae_ema_update")


# one process per run: the overlay rewires sys.modules, torch.load and DistributedDataParallel
_CHECKPOINT_RUN = r"""
import argparse, contextlib, io, sys
import torch
sys.path.insert(0, %(root)r)
sys.path.insert(0, %(standin)r)
from multimae_b200 import overlay
if %(overlay)r:
    overlay.install()
else:
    overlay._legacy_checkpoint_load()          # the torch-version shim alone: checkpoints hold an argparse Namespace
import utils, utils.model, utils.model_ema
from multimae_b200.model_ema import ModelEma as Ours
if %(overlay)r:
    assert utils.ModelEma is Ours and utils.model_ema.ModelEma is Ours and utils.model.ModelEma is Ours
else:
    assert utils.ModelEma is not Ours


class Scaler:
    def state_dict(self):
        return {"scale": 1024.0}

    def load_state_dict(self, sd):
        print("scaler", sd)


def build(seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.LayerNorm(5), torch.nn.Linear(5, 3))


def digest(sd):
    return [(k, tuple(v.shape), v.double().sum().item(), v.double().abs().sum().item()) for k, v in sd.items()]


out = %(out)r
model = build(0)
ema = utils.ModelEma(model, decay=0.75, device="cpu")
assert utils.unwrap_model(ema) is ema.ema
opt = torch.optim.AdamW(model.parameters(), lr=0.1)
for step in range(3):
    model(torch.randn(4, 6)).square().sum().backward()
    opt.step()
    opt.zero_grad()
    ema.update(model)
args = argparse.Namespace(output_dir=out, auto_resume=True, resume="", model_ema=True, start_epoch=0)
utils.save_model(args=args, epoch=2, model=model, model_without_ddp=model, optimizer=opt, loss_scaler=Scaler(),
                 model_ema=ema)
saved = torch.load(out + "/checkpoint-2.pth")
assert list(saved["model_ema"]) == list(ema.ema.state_dict())
assert all(torch.equal(saved["model_ema"][k], v) for k, v in ema.ema.state_dict().items())
print("ema", digest(ema.ema.state_dict()))
# a resumed run: the script builds the model and its EMA, then auto_load_model
model2 = build(1)
ema2 = utils.ModelEma(model2, decay=0.75, device="cpu")
built = {k: v.clone() for k, v in ema2.ema.state_dict().items()}
opt2 = torch.optim.AdamW(model2.parameters(), lr=0.1)
text = io.StringIO()
with contextlib.redirect_stdout(text):
    utils.auto_load_model(args=args, model=model2, model_without_ddp=model2, optimizer=opt2, loss_scaler=Scaler(),
                          model_ema=ema2)
print(text.getvalue().replace(out, "<out>"), end="")
assert "Failed to find state_dict_ema, starting from loaded model weights" in text.getvalue()
assert all(torch.equal(v, built[k]) for k, v in ema2.ema.state_dict().items())
assert all(torch.equal(v, model.state_dict()[k]) for k, v in model2.state_dict().items())
print("start_epoch", args.start_epoch)
# the call that does load: a dict with 'state_dict_ema'
text = io.StringIO()
with contextlib.redirect_stdout(text):
    utils.checkpoint._load_checkpoint_for_ema(ema2, {"state_dict_ema": saved["model_ema"]})
print(text.getvalue(), end="")
assert all(torch.equal(v, saved["model_ema"][k]) for k, v in ema2.ema.state_dict().items())
print("ok")
"""


def test_overlay_checkpoint_round_trip_matches_the_reference(tmp_path):
    """The same script run with the overlay's ModelEma and with the reference's: identical output, messages included."""
    outputs = []
    for use_overlay in (True, False):
        out = tmp_path / ("overlay" if use_overlay else "reference")
        out.mkdir()
        code = _CHECKPOINT_RUN % dict(root=ROOT, standin=STANDIN, overlay=use_overlay, out=str(out))
        res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0 and res.stdout.endswith("ok\n"), res.stdout + res.stderr[-3000:]
        outputs.append(res.stdout)
    assert outputs[0] == outputs[1], outputs
    assert "Failed to find state_dict_ema" in outputs[0] and "Loaded state_dict_ema" in outputs[0]
