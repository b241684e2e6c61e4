"""GPU: the model EMA of classification fine-tuning (run_finetuning_cls.py --model_ema) through mmae_ema_update.

The EMA is held bitwise to the reference's update `ema_v.copy_(ema_v * decay + (1. - decay) * model_v)`, restated here
and run with torch on the same GPU tensors: for multivit_base + 1000 classes, for a small model with odd-sized tensors,
and for direct calls with unaligned views and more segments than one launch holds.  Nothing here reads the reference
checkout; the reference's utils package is played by the stand-in under tests/ema_standin."""
import ctypes
import math
import os
import sys

import pytest
import torch

from cls_head_oracle import soft_target_ce
from test_cuda_cls_head import _mixup, _param_groups, _small

pytestmark = pytest.mark.gpu

STANDIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ema_standin")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _lib():
    from multimae_b200 import _lib as L
    return L.lib()


def _restated_update(ema_sd, model_sd, decay):
    for k, e in ema_sd.items():
        e.copy_(e * decay + (1. - decay) * model_sd[k].detach())


def _perturb(model, g, frozen_too=False):
    """A training step's worth of change to every trainable tensor; the frozen position tables stay as they are unless
    `frozen_too`."""
    with torch.no_grad():
        for p in model.parameters():
            if p.requires_grad or frozen_too:
                p.add_(torch.randn(p.shape, generator=g).to(p.device) * 0.01)


def _base():
    from test_model_ema_host import _cls_model
    return _cls_model(base=True)


def _odd():
    """37-class head (rows of 37 and a 37-element bias), a semantic-segmentation input with its class embedding, a
    learnable position table next to a frozen one."""
    from functools import partial
    from multimae_b200.input_adapters import PatchedInputAdapter, SemSegInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import LinearOutputAdapter
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=64,
                                      sincos_pos_emb=False, learnable_pos_emb=True),
           "semseg": SemSegInputAdapter(num_classes=13, stride_level=4, patch_size_full=16, image_size=64,
                                        dim_class_emb=64)}
    return MultiViT(ins, {"cls": LinearOutputAdapter(num_classes=37)}, num_global_tokens=1, dim_tokens=128, depth=2,
                    num_heads=2, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


@pytest.mark.parametrize("decay", [0.9999, 0.5])
@pytest.mark.parametrize("which", ["multivit_base", "odd"])
def test_bitwise_equal_to_the_reference_update(dev, which, decay):
    from multimae_b200.model_ema import ModelEma
    torch.manual_seed(0)
    model = (_base() if which == "multivit_base" else _odd()).to(dev)
    sd = model.state_dict()
    if which == "odd":
        assert sd["output_adapters.cls.head.bias"].numel() == 37 and "input_adapters.semseg.class_emb.weight" in sd
        assert model.input_adapters["rgb"].pos_emb.requires_grad and not model.input_adapters["semseg"].pos_emb.requires_grad
    ema = ModelEma(model, decay=decay)
    restated = {k: v.clone() for k, v in ema.ema.state_dict().items()}
    lib = _lib()
    g = torch.Generator().manual_seed(1)
    for _ in range(5):
        _perturb(model, g)
        before = lib.mmae_launch_count()
        ema.update(model)
        assert lib.mmae_launch_count() - before == 1                  # every pair in one launch
        _restated_update(restated, model.state_dict(), decay)
    torch.cuda.synchronize()
    got = ema.ema.state_dict()
    assert list(got) == list(restated)
    for k, v in restated.items():
        assert torch.equal(got[k], v), (k, float((got[k] - v).abs().max()))
    # the averaged values did move away from the live ones (the comparison is not between unchanged tensors)
    assert not torch.equal(got["encoder.0.attn.qkv.weight"], sd["encoder.0.attn.qkv.weight"])


def test_direct_call_with_unaligned_views_and_several_launches(dev):
    """600 segments (0 to ~5000 elements, a few hundred thousand in one) at every 4-byte offset mod 16, packed back to back
    in two buffers: three launches of up to 256 non-empty segments; the gaps between segments stay untouched."""
    g = torch.Generator().manual_seed(5)
    sizes = torch.randint(0, 5000, (600,), generator=g).tolist()
    sizes[7], sizes[300], sizes[301] = 0, 300_001, 3
    gaps = torch.randint(0, 4, (600, 2), generator=g).tolist()
    d_off, s_off, d_at, s_at = [], [], 0, 0
    for n, (gd, gs) in zip(sizes, gaps):
        d_at, s_at = d_at + gd, s_at + gs
        d_off.append(d_at)
        s_off.append(s_at)
        d_at, s_at = d_at + n, s_at + n
    dst = torch.randn(d_at + 4, generator=g).to(dev)
    src = torch.randn(s_at + 4, generator=g).to(dev)
    assert {o % 4 for o in d_off} == {0, 1, 2, 3} and {o % 4 for o in s_off} == {0, 1, 2, 3}
    decay = 0.9999
    want = dst.clone()
    for n, do, so in zip(sizes, d_off, s_off):
        e = want[do:do + n]
        e.copy_(e * decay + (1. - decay) * src[so:so + n])
    P, N = ctypes.c_void_p * 600, ctypes.c_int64 * 600
    lib = _lib()
    before = lib.mmae_launch_count()
    from multimae_b200 import _lib as L
    L.check(lib.mmae_ema_update(P(*[dst.data_ptr() + 4 * o for o in d_off]), P(*[src.data_ptr() + 4 * o for o in s_off]),
                                N(*sizes), 600, decay, 1.0 - decay, L.current_stream()), "mmae_ema_update")
    nonempty = sum(1 for n in sizes if n)
    assert lib.mmae_launch_count() - before == math.ceil(nonempty / 256) == 3
    torch.cuda.synchronize()
    assert torch.equal(dst, want), float((dst - want).abs().max())


def test_train_one_epoch_leaves_the_live_model_alone(dev):
    """run_finetuning_cls.py:497-537 restated over the overlay classes with --model_ema: the EMA is built after .to(device)
    and before the DistributedDataParallel stand-in, and updated through it after every optimizer step.  The update
    changes neither a parameter nor a gradient of the live model, and the EMA equals the restated update."""
    from multimae_b200 import multimae as mm
    from multimae_b200 import overlay
    from multimae_b200.model_ema import ModelEma
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True
    try:
        torch.manual_seed(0)
        C, B, update_freq, decay = 37, 8, 2, 0.99
        model = _small(num_classes=C, drop_path_rate=0.1).to(dev)
        model_ema = ModelEma(model, decay=decay, device="", resume="")
        restated = {k: v.clone() for k, v in model_ema.ema.state_dict().items()}
        model = overlay._IdentityDDP(model, device_ids=[0])
        model_without_ddp = model.module
        optimizer = torch.optim.AdamW(_param_groups(model_without_ddp, 0.05, 0.65), lr=1e-3)
        loss_scaler = NativeScalerWithGradNormCount()
        g = torch.Generator().manual_seed(3)
        data = [({"rgb": torch.randn(B, 3, 64, 64, generator=g), "depth": torch.randn(B, 1, 64, 64, generator=g)},
                 torch.randint(0, C, (B,), generator=g)) for _ in range(update_freq)]
        lib = _lib()
        model.train(True)
        optimizer.zero_grad()
        updates = 0
        for data_iter_step in range(4 * update_freq):
            samples, targets = data[data_iter_step % update_freq]
            samples = {k: v.to(dev, non_blocking=True) for k, v in samples.items()}
            targets = targets.to(dev, non_blocking=True)
            mixed = {}
            for k, v in samples.items():
                mixed[k], soft = _mixup(v, targets, C, lam=0.7)
            with torch.cuda.amp.autocast():
                loss = soft_target_ce(model(mixed)["cls"], soft)
            assert math.isfinite(loss.item())
            loss /= update_freq
            loss_scaler(loss, optimizer, clip_grad=1.0, parameters=model.parameters(), create_graph=False,
                        update_grad=(data_iter_step + 1) % update_freq == 0)
            if (data_iter_step + 1) % update_freq == 0:
                optimizer.zero_grad()
                live = model_without_ddp.state_dict()
                params = {k: v.clone() for k, v in live.items()}
                grads = model_without_ddp.grad_arena().flat.clone()
                before = lib.mmae_launch_count()
                model_ema.update(model)
                assert lib.mmae_launch_count() - before == 1
                torch.cuda.synchronize()
                assert all(torch.equal(live[k], v) for k, v in params.items())
                assert torch.equal(model_without_ddp.grad_arena().flat, grads)
                _restated_update(restated, live, decay)
                got = model_ema.ema.state_dict()
                assert all(torch.equal(got[k], v) for k, v in restated.items())
                updates += 1
            torch.cuda.synchronize()
        assert updates == 4
        assert model_ema.ema._arena is not model_without_ddp._arena
    finally:
        mm.AUTO_OWN_GRADIENTS = old


@pytest.fixture()
def utils_standin(monkeypatch):
    """The reference's `utils` package (stand-in) with the three names overlay.install() rebinds rebound; sys.modules
    and sys.path are restored afterwards."""
    from multimae_b200.model_ema import ModelEma
    saved = {k: v for k, v in sys.modules.items() if k == "utils" or k.startswith("utils.")}
    for k in saved:
        del sys.modules[k]
    monkeypatch.syspath_prepend(STANDIN)
    import utils
    import utils.model
    import utils.model_ema
    utils.ModelEma = utils.model_ema.ModelEma = utils.model.ModelEma = ModelEma
    yield utils
    for k in [k for k in sys.modules if k == "utils" or k.startswith("utils.")]:
        del sys.modules[k]
    sys.modules.update(saved)


def test_checkpoint_round_trip_and_eval_forward(dev, tmp_path, utils_standin):
    """utils.save_model stores get_state_dict(model_ema); a fresh ModelEma loads it through _load_checkpoint with a
    'state_dict_ema' key bitwise.  The EMA copy's no-grad eval forward, run once before the updates (so that cached
    position tables exist) and once after, equals that of a fresh multivit_base loaded with the EMA's state_dict."""
    import argparse
    from multimae_b200.model_ema import ModelEma
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    utils = utils_standin
    torch.manual_seed(0)
    model = _base().to(dev)
    ema = utils.ModelEma(model, decay=0.5)
    x = torch.randn(4, 3, 224, 224, device=dev)
    with torch.no_grad(), torch.cuda.amp.autocast():
        ema.ema(x)
    g = torch.Generator().manual_seed(2)
    pos = ema.ema.input_adapters["rgb"].pos_emb.clone()
    for _ in range(3):
        _perturb(model, g, frozen_too=True)
        ema.update(model)
    assert not torch.equal(ema.ema.input_adapters["rgb"].pos_emb, pos)     # a table the first forward may have cached
    assert utils.unwrap_model(ema) is ema.ema
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4)
    args = argparse.Namespace(output_dir=str(tmp_path))
    utils.save_model(args=args, epoch=0, model=model, model_without_ddp=model, optimizer=opt,
                     loss_scaler=NativeScalerWithGradNormCount(), model_ema=ema)
    ck = torch.load(str(tmp_path / "checkpoint-0.pth"), map_location="cpu", weights_only=False)
    esd = ema.ema.state_dict()
    assert list(ck["model_ema"]) == list(esd)
    assert all(torch.equal(ck["model_ema"][k], v.cpu()) for k, v in esd.items())
    torch.manual_seed(7)
    fresh = ModelEma(_base().to(dev))
    utils.checkpoint._load_checkpoint_for_ema(fresh, {"state_dict_ema": ck["model_ema"]})
    assert all(torch.equal(fresh.ema.state_dict()[k], v) for k, v in esd.items())
    torch.manual_seed(8)
    plain = _base().to(dev)
    plain.load_state_dict(esd)
    plain.eval()
    with torch.no_grad(), torch.cuda.amp.autocast():
        want = plain(x)["cls"]
        got = ema.ema(x)["cls"]
        got_fresh = fresh.ema(x)["cls"]
    torch.cuda.synchronize()
    assert torch.isfinite(want).all() and torch.equal(got, want) and torch.equal(got_fresh, want)


def test_cpu_device_matches_the_restatement(dev):
    """--model_ema_force_cpu: model on the GPU, EMA on the host, the reference's loop there."""
    from multimae_b200.model_ema import ModelEma
    torch.manual_seed(0)
    model = _odd().to(dev)
    ema = ModelEma(model, decay=0.9999, device="cpu")
    restated = {k: v.clone() for k, v in ema.ema.state_dict().items()}
    assert all(v.device.type == "cpu" for v in restated.values())
    lib = _lib()
    before = lib.mmae_launch_count()
    g = torch.Generator().manual_seed(4)
    for _ in range(3):
        _perturb(model, g)
        ema.update(model)
        _restated_update(restated, {k: v.cpu() for k, v in model.state_dict().items()}, 0.9999)
    assert lib.mmae_launch_count() == before
    got = ema.ema.state_dict()
    assert all(torch.equal(got[k], v) for k, v in restated.items())
