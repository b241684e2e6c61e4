"""GPU: the classification head of fine-tuning (LinearOutputAdapter -> mmae_clshead_*) and the body of the reference's
run_finetuning_cls.py train_one_epoch over the overlay classes.  Nothing here reads the reference checkout."""
import math

import pytest
import torch

from cls_head_oracle import cls_head, encoder_tokens, soft_target_ce, vit_config
from helpers import load_fixture, rel_l2
from test_cuda_parity import BF16_TOL, _check_grads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _small(num_classes=10, mean_pool=True, drop_path_rate=0.0, size=64):
    from test_cls_head_host import _build
    return _build(num_classes=num_classes, mean_pool=mean_pool, drop_path_rate=drop_path_rate, size=size)


@pytest.mark.parametrize("mode", ["mean", "last"])
def test_fixture_model_on_cuda(golden_dir, dev, mode):
    """The reference's MultiViT + LinearOutputAdapter(10) recorded by make_golden_cls.py: logits and every gradient."""
    fx = load_fixture(golden_dir, "cls_head.pt")
    model = _small(mean_pool=(mode == "mean"))
    model.load_state_dict(fx["state_dict"])
    model = model.to(dev).train()
    logits = model({k: v.to(dev) for k, v in fx["inputs"].items()})["cls"]
    assert logits.dtype == torch.float32 and logits.shape == (3, 10)
    assert rel_l2(logits, fx["logits"][mode]) < BF16_TOL, rel_l2(logits, fx["logits"][mode])
    loss = soft_target_ce(logits, fx["target"].to(dev))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss.detach()) - float(fx["loss"][mode])) < BF16_TOL * abs(float(fx["loss"][mode]))
    got = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
    ref = fx["grads_" + mode]
    assert set(got) == set(ref)
    _check_grads(got, ref)
    for k in ref:
        if k.startswith("output_adapters.cls."):
            assert rel_l2(got[k], ref[k]) < BF16_TOL, (k, rel_l2(got[k], ref[k]))


_ENC = {}
MODEL_TOL = 2e-2


def _oracle_base_tokens(B):
    """multivit_base encoder tokens at 224 x 224 rgb (N = 197) from the oracle, and the state they were computed with."""
    if B not in _ENC:
        from multimae_b200.input_adapters import PatchedInputAdapter
        from multimae_b200.multimae import multivit_base
        torch.manual_seed(0)
        enc_model = multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16,
                                                              image_size=224)}, None)
        sd = {k: v.clone() for k, v in enc_model.state_dict().items()}
        g = torch.Generator().manual_seed(9)
        with torch.no_grad():
            for k, v in sd.items():
                if k.endswith(".bias") or k == "global_tokens":
                    v.add_(torch.randn(v.shape, generator=g) * 0.05)
        cfg = vit_config(("rgb",), 768, 12, 12, 224)
        x = {"rgb": torch.randn(B, 3, 224, 224, generator=g)}
        with torch.no_grad():
            enc = encoder_tokens(sd, x, cfg)
        _ENC[B] = (sd, x, enc)
    return _ENC[B]


@pytest.mark.parametrize("num_classes", [1000, 101, 1, 0])
@pytest.mark.parametrize("mean_pool", [True, False])
def test_multivit_base_224_against_oracle(dev, num_classes, mean_pool):
    """multivit_base + LinearOutputAdapter at 224 x 224 (N = 197), B = 3 and 5: logits of the whole model against the oracle
    encoder + fp32 head; and the head alone on the oracle's own encoder tokens - output, token gradient and the four
    parameter gradients against torch autograd in fp32 (class counts whose rows are not 16-byte aligned included).

    The whole-model figure carries the bf16 encoder's own error (1e-2 on its tokens, test_cuda_parity), which with one
    logit per sample is not averaged over many outputs: it gets MODEL_TOL.  The head itself is held to BF16_TOL."""
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    from multimae_b200.output_adapters import LinearOutputAdapter
    model = multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=224)},
                          {"cls": LinearOutputAdapter(num_classes, use_mean_pooling=mean_pool)})
    head = model.output_adapters["cls"]
    with torch.no_grad():
        head.norm.weight.add_(0.1 * torch.randn(768))
        head.norm.bias.add_(0.05 * torch.randn(768))
        if num_classes:
            head.head.bias.add_(0.05 * torch.randn(num_classes))
    hsd = {"output_adapters.cls." + k: v.clone() for k, v in head.state_dict().items()}
    for B in (3, 5):
        sd, x, enc = _oracle_base_tokens(B)
        model.load_state_dict({**sd, **hsd})
        model = model.to(dev).train()
        ref = cls_head(enc, hsd, mean_pool=mean_pool)
        out = model({"rgb": x["rgb"].to(dev)})["cls"]
        assert out.shape == ref.shape == (B, num_classes or 768)
        assert rel_l2(out, ref) < MODEL_TOL, (B, rel_l2(out, ref))
        # the head alone on identical input: forward and backward against fp32 autograd
        p = {k: v.clone().requires_grad_(True) for k, v in hsd.items()}
        e = enc.clone().requires_grad_(True)
        r = cls_head(e, p, mean_pool=mean_pool)
        dout = torch.randn(r.shape, generator=torch.Generator().manual_seed(B))
        r.backward(dout)
        ed = enc.to(dev).requires_grad_(True)
        head.zero_grad(set_to_none=True)
        got = head(ed)
        got.backward(dout.to(dev))
        torch.cuda.synchronize()
        assert rel_l2(got, r) < BF16_TOL, (B, rel_l2(got, r))
        assert rel_l2(ed.grad, e.grad) < BF16_TOL, (B, rel_l2(ed.grad, e.grad))
        if mean_pool:          # every token receives dpooled / N
            assert torch.equal(ed.grad[:, 0], ed.grad[:, 1]) and torch.equal(ed.grad[:, 0], ed.grad[:, -1])
        else:                  # only the global token
            assert not ed.grad[:, :-1].any()
        for k, v in p.items():
            g = dict(head.named_parameters())[k[len("output_adapters.cls."):]].grad
            assert rel_l2(g, v.grad) < BF16_TOL, (B, k, rel_l2(g, v.grad))
        model.cpu()


def test_eval_forward_matches_training_forward(dev):
    """The script's evaluate(): torch.no_grad() + model.eval() at B = 192 and a ragged last batch issue the same kernels
    as the training forward (drop_path 0), so the logits are bitwise equal."""
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    from multimae_b200.output_adapters import LinearOutputAdapter
    torch.manual_seed(1)
    model = multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=224)},
                          {"cls": LinearOutputAdapter(1000)}).to(dev)
    for B in (192, 77):
        x = torch.randn(B, 3, 224, 224, device=dev)
        with torch.cuda.amp.autocast():
            train = model.train()(x)["cls"]
        with torch.no_grad(), torch.cuda.amp.autocast():
            ev = model.eval()(x)["cls"]
        torch.cuda.synchronize()
        assert ev.shape == (B, 1000) and ev.grad_fn is None and train.grad_fn is not None
        assert torch.isfinite(ev).all() and torch.equal(ev, train.detach()), B


def _param_groups(model, weight_decay, layer_decay):
    """utils/optim_factory.py get_parameter_groups with LayerDecayValueAssigner (run_finetuning_cls.py:369-389)."""
    num_layers = model.get_num_layers()
    values = [layer_decay ** (num_layers + 1 - i) for i in range(num_layers + 2)]
    skip = model.no_weight_decay()

    def layer_id(name):
        if name in ("cls_token", "mask_token", "pos_embed", "global_tokens") or name.startswith("input_adapters"):
            return 0
        if name.startswith("encoder"):
            return int(name.split(".")[1]) + 1
        return len(values) - 1
    groups = {}
    for name, p in model.named_parameters():
        if not p.requires_grad:
            continue
        no_decay = len(p.shape) == 1 or name.endswith(".bias") or name in skip
        lid = layer_id(name)
        key = "layer_%d_%s" % (lid, "no_decay" if no_decay else "decay")
        g = groups.setdefault(key, {"weight_decay": 0.0 if no_decay else weight_decay, "params": [],
                                    "lr_scale": values[lid]})
        g["params"].append(p)
    return list(groups.values())


def _mixup(samples, targets, num_classes, lam, smoothing=0.1):
    """Mixup with label smoothing (timm's Mixup, mode 'batch'): a fixed lam, the batch mixed with its flip."""
    off, on = smoothing / num_classes, 1.0 - smoothing + smoothing / num_classes
    y = torch.full((targets.shape[0], num_classes), off, device=targets.device).scatter_(1, targets[:, None], on)
    return samples * lam + samples.flip(0) * (1 - lam), y * lam + y.flip(0) * (1 - lam)


def test_finetune_cls_train_one_epoch_sequence(dev):
    """run_finetuning_cls.py:497-560 restated line by line over the overlay classes with the REAL library: autocast, mixup
    soft targets with SoftTargetCrossEntropy, layer-decay parameter groups on the stock torch.optim.AdamW, loss scaling on,
    update_freq = 2, clip_grad, the DistributedDataParallel stand-in; the loss falls over 10 steps on a fixed batch."""
    from multimae_b200 import multimae as mm
    from multimae_b200 import overlay
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True                                   # what overlay.install() sets
    try:
        torch.manual_seed(0)
        C, B, update_freq, max_norm = 37, 8, 2, 1.0
        model = _small(num_classes=C, drop_path_rate=0.1).to(dev)
        model = overlay._IdentityDDP(model, device_ids=[0])
        model_without_ddp = model.module
        optimizer = torch.optim.AdamW(_param_groups(model_without_ddp, 0.05, 0.65), lr=1e-3)
        loss_scaler = NativeScalerWithGradNormCount()
        g = torch.Generator().manual_seed(3)
        data = [({"rgb": torch.randn(B, 3, 64, 64, generator=g), "depth": torch.randn(B, 1, 64, 64, generator=g)},
                 torch.randint(0, C, (B,), generator=g)) for _ in range(update_freq)]
        model.train(True)
        optimizer.zero_grad()
        losses, norms = [], []
        for data_iter_step in range(10 * update_freq):
            for i, param_group in enumerate(optimizer.param_groups):
                param_group["lr"] = 1e-3 * param_group["lr_scale"]
            samples, targets = data[data_iter_step % update_freq]
            samples = {k: v.to(dev, non_blocking=True) for k, v in samples.items()}
            targets = targets.to(dev, non_blocking=True)
            mixed = {}
            for k, v in samples.items():
                mixed[k], soft = _mixup(v, targets, C, lam=0.7)
            with torch.cuda.amp.autocast():
                outputs = model(mixed)["cls"]
                loss = soft_target_ce(outputs, soft)
            loss_value = loss.item()
            assert math.isfinite(loss_value)
            loss /= update_freq
            grad_norm = loss_scaler(loss, optimizer, clip_grad=max_norm, parameters=model.parameters(), create_graph=False,
                                    update_grad=(data_iter_step + 1) % update_freq == 0)
            if (data_iter_step + 1) % update_freq == 0:
                arena = model_without_ddp.grad_arena()
                after = float(arena.flat.norm())
                assert arena.owned and not arena.accumulating
                # the returned norm is the pre-clip one; the gradients the optimizer stepped with are clipped to max_norm
                assert after <= max_norm * (1 + 1e-4), after
                if float(grad_norm) > max_norm:
                    assert abs(after - max_norm * float(grad_norm) / (float(grad_norm) + 1e-6)) < 1e-4 * max_norm
                optimizer.zero_grad()
                norms.append(float(grad_norm))
            else:
                assert grad_norm is None
            assert loss_scaler.state_dict()["scale"] == 65536.0
            torch.cuda.synchronize()
            losses.append(loss_value)
        assert any(n > max_norm for n in norms), norms
        first = sum(losses[:update_freq]) / update_freq
        last = sum(losses[-update_freq:]) / update_freq
        assert last < 0.9 * first, losses
        print("fine-tuning sequence: losses %s, pre-clip grad norms %s" % ([round(v, 4) for v in losses[::update_freq]],
                                                                           [round(v, 3) for v in norms]))
    finally:
        mm.AUTO_OWN_GRADIENTS = old


def test_gradient_accumulation_matches_concatenated_batch(dev):
    """update_freq = 2 through NativeScalerWithGradNormCount(update_grad=False): the accumulated gradient of two half
    batches (each loss / 2) equals the gradient of the concatenated batch (drop_path 0: no draws that could differ)."""
    from multimae_b200 import multimae as mm
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    torch.manual_seed(0)
    C = 101
    model = _small(num_classes=C).to(dev).train()
    g = torch.Generator().manual_seed(4)
    x = {"rgb": torch.randn(8, 3, 64, 64, generator=g).to(dev), "depth": torch.randn(8, 1, 64, 64, generator=g).to(dev)}
    soft = torch.softmax(torch.randn(8, C, generator=g), -1).to(dev)
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True
    try:
        class _NoStep:
            param_groups = []

            def step(self):
                pass
        scaler = NativeScalerWithGradNormCount()
        for half in (slice(0, 4), slice(4, 8)):
            loss = soft_target_ce(model({k: v[half] for k, v in x.items()})["cls"], soft[half]) / 2
            scaler(loss, _NoStep(), parameters=model.parameters(), update_grad=half.start == 4)
        torch.cuda.synchronize()
        acc = model.grad_arena().flat.clone()
        loss = soft_target_ce(model(x)["cls"], soft)
        scaler(loss, _NoStep(), parameters=model.parameters())
        torch.cuda.synchronize()
        full = model.grad_arena().flat.clone()
    finally:
        mm.AUTO_OWN_GRADIENTS = old
    assert float(full.norm()) > 0 and rel_l2(acc, full) < 1e-3, rel_l2(acc, full)
