"""GPU: the grouped flat AdamW (multimae_b200.optim.GroupedFlatAdamW -> mmae_adamw_step_groups) against torch.optim.AdamW
and a float64 restatement of its update, over multivit_base + a 1000-class head with the layer-decay groups of the
fine-tuning scripts (tests/adamw_standin).

Error measure: |x - x64| in fp32 ulps of the magnitude of the terms that form x (b1|m| + (1-b1)|g| for exp_avg,
b2 v + (1-b2) g^2 for exp_avg_sq, |p (1 - lr wd)| + (lr/bc1) scale(m) / denom for the parameter), with x64 the float64
update applied to the SAME fp32 state the optimizer started the step from.  Under cancellation this is the quantity a
correctly ordered fp32 evaluation keeps small; an error in ulps of the result itself is unbounded there, for torch too."""
import gc
import io
import math

import pytest
import torch

from test_flat_adamw_host import _cls_base, _factory, _groups

pytestmark = pytest.mark.gpu

# the new class's budget: every parameter / moment element within this many fp32 ulps of its float64 restatement.  The
# test also holds torch.optim.AdamW's own fp32 result to it and requires torch to need at least a quarter of it.
ULP_BUDGET = 5.0
BETAS, EPS = (0.9, 0.999), 1e-8


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _release():
    yield
    for obj in gc.get_objects():           # free the bf16 twins' registry slots of this test's optimizers
        if type(obj).__name__ == "GroupedFlatAdamW":
            obj.release_mirror()
    gc.collect()


def _ulp(scale):
    scale = scale.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(scale)) - 23)


def _reference(p, g, m, v, step, lr, wd, b1, b2, eps):
    """Float64 AdamW step (torch's decoupled order) from fp32 state; returns the new values and their error scales."""
    p, g, m, v = (t.double() for t in (p, g, m, v))
    pd = p * (1 - lr * wd)
    m1 = m + (1 - b1) * (g - m)
    v1 = v * b2 + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    denom = v1.sqrt() / math.sqrt(bc2) + eps
    p1 = pd - (lr / bc1) * m1 / denom
    sm = b1 * m.abs() + (1 - b1) * g.abs()
    sv = v1
    sp = pd.abs() + (lr / bc1) * sm / denom
    return (p1, m1, v1), (sp, sm, sv)


class _Err:
    def __init__(self):
        self.worst = [0.0, 0.0, 0.0]

    def add(self, got, ref, scale):
        for k, (x, r, s) in enumerate(zip(got, ref, scale)):
            e = float(((x.double() - r).abs() / _ulp(s)).max())
            self.worst[k] = max(self.worst[k], e)

    def max(self):
        return max(self.worst)


def _state_of(opt, p):
    st = opt.state.get(p, {})
    if "exp_avg" not in st:
        return torch.zeros_like(p), torch.zeros_like(p), 0.0
    return st["exp_avg"].clone(), st["exp_avg_sq"].clone(), float(st["step"])


def _pair(dev, seed=0):
    """(model, GroupedFlatAdamW) and (model, torch.optim.AdamW) from one initial state, with the script's groups."""
    from multimae_b200 import optim as O
    a = _cls_base(seed).to(dev)
    b = _cls_base(seed + 100).to(dev)
    b.load_state_dict(a.state_dict())
    ours = O.GroupedFlatAdamW(_groups(a), lr=1e-3, betas=BETAS, eps=EPS, weight_decay=0.0)
    stock = torch.optim.AdamW(_groups(b), lr=1e-3, betas=BETAS, eps=EPS, weight_decay=0.0)
    return (a, ours), (b, stock)


def _set_grads(models, it, dev):
    gen = torch.Generator(device=dev).manual_seed(1000 + it)
    for named in zip(*[[p for p in m.parameters() if p.requires_grad] for m in models]):
        g = torch.randn(named[0].shape, generator=gen, device=dev) * 1e-2
        g[..., ::7] *= 1e-4                        # a spread of magnitudes: some entries near eps after the sqrt
        for p in named:
            if p.grad is None:
                p.grad = g.clone()
            else:
                p.grad.copy_(g)


def _step_and_check(opt, model, err, dev):
    """One opt.step(), checked element-wise against the float64 restatement from the state it started from."""
    before = {}
    for g in opt.param_groups:
        for p in g["params"]:
            if p.requires_grad:
                m, v, step = _state_of(opt, p)
                before[p] = (p.detach().clone(), p.grad.clone(), m, v, step, g["lr"], g["weight_decay"])
    opt.step()
    torch.cuda.synchronize()
    for p, (p0, g0, m0, v0, step, lr, wd) in before.items():
        ref, scale = _reference(p0, g0, m0, v0, step + 1, lr, wd, *BETAS, EPS)
        st = opt.state[p]
        err.add((p.detach(), st["exp_avg"], st["exp_avg_sq"]), ref, scale)


def test_parity_with_torch_and_float64(dev):
    (a, ours), (b, stock) = _pair(dev)
    e_ours, e_torch = _Err(), _Err()
    same = total = 0
    decays = [g["weight_decay"] > 0 for g in ours.param_groups]
    assert decays == [g["weight_decay"] > 0 for g in stock.param_groups] and any(decays) and not all(decays)
    for it in range(10):
        for opt in (ours, stock):
            for g, decay in zip(opt.param_groups, decays):
                g["lr"] = 1e-3 * (0.8 ** it) * g["lr_scale"]
                if decay:
                    g["weight_decay"] = 0.05 - 0.003 * it
        _set_grads([a, b], it, dev)
        _step_and_check(ours, a, e_ours, dev)
        _step_and_check(stock, b, e_torch, dev)
        assert float(ours._step[0]) == it + 1
        # the bf16 twin is bf16(params), bit for bit, after every step
        assert torch.equal(ours.flat_bf16, ours.flat_params.to(torch.bfloat16))
        pa = [p for p in a.parameters() if p.requires_grad]
        pb = [p for p in b.parameters() if p.requires_grad]
        same += sum(int((x == y).sum()) for x, y in zip(pa, pb))
        total += sum(x.numel() for x in pa)
    print("grouped flat AdamW: max error over 10 steps (ulps of the terms' magnitude; param, exp_avg, exp_avg_sq): "
          "ours %s, torch %s; parameters bitwise equal to torch: %.4f%%"
          % ([round(x, 3) for x in e_ours.worst], [round(x, 3) for x in e_torch.worst], 100.0 * same / total))
    assert e_ours.max() <= ULP_BUDGET, e_ours.worst
    assert e_torch.max() <= ULP_BUDGET, e_torch.worst
    assert e_torch.max() >= ULP_BUDGET / 4, e_torch.worst


def test_skipped_step_changes_nothing_and_the_next_step_is_exact(dev):
    (a, ours), (b, twin) = _pair(dev)[0], _pair(dev, seed=0)[0]
    found = torch.zeros(1, device=dev)
    _set_grads([a, b], 0, dev)
    ours.fused_step(found_inf=found)
    twin.fused_step(found_inf=found)
    snap = [t.clone() for t in (ours.flat_params, ours.exp_avg, ours.exp_avg_sq, ours.flat_bf16, ours._step)]
    # a step with non-finite gradients: the scaler's found_inf is set; the arena may hold anything
    for p in a.parameters():
        if p.requires_grad:
            p.grad.fill_(float("nan"))
    ours.fused_step(found_inf=torch.ones(1, device=dev))
    torch.cuda.synchronize()
    after = (ours.flat_params, ours.exp_avg, ours.exp_avg_sq, ours.flat_bf16, ours._step)
    assert all(torch.equal(x, y) for x, y in zip(snap, after))
    assert float(ours._step[0]) == 1.0
    _set_grads([a, b], 1, dev)
    ours.fused_step(found_inf=found)
    twin.fused_step(found_inf=found)
    torch.cuda.synchronize()
    for x, y in zip((ours.flat_params, ours.exp_avg, ours.exp_avg_sq, ours.flat_bf16, ours._step),
                    (twin.flat_params, twin.exp_avg, twin.exp_avg_sq, twin.flat_bf16, twin._step)):
        assert torch.equal(x, y)
    assert float(ours._step[0]) == 2.0


def test_steps_without_host_sync(dev):
    (a, ours), _ = _pair(dev)
    _set_grads([a], 0, dev)
    found = torch.zeros(1, device=dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for it in range(3):
            for g in ours.param_groups:
                g["lr"] = 1e-3 * g["lr_scale"] / (it + 1)
            ours.step()
            ours.fused_step(found_inf=found)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert float(ours._step[0]) == 6.0


@pytest.mark.parametrize("direction", ["ours_to_torch", "torch_to_ours"])
def test_checkpoint_resume_across_optimizers(dev, direction):
    from multimae_b200 import optim as O
    (a, ours), (b, stock) = _pair(dev)
    src_model, src = (a, ours) if direction == "ours_to_torch" else (b, stock)
    for it in range(3):
        _set_grads([src_model], it, dev)
        src.step()
    # through a file, as utils.save_model / auto_load_model do (torch.save; torch.load with map_location="cpu")
    buf = io.BytesIO()
    torch.save(src.state_dict(), buf)
    buf.seek(0)
    sd = torch.load(buf, map_location="cpu", weights_only=False)
    # resume: a fresh model with the trained weights, a fresh optimizer of the other kind
    dst_model = _cls_base(7).to(dev)
    dst_model.load_state_dict(src_model.state_dict())
    if direction == "ours_to_torch":
        dst = torch.optim.AdamW(_groups(dst_model), lr=1e-3, betas=BETAS, eps=EPS, weight_decay=0.0)
    else:
        dst = O.GroupedFlatAdamW(_groups(dst_model), lr=1e-3, betas=BETAS, eps=EPS, weight_decay=0.0)
    dst.load_state_dict(sd)
    for opt in (src, dst):
        for g in opt.param_groups:
            g["lr"] = 5e-4 * g["lr_scale"]
    _set_grads([src_model, dst_model], 3, dev)
    e_src, e_dst = _Err(), _Err()
    _step_and_check(src, src_model, e_src, dev)
    _step_and_check(dst, dst_model, e_dst, dev)
    print("resume %s: error of the next step (ulps) source %s, resumed %s" % (direction, e_src.worst, e_dst.worst))
    assert e_src.max() <= ULP_BUDGET and e_dst.max() <= ULP_BUDGET
    for p, q in zip([p for p in src_model.parameters() if p.requires_grad],
                    [p for p in dst_model.parameters() if p.requires_grad]):
        assert float(((p - q).abs() / _ulp(p.detach().abs().double() + 1e-3)).max()) <= 2 * ULP_BUDGET
    assert all(float(s["step"]) == 4.0 for s in dst.state_dict()["state"].values())


def _mixup(samples, targets, num_classes, lam, smoothing=0.1):
    off, on = smoothing / num_classes, 1.0 - smoothing + smoothing / num_classes
    y = torch.full((targets.shape[0], num_classes), off, device=targets.device).scatter_(1, targets[:, None], on)
    return samples * lam + samples.flip(0) * (1 - lam), y * lam + y.flip(0) * (1 - lam)


def _train(dev, flat, steps=3, update_freq=2):
    """run_finetuning_cls.py train_one_epoch (lines 497-560) restated: autocast, mixup soft targets, loss scaling,
    clip_grad, update_freq, the optimizer built by create_optimizer with the script's layer-decay assigner."""
    import argparse
    from cls_head_oracle import soft_target_ce
    from multimae_b200 import overlay
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from test_cls_head_host import _build
    f = _factory()
    f.optim = overlay._FactoryOptim(torch.optim) if flat else torch.optim
    torch.manual_seed(0)
    C, B = 37, 8
    model = overlay._IdentityDDP(_build(num_classes=C).to(dev), device_ids=[0])
    model_without_ddp = model.module
    start = {n: p.detach().clone() for n, p in model_without_ddp.named_parameters()}
    lda = f.layer_decay_assigner(model_without_ddp, 0.65)
    args = argparse.Namespace(opt="adamw", lr=1e-3, weight_decay=0.05, opt_eps=1e-8, opt_betas=None, momentum=0.9)
    optimizer = f.create_optimizer(args, model_without_ddp, skip_list=model_without_ddp.no_weight_decay(),
                                   get_num_layer=lda.get_layer_id, get_layer_scale=lda.get_scale)
    loss_scaler = NativeScalerWithGradNormCount()
    g = torch.Generator().manual_seed(3)
    data = [({"rgb": torch.randn(B, 3, 64, 64, generator=g), "depth": torch.randn(B, 1, 64, 64, generator=g)},
             torch.randint(0, C, (B,), generator=g)) for _ in range(update_freq * steps)]
    model.train(True)
    optimizer.zero_grad()
    losses = []
    for data_iter_step in range(steps * update_freq):
        it = data_iter_step // update_freq
        for param_group in optimizer.param_groups:
            param_group["lr"] = 1e-3 * (0.9 ** it) * param_group["lr_scale"]
            if param_group["weight_decay"] > 0:
                param_group["weight_decay"] = 0.05 - 0.01 * it
        samples, targets = data[data_iter_step]
        samples = {k: v.to(dev, non_blocking=True) for k, v in samples.items()}
        targets = targets.to(dev, non_blocking=True)
        mixed = {}
        for k, v in samples.items():
            mixed[k], soft = _mixup(v, targets, C, lam=0.7)
        with torch.cuda.amp.autocast():
            outputs = model(mixed)["cls"]
            loss = soft_target_ce(outputs, soft)
        losses.append(loss.item())
        loss /= update_freq
        loss_scaler(loss, optimizer, clip_grad=1.0, parameters=model.parameters(), create_graph=False,
                    update_grad=(data_iter_step + 1) % update_freq == 0)
        if (data_iter_step + 1) % update_freq == 0:
            optimizer.zero_grad()
    torch.cuda.synchronize()
    end = {n: p.detach().clone() for n, p in model_without_ddp.named_parameters()}
    return optimizer, losses, start, end


def test_finetune_cls_loop_through_the_factory(dev):
    from multimae_b200 import multimae as mm
    from multimae_b200.optim import GroupedFlatAdamW
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True                                   # what overlay.install() sets
    try:
        stock, l_stock, s0, e_stock = _train(dev, flat=False)
        ours, l_ours, s1, e_ours = _train(dev, flat=True)
    finally:
        mm.AUTO_OWN_GRADIENTS = old
    assert type(stock) is torch.optim.AdamW and type(ours) is GroupedFlatAdamW
    assert all(math.isfinite(v) for v in l_stock + l_ours)
    assert all(torch.equal(s0[k], s1[k]) for k in s0)
    assert float(ours._step[0]) == 3.0
    # the parameters moved by three Adam steps (each up to ~lr per element); the two runs agree to a small fraction
    disp = torch.cat([(e_stock[k] - s0[k]).flatten() for k in s0])
    diff = torch.cat([(e_ours[k] - e_stock[k]).flatten() for k in s0])
    rel = float(diff.norm() / disp.norm())
    print("fine-tuning loop: losses stock %s, flat %s; |p_flat - p_stock| / |displacement| = %.2e, max |diff| %.2e"
          % ([round(v, 4) for v in l_stock], [round(v, 4) for v in l_ours], rel, float(diff.abs().max())))
    assert float(disp.norm()) > 0 and rel < 2e-2, rel
    assert float(diff.abs().max()) <= 3 * 1e-3


def test_table_longer_than_one_launch(dev):
    """48 blocks of a 64-wide MultiViT, each parameter in the other group from its neighbours: ~580 segments, two launches
    of the update kernel (+ the step-count advance); every element against the float64 restatement."""
    from functools import partial
    from multimae_b200 import _lib as L
    from multimae_b200 import optim as O
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    torch.manual_seed(0)
    model = MultiViT({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=32)}, None,
                     dim_tokens=64, depth=48, num_heads=2, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6)).to(dev)
    params = [p for p in model.parameters() if p.requires_grad]
    groups = [{"params": params[0::2], "weight_decay": 0.05}, {"params": params[1::2], "weight_decay": 0.0}]
    opt = O.GroupedFlatAdamW(groups, lr=1e-3, betas=BETAS, eps=EPS)
    assert len(opt.segments) == len(params) > 448 and [s[2] for s in opt.segments[:4]] == [0, 1, 0, 1]
    err = _Err()
    start = [p.detach().clone() for p in params]
    for it in range(2):
        _set_grads([model], it, dev)
        before = L.lib().mmae_launch_count()
        _step_and_check(opt, model, err, dev)
        assert L.lib().mmae_launch_count() - before == 3
    print("long table: %d segments, max error (ulps) %s" % (len(opt.segments), err.worst))
    assert err.max() <= ULP_BUDGET
    assert all(not torch.equal(p, s) for p, s in zip(params, start))
    assert torch.equal(opt.flat_bf16, opt.flat_params.to(torch.bfloat16))
