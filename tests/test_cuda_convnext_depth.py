"""GPU: depth fine-tuning with the ConvNeXt head (run_finetuning_depth.py --output_adapter convnext): the LayerNorm kernels
for row widths that are multiples of 32 but not of 128, the head at 96 channels per pixel, multivit_base + head, and the
body of the script's train_one_epoch over the overlay classes.  Nothing here reads the reference checkout.

The script runs its forward under autocast(enabled=False); here, as for every script, the GEMMs take bf16 operands with
fp32 accumulation, so the tolerances are the bf16 budgets of the semantic-segmentation head tests."""
import math

import pytest
import torch

from cls_head_oracle import vit_config
from convnext_depth_oracle import depth_loss, fill_, inputs, masked_berhu_loss
from convnext_head_oracle import convnext_head
from helpers import load_fixture, rel_l2
from test_convnext_depth_host import _model, oracle_outputs
from test_cuda_convnext_head import BF16_TOL, MODEL_TOL, _digest_err, _enc_tokens, _head_params, _info, _param_groups

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------------ narrow LayerNorm
@pytest.mark.parametrize("D", [32, 64, 96, 160, 992])
@pytest.mark.parametrize("M", [1, 13, 4099, 65541])
def test_layernorm_narrow_against_float64(dev, D, M):
    """Forward (bf16 and fp32 outputs, mean, rstd, a strided input) and backward (fp32 and bf16 dy, with and without
    dx_resid; dgamma / dbeta accumulated into non-zero buffers) against float64, on ragged row counts."""
    from multimae_b200 import kernels as K
    g = torch.Generator(device=dev).manual_seed(D * 7 + M)
    base = torch.randn(M, D + 32, device=dev, generator=g) * 2.0 + 0.5
    x = base[:, 16:16 + D]                                          # leading dimension D + 32
    gamma = 1.0 + 0.1 * torch.randn(D, device=dev, generator=g)
    beta = 0.1 * torch.randn(D, device=dev, generator=g)
    yb, yf, mean, rstd = K.layernorm_fwd(x, gamma, beta, 1e-6, out_bf16=True, out_f32=True)
    x64 = x.double()
    m64 = x64.mean(1)
    r64 = torch.rsqrt(((x64 - m64[:, None]) ** 2).mean(1) + 1e-6)
    xh = (x64 - m64[:, None]) * r64[:, None]
    y64 = xh * gamma.double() + beta.double()
    torch.cuda.synchronize()
    assert rel_l2(yf, y64) < 1e-6 and rel_l2(mean, m64) < 1e-6 and rel_l2(rstd, r64) < 1e-6
    assert rel_l2(yb, y64) < 4e-3 and torch.equal(yb, yf.to(torch.bfloat16))
    for dy_bf16 in (False, True):
        dy = torch.randn(M, D, device=dev, generator=g)
        if dy_bf16:
            dy = dy.to(torch.bfloat16)
        resid = torch.randn(M, D, device=dev, generator=g) if dy_bf16 else None
        dg0, db0 = torch.randn(D, device=dev, generator=g), torch.randn(D, device=dev, generator=g)
        dgamma, dbeta = dg0.clone(), db0.clone()
        dx = K.layernorm_bwd(dy, x, mean, rstd, gamma, dgamma, dbeta, dx_resid=resid)
        d64 = dy.double()
        gg = d64 * gamma.double()
        dx64 = r64[:, None] * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
        if resid is not None:
            dx64 = dx64 + resid.double()
        torch.cuda.synchronize()
        assert rel_l2(dx, dx64) < 1e-5, (dy_bf16, rel_l2(dx, dx64))
        assert rel_l2(dgamma - dg0, (d64 * xh).sum(0)) < 1e-5
        assert rel_l2(dbeta - db0, d64.sum(0)) < 1e-5


# ------------------------------------------------------------------------------------------------ the fixture model
def test_fixture_model_on_cuda(golden_dir, dev):
    """The reference's MultiViT + the 32- and 96-channel heads recorded by make_golden_convnext_depth.py: outputs, the
    berhu + L1 loss against the fixed mask_valid, and every parameter gradient.

    Each output and gradient is held to BF16_TOL, or to twice the error of the reference's own math under bf16 autocast
    where that is larger (the two round at different points: autocast also rounds the depthwise convolution's operands,
    this path keeps them fp32).  The 32-channel head's single output channel is a sum of 32 products that largely cancel
    (output RMS 0.16): the fp32 restatement run under CPU bf16 autocast is 2.3 % away from the recording there (0.9 % for
    the 96-channel head) and 10 % on that head's proj_dec weight gradient."""
    from oracle import multimae_oracle as O
    fx = load_fixture(golden_dir, "convnext_depth.pt")
    model = _model()
    fill_(model.named_parameters())
    p = {k: v.detach().clone() for k, v in model.state_dict().items()}
    train = O.trainable(p)
    for v in train.values():
        v.requires_grad_(True)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        ref_bf16 = oracle_outputs(p, fx["inputs"])
    depth_loss({k: v.float() for k, v in ref_bf16.items()}, fx["target"], fx["mask_valid"]).backward()
    model = model.to(dev).train()
    outs = model({k: v.to(dev) for k, v in fx["inputs"].items()})
    for k, ref in fx["outputs"].items():
        assert outs[k].dtype == torch.float32 and outs[k].shape == ref.shape
        err, own = rel_l2(outs[k], ref), rel_l2(ref_bf16[k].float(), ref)
        print("output %s: %.2e (the reference under bf16 autocast: %.2e)" % (k, err, own))
        assert err < max(BF16_TOL, 2 * own), (k, err, own)
    loss = depth_loss(outs, fx["target"], fx["mask_valid"])
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss.detach()) - float(fx["loss"])) < BF16_TOL * abs(float(fx["loss"]))
    got = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
    assert set(got) == set(fx["grads"])
    numel = {k: math.prod(s) for k, s in fx["schema"]}
    G = math.sqrt(sum(float(r["norm"]) ** 2 for r in fx["grads"].values()))
    total = sum(numel[k] for k in fx["grads"])
    scale = {k: G * math.sqrt(numel[k] / total) for k in fx["grads"]}
    errs = {k: _digest_err(got[k], ref, scale[k]) for k, ref in fx["grads"].items()}
    own = {k: _digest_err(train[k].grad, ref, scale[k]) for k, ref in fx["grads"].items()}
    worst = max(errs, key=lambda k: errs[k] / max(BF16_TOL, 2 * own[k]))
    print("fixture gradients: worst %s %.2e (the reference under bf16 autocast: %.2e)" % (worst, errs[worst], own[worst]))
    assert errs[worst] < max(BF16_TOL, 2 * own[worst]), (worst, errs[worst], own[worst])


# ------------------------------------------------------------------------------------------------ the script's shapes
@pytest.mark.parametrize("main,depth,K", [(("rgb",), 4, 1), (("rgb", "depth"), 2, 1), (("rgb",), 2, 3)])
def test_adapter_against_fp32_restatement(dev, main, depth, K):
    """The adapter alone at the script's shapes: B = 4, 256 x 256, embed 6144, 64 predictions per patch (C = 96, s = 8),
    one output channel (and three, a regression head with more outputs); output, encoder-token gradient and every
    parameter gradient against fp32 torch autograd."""
    from multimae_b200.output_adapters import ConvNeXtAdapter
    torch.manual_seed(len(main) * 10 + depth + K)
    ad = ConvNeXtAdapter(K, embed_dim=6144, preds_per_patch=64, depth=depth, main_tasks=list(main))
    ad.init(768)
    p = _head_params(ad, dev, depth)
    B, H, W = 4, 256, 256
    info = _info(H, W, ("rgb", "depth"))
    enc = torch.randn(B, info["num_task_tokens"] + 1, 768, device=dev)
    e_ref = enc.clone().requires_grad_(True)
    n = info["tasks"]["rgb"]["num_tokens"]
    ref = convnext_head(e_ref, p, [info["tasks"][t]["start_idx"] for t in main], n, H, W, 64, depth, prefix="h.")
    dout = torch.randn(ref.shape, device=dev)
    ref.backward(dout)
    e = enc.clone().requires_grad_(True)
    out = ad(e, info)
    out.backward(dout)
    torch.cuda.synchronize()
    assert out.shape == (B, K, H, W)
    errs = {"out": rel_l2(out, ref), "enc": rel_l2(e.grad, e_ref.grad)}
    for k, v in ad.named_parameters():
        errs[k] = rel_l2(v.grad, p["h." + k].grad)
    worst = max(errs, key=errs.get)
    print("main=%s depth=%d K=%d: out %.2e enc %.2e worst %s %.2e" % (main, depth, K, errs["out"], errs["enc"], worst,
                                                                     errs[worst]))
    assert errs[worst] < BF16_TOL, (worst, errs[worst])
    if "depth" not in main:
        assert not e.grad[:, n:2 * n].any()
    assert not e.grad[:, -1].any()


def test_multivit_base_against_oracle(dev):
    """multivit_base on rgb + depth at 256 x 256 with the script's head (main tasks rgb-depth, depth 4): output and every
    parameter gradient against the oracle encoder + the fp32 head."""
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    from multimae_b200.output_adapters import ConvNeXtAdapter
    from oracle import multimae_oracle as O
    torch.manual_seed(256)
    tasks, ch, size, B = ("rgb", "depth"), {"rgb": 3, "depth": 1}, 256, 2
    model = multivit_base({t: PatchedInputAdapter(num_channels=ch[t], stride_level=1, patch_size_full=16, image_size=size)
                           for t in tasks},
                          {"depth": ConvNeXtAdapter(1, preds_per_patch=64, main_tasks=list(tasks))})
    g = torch.Generator().manual_seed(257)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith(".bias") or n == "global_tokens":
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif n.endswith("norm.weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    sd = {k: v.detach().clone().to(dev) for k, v in model.state_dict().items()}
    x = {t: torch.randn(B, ch[t], size, size, generator=g).to(dev) for t in tasks}
    model = model.to(dev).train()
    train = O.trainable(sd)
    for v in train.values():
        v.requires_grad_(True)
    enc = _enc_tokens(sd, x, vit_config(tasks, 768, 12, 12, size))
    n = (size // 16) ** 2
    ref = convnext_head(enc, sd, [0, n], n, size, size, 64, 4, prefix="output_adapters.depth.")
    out = model(x)["depth"]
    dout = torch.randn(ref.shape, device=dev)
    ref.backward(dout)
    out.backward(dout)
    torch.cuda.synchronize()
    assert rel_l2(out, ref) < MODEL_TOL, rel_l2(out, ref)
    got = {k: p.grad for k, p in model.named_parameters() if p.requires_grad}
    errs = {k: rel_l2(got[k], v.grad) for k, v in train.items() if v.grad is not None}
    glob = float(torch.cat([(got[k] - train[k].grad).flatten() for k in errs]).norm()
                 / torch.cat([train[k].grad.flatten() for k in errs]).norm())
    head = {k: v for k, v in errs.items() if k.startswith("output_adapters.")}
    worst = max(head, key=head.get)
    print("out %.2e, global grad %.2e, worst head grad %s %.2e" % (rel_l2(out, ref), glob, worst, head[worst]))
    assert glob < MODEL_TOL and head[worst] < MODEL_TOL and sorted(errs.values())[len(errs) // 2] < MODEL_TOL


def test_eval_forward_bitwise_repeatable(dev):
    """The torch.no_grad() eval forward of the script's head (batch 6 = 1.5 x 4, as the script's validation loader) is
    bitwise repeatable and equals the training forward."""
    from multimae_b200.output_adapters import ConvNeXtAdapter
    torch.manual_seed(5)
    ad = ConvNeXtAdapter(1, embed_dim=6144, preds_per_patch=64, depth=4)
    ad.init(768)
    _head_params(ad, dev, 5)
    info = _info(256, 256, ("rgb",))
    enc = torch.randn(6, 257, 768, device=dev)
    with torch.no_grad():
        ev = [ad.eval()(enc, info) for _ in range(2)]
    train = ad.train()(enc.clone().requires_grad_(True), info)
    torch.cuda.synchronize()
    assert ev[0].grad_fn is None and torch.equal(ev[0], ev[1]) and torch.equal(ev[0], train.detach())


# ------------------------------------------------------------------------------------------------ train_one_epoch
def _small_depth(size=64, dpe=0.1):
    from functools import partial

    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import ConvNeXtAdapter
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=size),
           "depth": PatchedInputAdapter(num_channels=1, stride_level=1, patch_size_full=16, image_size=size)}
    outs = {"depth": ConvNeXtAdapter(1, preds_per_patch=64, depth=2, main_tasks=["rgb", "depth"])}
    return MultiViT(ins, outs, num_global_tokens=1, dim_tokens=128, depth=2, num_heads=2, mlp_ratio=4, qkv_bias=True,
                    drop_path_rate=dpe, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def test_finetune_depth_train_one_epoch_sequence(dev):
    """run_finetuning_depth.py's train_one_epoch step restated over the overlay classes with the REAL library: the script's
    inline masking of the depth input, autocast(enabled=False), masked berhu, NativeScalerWithGradNormCount(enabled=False),
    layer-decay groups; two steps on the stock torch.optim.AdamW, then two on GroupedFlatAdamW (MMAE_FLAT_ADAMW=1).  Each
    step's loss and gradient norm match the fp32 oracle's at the same parameter values (eval-mode drop path: rate 0)."""
    from multimae_b200 import multimae as mm
    from multimae_b200 import overlay
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import GroupedFlatAdamW, adamw_or_stock
    from oracle import multimae_oracle as O
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True
    try:
        torch.manual_seed(0)
        model = overlay._IdentityDDP(_small_depth(dpe=0.0).to(dev), device_ids=[0])
        model_without_ddp = model.module
        loss_scaler = NativeScalerWithGradNormCount(enabled=False)
        x, target, mask_valid = inputs(dict(B=4, H=64, W=64))
        tasks_dict = {"rgb": x["rgb"].to(dev), "depth": target.to(dev), "mask_valid": mask_valid.to(dev)}
        cfg = vit_config(("rgb", "depth"), 128, 2, 2, 64)
        losses = []
        for phase, make in (("stock", lambda groups: torch.optim.AdamW(groups, lr=1e-4)),
                            ("flat", lambda groups: adamw_or_stock(groups, lr=1e-4))):
            optimizer = make(_param_groups(model_without_ddp, 1e-4, 0.75))
            assert isinstance(optimizer, GroupedFlatAdamW) == (phase == "flat")
            model.train(True)
            for step in range(2):
                for group in optimizer.param_groups:
                    group["lr"] = 1e-4 * group["lr_scale"]
                input_dict = {t: v for t, v in tasks_dict.items() if t in ("rgb", "depth")}
                input_dict = {t: v.clone() for t, v in input_dict.items()}
                for task in input_dict:                                     # run_finetuning_depth.py:690-695
                    if task in ["rgb"]:
                        continue
                    channels = input_dict[task].shape[1]
                    input_dict[task][~tasks_dict["mask_valid"].repeat_interleave(repeats=channels, dim=1)] = 0.0
                sd = {k: v.detach().clone() for k, v in model_without_ddp.state_dict().items()}
                train = O.trainable(sd)
                for v in train.values():
                    v.requires_grad_(True)
                enc = _enc_tokens(sd, input_dict, cfg)
                ref = convnext_head(enc, sd, [0, 16], 16, 64, 64, 64, 2, prefix="output_adapters.depth.")
                ref_loss = masked_berhu_loss(ref, tasks_dict["depth"], tasks_dict["mask_valid"])
                ref_loss.backward()
                ref_norm = float(torch.cat([v.grad.flatten() for v in train.values() if v.grad is not None]).norm())
                with torch.cuda.amp.autocast(enabled=False):
                    preds = model(input_dict, return_all_layers=False)
                    loss = masked_berhu_loss(preds["depth"].float(), tasks_dict["depth"], tasks_dict["mask_valid"])
                loss_value = loss.item()
                assert math.isfinite(loss_value)
                optimizer.zero_grad()
                grad_norm = loss_scaler(loss, optimizer, clip_grad=None, parameters=model.parameters(), create_graph=False)
                torch.cuda.synchronize()
                assert model_without_ddp.grad_arena().owned
                ref_loss = float(ref_loss.detach())
                lerr = abs(loss_value - ref_loss) / abs(ref_loss)
                gerr = abs(float(grad_norm) - ref_norm) / ref_norm
                print("%s step %d: loss %.5f (oracle %.5f), grad norm %.4f (oracle %.4f, %.2e)" % (
                    phase, step, loss_value, ref_loss, float(grad_norm), ref_norm, gerr))
                assert lerr < BF16_TOL and gerr < MODEL_TOL, (phase, step, lerr, gerr)
                losses.append(loss_value)
        assert losses[-1] < losses[0], losses
    finally:
        mm.AUTO_OWN_GRADIENTS = old
