"""GPU: the semantic-segmentation head of fine-tuning (ConvNeXtAdapter -> mmae_convnext_*) and the body of the reference's
run_finetuning_semseg.py train_one_epoch over the overlay classes.  Nothing here reads the reference checkout."""
import math

import pytest
import torch

from cls_head_oracle import vit_config
from convnext_head_oracle import convnext_head, fill_, inputs, seg_loss
from helpers import digest, load_fixture, rel_l2
from test_convnext_head_host import _model

pytestmark = pytest.mark.gpu

BF16_TOL = 1e-2       # the head: outputs and gradients, relative L2
MODEL_TOL = 2e-2      # multivit_base + head, whole model


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def _enc_tokens(p, x, cfg):
    """cls_head_oracle.encoder_tokens with the token indices on the inputs' device."""
    from oracle import multimae_oracle as O
    B, dev = next(iter(x.values())).shape[0], next(iter(x.values())).device
    total = sum((v.shape[-1] // 16) * (v.shape[-2] // 16) for v in x.values())
    ids = torch.arange(total, device=dev).unsqueeze(0).expand(B, -1).contiguous()
    return O.forward(p, x, cfg, ids, ids)[1]


def _digest_err(got, ref, scale):
    """Relative error of a gradient against its recorded digest (norm + strided samples), measured against
    max(its own norm, `scale`): the error of the full tensor is estimated from the samples."""
    d = digest(got.cpu())
    den = max(float(ref["norm"]), scale)
    full = float((d["samples"] - ref["samples"]).norm()) * float(ref["norm"]) / max(float(ref["samples"].norm()), 1e-30)
    return max(abs(float(d["norm"]) - float(ref["norm"])), full) / den


def test_fixture_model_on_cuda(golden_dir, dev):
    """The reference's MultiViT + two ConvNeXtAdapters recorded by make_golden_convnext.py: outputs, loss and every
    parameter gradient (stored as norm + strided samples)."""
    fx = load_fixture(golden_dir, "convnext_head.pt")
    model = _model()
    fill_(model.named_parameters())
    model = model.to(dev).train()
    outs = model({k: v.to(dev) for k, v in fx["inputs"].items()})
    for k, ref in fx["outputs"].items():
        assert outs[k].dtype == torch.float32 and outs[k].shape == ref.shape
        assert rel_l2(outs[k], ref) < BF16_TOL, (k, rel_l2(outs[k], ref))
    loss = seg_loss(outs, fx["labels"])
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss.detach()) - float(fx["loss"])) < BF16_TOL * abs(float(fx["loss"]))
    got = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
    assert set(got) == set(fx["grads"])
    # every gradient against max(its own norm, the norm it would have at the global RMS).  Some tensors of this small model
    # carry almost no gradient and are rounding-dominated under any bf16 arithmetic: the key part of the qkv bias gradient
    # is zero up to rounding (softmax ignores a per-query constant), and the x8 head's first block (dwconv / norm weight
    # gradients ~4000x below its final_layer's) moves by 13-14 % when the reference's own math runs under bf16 autocast
    numel = {k: math.prod(s) for k, s in fx["schema"]}
    G = math.sqrt(sum(float(r["norm"]) ** 2 for r in fx["grads"].values()))
    total = sum(numel[k] for k in fx["grads"])
    errs = {k: _digest_err(got[k], ref, G * math.sqrt(numel[k] / total)) for k, ref in fx["grads"].items()}
    own = {k: _digest_err(got[k], ref, 0.0) for k, ref in fx["grads"].items() if k.startswith("output_adapters.")}
    worst, worst_own = max(errs, key=errs.get), max(own, key=own.get)
    print("fixture gradients: worst %s %.2e; worst head gradient against its own norm %s %.2e" % (
        worst, errs[worst], worst_own, own[worst_own]))
    assert errs[worst] < BF16_TOL, (worst, errs[worst])


def _head_params(ad, dev, seed):
    """The adapter's parameters with perturbed biases and LayerNorm weights, as an oracle dict (prefix 'h.')."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in ad.named_parameters():
            if n.endswith(".bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif n.endswith("norm.weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    ad.to(dev)
    return {"h." + k: v.detach().clone().requires_grad_(True) for k, v in ad.named_parameters()}


def _info(H, W, tasks):
    n = (H // 16) * (W // 16)
    return {"image_size": (H, W), "num_task_tokens": n * len(tasks), "num_global_tokens": 1,
            "tasks": {t: {"num_tokens": n, "start_idx": i * n, "end_idx": (i + 1) * n} for i, t in enumerate(tasks)}}


@pytest.mark.parametrize("B,H,W,tasks,main,K", [
    (4, 512, 512, ("rgb",), ("rgb",), 150),
    (4, 512, 512, ("rgb",), ("rgb",), 151),
    (4, 512, 512, ("rgb",), ("rgb",), 40),
    (2, 512, 512, ("rgb", "depth"), ("rgb", "depth"), 150),
    (1, 512, 640, ("rgb",), ("rgb",), 41),
])
def test_adapter_against_fp32_restatement(dev, B, H, W, tasks, main, K):
    """The adapter alone at the shipped configs' shapes (embed 6144, 16 predictions per patch, depth 4) on identical encoder
    tokens: output, encoder-token gradient and every parameter gradient against fp32 torch autograd."""
    from multimae_b200.output_adapters import ConvNeXtAdapter
    torch.manual_seed(K)
    ad = ConvNeXtAdapter(K, embed_dim=6144, preds_per_patch=16, depth=4, main_tasks=list(main))
    ad.init(768)
    p = _head_params(ad, dev, K)
    info = _info(H, W, tasks)
    N = info["num_task_tokens"] + 1
    enc = torch.randn(B, N, 768, device=dev)
    e_ref = enc.clone().requires_grad_(True)
    n = info["tasks"]["rgb"]["num_tokens"]
    ref = convnext_head(e_ref, p, [info["tasks"][t]["start_idx"] for t in main], n, H, W, 16, 4, prefix="h.")
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
    print("B=%d %dx%d tasks=%s K=%d: out %.2e enc %.2e worst %s %.2e" % (B, H, W, main, K, errs["out"], errs["enc"], worst,
                                                                         errs[worst]))
    assert errs[worst] < BF16_TOL, (worst, errs[worst])
    other = [i for i, t in enumerate(tasks) if t not in main]
    assert not e.grad[:, -1].any()                       # the global token
    for i in other:
        assert not e.grad[:, i * n:(i + 1) * n].any()


def _oracle_model_case(dev, size, tasks, main, K, B, seed):
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    from multimae_b200.output_adapters import ConvNeXtAdapter
    from oracle import multimae_oracle as O
    torch.manual_seed(seed)
    ch = {"rgb": 3, "depth": 1}
    model = multivit_base({t: PatchedInputAdapter(num_channels=ch[t], stride_level=1, patch_size_full=16, image_size=size)
                           for t in tasks},
                          {"semseg": ConvNeXtAdapter(K, embed_dim=6144, preds_per_patch=16, depth=4, main_tasks=list(main))})
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith(".bias") or n == "global_tokens":
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif n.endswith("norm.weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    sd = {k: v.detach().clone().to(dev) for k, v in model.state_dict().items()}
    x = {t: torch.randn(B, ch[t], size, size, generator=g) for t in tasks}
    model = model.to(dev).train()
    cfg = vit_config(tasks, 768, 12, 12, size)
    train = O.trainable(sd)
    for v in train.values():
        v.requires_grad_(True)
    enc = _enc_tokens(sd, {k: v.to(dev) for k, v in x.items()}, cfg)
    n = (size // 16) ** 2
    ref = convnext_head(enc, sd, [tasks.index(t) * n for t in main], n, size, size, 16, 4,
                        prefix="output_adapters.semseg.")
    return model, sd, train, x, ref


@pytest.mark.parametrize("size,tasks,main,K,B", [(512, ("rgb",), ("rgb",), 150, 2),
                                                 (640, ("rgb", "depth"), ("rgb",), 41, 1)])
def test_multivit_base_against_oracle(dev, size, tasks, main, K, B):
    """multivit_base + ConvNeXtAdapter end to end: the ADE shape (512 x 512 rgb, 1025 encoder tokens) and the NYU shape
    (640 x 640 rgb-depth with main task rgb, 3201 encoder tokens): output and every parameter gradient against the oracle
    encoder + the fp32 head."""
    model, sd, train, x, ref = _oracle_model_case(dev, size, tasks, main, K, B, seed=size + K)
    out = model({k: v.to(dev) for k, v in x.items()})["semseg"]
    dout = torch.randn(ref.shape, device=dev)
    ref.backward(dout)
    out.backward(dout)
    torch.cuda.synchronize()
    assert rel_l2(out, ref) < MODEL_TOL, rel_l2(out, ref)
    got = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
    errs = {k: rel_l2(got[k], v.grad) for k, v in train.items() if v.grad is not None}
    glob = float(torch.cat([(got[k] - train[k].grad).flatten() for k in errs]).norm()
                 / torch.cat([train[k].grad.flatten() for k in errs]).norm())
    head = {k: v for k, v in errs.items() if k.startswith("output_adapters.")}
    worst = max(head, key=head.get)
    print("%d x %d %s: out %.2e, global grad %.2e, worst head grad %s %.2e, median %.2e" % (
        size, size, tasks, rel_l2(out, ref), glob, worst, head[worst], sorted(errs.values())[len(errs) // 2]))
    assert glob < MODEL_TOL and head[worst] < MODEL_TOL and sorted(errs.values())[len(errs) // 2] < MODEL_TOL


def _small_semseg(K=5, size=64):
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import ConvNeXtAdapter
    from functools import partial
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=size)}
    outs = {"semseg": ConvNeXtAdapter(K, embed_dim=2048, preds_per_patch=16, depth=2)}
    return MultiViT(ins, outs, num_global_tokens=1, dim_tokens=128, depth=2, num_heads=2, mlp_ratio=4, qkv_bias=True,
                    drop_path_rate=0.0, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def test_repeatable_and_eval_bitwise(dev):
    """Two forward + backward passes give bitwise-equal outputs, encoder-token gradients and depthwise-conv weight / bias
    gradients (no split-K, no atomics on that chain); the torch.no_grad() eval forward equals the training forward."""
    from multimae_b200.output_adapters import ConvNeXtAdapter
    torch.manual_seed(3)
    ad = ConvNeXtAdapter(150, embed_dim=6144, preds_per_patch=16, depth=4)
    ad.init(768)
    _head_params(ad, dev, 3)
    info = _info(512, 512, ("rgb",))
    enc = torch.randn(4, 1025, 768, device=dev)
    dout = torch.randn(4, 150, 512, 512, device=dev)
    runs = []
    for _ in range(2):
        ad.zero_grad(set_to_none=True)
        e = enc.clone().requires_grad_(True)
        out = ad.train()(e, info)
        out.backward(dout)
        torch.cuda.synchronize()
        runs.append((out.detach().clone(), e.grad.clone(),
                     {k: v.grad.clone() for k, v in ad.named_parameters() if "dwconv" in k}))
    assert torch.equal(runs[0][0], runs[1][0])
    assert torch.equal(runs[0][1], runs[1][1])
    for k in runs[0][2]:
        assert torch.equal(runs[0][2][k], runs[1][2][k]), k
    with torch.no_grad():
        ev = ad.eval()(enc, info)
    torch.cuda.synchronize()
    assert ev.grad_fn is None and torch.equal(ev, runs[0][0])
    # the same through a model under autocast, as the script's evaluate()
    model = _small_semseg().to(dev)
    x = torch.randn(3, 3, 64, 64, device=dev)
    with torch.autocast("cuda", dtype=torch.float16):
        train = model.train()(x)["semseg"]
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        ev = model.eval()(x)["semseg"]
    torch.cuda.synchronize()
    assert torch.equal(ev, train.detach())


def _param_groups(model, weight_decay, layer_decay):
    """utils/optim_factory.py get_parameter_groups with LayerDecayValueAssigner (run_finetuning_semseg.py)."""
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
        g = groups.setdefault(key, {"weight_decay": 0.0 if no_decay else weight_decay, "params": [], "lr_scale": values[lid]})
        g["params"].append(p)
    return list(groups.values())


def test_finetune_semseg_train_one_epoch_sequence(dev):
    """run_finetuning_semseg.py's train_one_epoch step restated over the overlay classes with the REAL library, two steps:
    autocast, CrossEntropyLoss(ignore_index=255), NativeScalerWithGradNormCount with loss scaling, layer-decay parameter
    groups on the stock torch.optim.AdamW, arena-owned gradients.  Each step's gradient norm matches the fp32 oracle's at
    the same parameter values."""
    from multimae_b200 import multimae as mm
    from multimae_b200 import overlay
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from oracle import multimae_oracle as O
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True
    try:
        torch.manual_seed(0)
        K, B = 5, 4
        model = overlay._IdentityDDP(_small_semseg(K).to(dev), device_ids=[0])
        model_without_ddp = model.module
        optimizer = torch.optim.AdamW(_param_groups(model_without_ddp, 0.05, 0.75), lr=1e-4)
        loss_scaler = NativeScalerWithGradNormCount()
        criterion = torch.nn.CrossEntropyLoss(ignore_index=255)
        g = torch.Generator().manual_seed(7)
        x = torch.randn(B, 3, 64, 64, generator=g).to(dev)
        target = torch.randint(0, K, (B, 64, 64), generator=g)
        target[torch.rand(target.shape, generator=g) < 0.1] = 255
        target = target.to(dev)
        cfg = vit_config(("rgb",), 128, 2, 2, 64)
        model.train(True)
        for step in range(2):
            for group in optimizer.param_groups:
                group["lr"] = 1e-4 * group["lr_scale"]
            sd = {k: v.detach().clone() for k, v in model_without_ddp.state_dict().items()}
            train = O.trainable(sd)
            for v in train.values():
                v.requires_grad_(True)
            enc = _enc_tokens(sd, {"rgb": x}, cfg)
            ref = convnext_head(enc, sd, [0], 16, 64, 64, 16, 2, prefix="output_adapters.semseg.")
            criterion(ref, target).backward()
            ref_norm = float(torch.cat([v.grad.flatten() for v in train.values() if v.grad is not None]).norm())
            with torch.autocast("cuda", dtype=torch.float16):
                preds = model({"rgb": x})
                loss = criterion(preds["semseg"], target)
            loss_value = loss.item()
            assert math.isfinite(loss_value)
            optimizer.zero_grad()
            grad_norm = loss_scaler(loss, optimizer, clip_grad=None, parameters=model.parameters(), create_graph=False,
                                    update_grad=True)
            torch.cuda.synchronize()
            arena = model_without_ddp.grad_arena()
            assert arena.owned and loss_scaler.state_dict()["scale"] == 65536.0
            err = abs(float(grad_norm) - ref_norm) / ref_norm
            print("step %d: loss %.4f, grad norm %.4f (oracle %.4f, %.2e)" % (step, loss_value, float(grad_norm), ref_norm, err))
            assert err < MODEL_TOL, (step, float(grad_norm), ref_norm)
    finally:
        mm.AUTO_OWN_GRADIENTS = old
