"""GPU: the Segmenter head of semantic-segmentation fine-tuning (SegmenterMaskTransformerAdapter -> mmae_segmenter_*) and
the body of the reference's run_finetuning_semseg.py train_one_epoch over the overlay classes.  Nothing here reads the
reference checkout."""
import math
from functools import partial

import pytest
import torch

from helpers import load_fixture, rel_l2
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from segmenter_head_oracle import cosine_mask, fill_, seg_loss, segmenter_head
from test_cuda_convnext_head import _digest_err, _info, _param_groups
from test_segmenter_head_host import _model

pytestmark = pytest.mark.gpu

BF16_TOL = 1e-2       # the head: outputs and gradients, relative L2
FEW_CLASSES_TOL = 3e-2   # heads of 8 to 13 classes: the class LayerNorm divides by the spread of that few cosines
FIXTURE_OUT_TOL, FIXTURE_GRAD_TOL = 4e-2, 1e-1     # the tiny fixture model (test_fixture_model_on_cuda says why)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


def test_fixture_model_on_cuda(golden_dir, dev):
    """The reference's MultiViT + two Segmenter heads recorded by make_golden_segmenter.py: outputs, loss and every
    parameter gradient (stored as norm + strided samples), measured against max(its own norm, its share of the global norm).
    The fixture's heads have 9 and 13 classes on a 12-patch, 128-wide model: mask_norm divides by the spread of that few
    cosines, forwards and again backwards, which multiplies what any half-precision arithmetic in front of it differs by.
    torch's own bf16 autocast of the same math on this fixture (the oracle on the CPU) differs from fp32 by 3.3e-2 in the
    outputs and 1.05e-1 over all gradients (1.3e-1 on semseg.proj_dec.bias); FIXTURE_OUT_TOL / FIXTURE_GRAD_TOL are set
    from that.  What holds the kernels to BF16_TOL is the head at 41 classes and more, and the mask kernel alone, below."""
    fx = load_fixture(golden_dir, "segmenter_head.pt")
    model = _model()
    fill_(model.named_parameters())
    model = model.to(dev).train()
    outs = model({k: v.to(dev) for k, v in fx["inputs"].items()})
    out_err = {k: rel_l2(outs[k], ref) for k, ref in fx["outputs"].items()}
    for k, ref in fx["outputs"].items():
        assert outs[k].dtype == torch.float32 and outs[k].shape == ref.shape
    loss = seg_loss(outs, fx["labels"])
    loss.backward()
    torch.cuda.synchronize()
    got = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
    assert set(got) == set(fx["grads"])
    numel = {k: math.prod(s) for k, s in fx["schema"]}
    G = math.sqrt(sum(float(r["norm"]) ** 2 for r in fx["grads"].values()))
    total = sum(numel[k] for k in fx["grads"])
    errs = {k: _digest_err(got[k], ref, G * math.sqrt(numel[k] / total)) for k, ref in fx["grads"].items()}
    # all tensors together (each one's error weighted by the norm it was measured against), and the heads' own tensors one
    # by one.  Single small encoder tensors of this formula-filled model are rounding-dominated under any bf16 arithmetic
    # (the key part of a qkv bias gradient is zero up to rounding: softmax ignores a per-query constant).
    scale = {k: max(float(fx["grads"][k]["norm"]), G * math.sqrt(numel[k] / total)) for k in errs}
    glob = math.sqrt(sum((errs[k] * scale[k]) ** 2 for k in errs)) / math.sqrt(sum(v * v for v in scale.values()))
    head = {k: v for k, v in errs.items() if k.startswith("output_adapters.")}
    worst, worst_head = max(errs, key=errs.get), max(head, key=head.get)
    loss_err = abs(float(loss.detach()) - float(fx["loss"])) / abs(float(fx["loss"]))
    print("fixture: outputs %s, loss %.2e, all gradients %.2e, worst head gradient %s %.2e, worst %s %.2e" % (
        {k: "%.2e" % v for k, v in out_err.items()}, loss_err, glob, worst_head, head[worst_head], worst, errs[worst]))
    assert max(out_err.values()) < FIXTURE_OUT_TOL, out_err
    assert loss_err < BF16_TOL
    assert glob < FIXTURE_GRAD_TOL and head[worst_head] < FIXTURE_GRAD_TOL, (glob, worst_head, head[worst_head])


def _head(K, dev, seed, depth=2, main=("rgb",), E=768, heads=12, **kw):
    """The adapter with perturbed biases / LayerNorm weights on the device, and its parameters as an oracle dict ('h.')."""
    from multimae_b200.output_adapters import SegmenterMaskTransformerAdapter
    torch.manual_seed(seed)
    ad = SegmenterMaskTransformerAdapter(K, depth=depth, num_heads=heads, embed_dim=E, main_tasks=list(main),
                                         **dict(dict(drop_path_rate=0.0), **kw))
    ad.init(768)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        # class tokens that differ from each other, as trained ones do: at the initial std of 0.02 every class token leaves
        # the blocks nearly equal, the cosines of a patch differ by ~1e-2 over the classes, and mask_norm, which divides by
        # that spread, multiplies the rounding of any half-precision arithmetic several times over
        ad.cls_emb.mul_(25.0)
        for n, p in ad.named_parameters():
            if n.endswith(".bias"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
            elif "norm" in n and n.endswith(".weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    ad.to(dev)
    return ad, {"h." + k: v.detach().clone().requires_grad_(True) for k, v in ad.named_parameters()}


def _compare(ad, p, enc, info, main, depth, heads, scales=None, zero_sample=False):
    H, W = info["image_size"]
    n = info["tasks"]["rgb"]["num_tokens"]
    e_ref = enc.clone().requires_grad_(True)
    ref = segmenter_head(e_ref, p, [info["tasks"][t]["start_idx"] for t in main], n, H, W, depth, heads, prefix="h.",
                         scales=scales)
    dout = torch.randn(ref.shape, device=enc.device)
    ref.backward(dout)
    e = enc.clone().requires_grad_(True)
    out = ad(e, info)
    out.backward(dout)
    torch.cuda.synchronize()
    assert out.shape == ref.shape and bool(torch.isfinite(out).all())
    errs = {"out": rel_l2(out, ref), "enc": rel_l2(e.grad, e_ref.grad)}
    for k, v in ad.named_parameters():
        errs[k] = rel_l2(v.grad, p["h." + k].grad)
    return errs, e


@pytest.mark.parametrize("B,H,W,tasks,main,K,depth", [
    (4, 512, 512, ("rgb",), ("rgb",), 151, 2),
    (2, 512, 640, ("rgb",), ("rgb",), 41, 2),
    (2, 256, 320, ("rgb", "depth"), ("rgb", "depth"), 13, 1),
    (2, 256, 320, ("rgb", "depth"), ("rgb",), 8, 2),
    (1, 320, 256, ("rgb",), ("rgb",), 256, 1),
])
def test_adapter_against_fp32_restatement(dev, B, H, W, tasks, main, K, depth):
    """The adapter alone at width 768 with 12 heads on identical encoder tokens: output, encoder-token gradient and every
    parameter gradient against fp32 torch autograd; depth 1 runs one unchained block, depth 2 the chained pair."""
    ad, p = _head(K, dev, K, depth=depth, main=main)
    info = _info(H, W, tasks)
    enc = torch.randn(B, info["num_task_tokens"] + 1, 768, device=dev)
    errs, e = _compare(ad.train(), p, enc, info, main, depth, 12)
    worst = max(errs, key=errs.get)
    print("B=%d %dx%d tasks=%s K=%d depth=%d: out %.2e enc %.2e worst %s %.2e" % (B, H, W, main, K, depth, errs["out"],
                                                                                errs["enc"], worst, errs[worst]))
    assert errs[worst] < (BF16_TOL if K >= 41 else FEW_CLASSES_TOL), (worst, errs[worst])
    n = info["tasks"]["rgb"]["num_tokens"]
    assert not e.grad[:, -1].any()                       # the global token
    for i, t in enumerate(tasks):
        if t not in main:
            assert not e.grad[:, i * n:(i + 1) * n].any()


def _mask_alone(dev, B, n, K, E, zero_row=True, guard=64):
    """mmae_segmenter_mask_forward / _backward on bf16 P, C against fp64 torch on the same bf16-rounded operands; every
    output sits between guard bands."""
    lib = L.lib()
    g = torch.Generator().manual_seed(K)
    P = torch.randn(B * n, E, generator=g).to(dev).bfloat16()
    C = torch.randn(B * K, E, generator=g).to(dev).bfloat16()
    if zero_row:
        P[1] = 0
    gamma = (1 + 0.1 * torch.randn(K, generator=g)).to(dev)
    beta = (0.1 * torch.randn(K, generator=g)).to(dev)
    rp = 1.0 / P.float().norm(dim=1).clamp_min(1e-12)
    rc = 1.0 / C.float().norm(dim=1).clamp_min(1e-12)
    Kp = (K + 7) // 8 * 8
    SENT = 512.0                                                       # exact in bf16

    def banded(numel, dtype=torch.float32):
        t = torch.full((numel + 2 * guard,), SENT, dtype=dtype, device=dev)
        return t, t[guard:guard + numel]

    cm_f, cmap = banded(B * n * Kp)
    mean_f, mean = banded(B * n)
    rstd_f, rstd = banded(B * n)
    L.check(lib.mmae_segmenter_mask_forward(P.data_ptr(), C.data_ptr(), rp.data_ptr(), rc.data_ptr(), gamma.data_ptr(),
                                            beta.data_ptr(), 1e-6, B, n, K, E, cmap.data_ptr(), mean.data_ptr(),
                                            rstd.data_ptr(), torch.cuda.current_stream().cuda_stream), "mask_forward")
    P64 = P.double().view(B, n, E).requires_grad_(True)
    C64 = C.double().view(B, K, E).requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    ref = cosine_mask(P64, C64, g64, b64)
    got = cmap.view(B * n, Kp)
    dy = torch.randn(B, n, K, device=dev)
    ref.backward(dy.double())
    dcm = torch.zeros(B * n, Kp, device=dev)
    dcm[:, :K] = dy.view(B * n, K)
    dP_f, dP = banded(B * n * E, torch.bfloat16)
    dC_f, dC = banded(B * K * E, torch.bfloat16)
    dg_f, dg = banded(K)
    db_f, db = banded(K)
    dg.zero_()
    db.zero_()
    nws = lib.mmae_segmenter_mask_workspace_bytes(B, n, K)
    ws_f = torch.full((nws + 2 * guard,), 0x5A, dtype=torch.uint8, device=dev)
    L.check(lib.mmae_segmenter_mask_backward(P.data_ptr(), C.data_ptr(), rp.data_ptr(), rc.data_ptr(), gamma.data_ptr(),
                                             mean.data_ptr(), rstd.data_ptr(), dcm.data_ptr(), B, n, K, E, dP.data_ptr(),
                                             dC.data_ptr(), dg.data_ptr(), db.data_ptr(), ws_f.data_ptr() + guard,
                                             torch.cuda.current_stream().cuda_stream), "mask_backward")
    torch.cuda.synchronize()
    for full in (cm_f, mean_f, rstd_f, dP_f, dC_f, dg_f, db_f):
        assert bool((full[:guard].float() == SENT).all()) and bool((full[-guard:].float() == SENT).all())
    assert bool((ws_f[:guard] == 0x5A).all()) and bool((ws_f[-guard:] == 0x5A).all())
    assert not got[:, K:].any()                                        # pad columns of the class map are zero
    return dict(fwd=rel_l2(got[:, :K].double(), ref.detach().view(B * n, K)),
                dP=rel_l2(dP.double().view(B, n, E), P64.grad), dC=rel_l2(dC.double().view(B, K, E), C64.grad),
                dgamma=rel_l2(dg.double(), g64.grad), dbeta=rel_l2(db.double(), b64.grad))


@pytest.mark.parametrize("B,n,K,E", [(4, 1024, 151, 768), (2, 1280, 41, 768), (3, 12, 13, 128), (2, 100, 8, 256),
                                     (1, 77, 256, 1024)])
def test_mask_kernel_alone_and_guard_bands(dev, B, n, K, E):
    """Forward and the parameter gradients hold fp32-accumulation accuracy; dP / dC leave as bf16 (one rounding, 2^-9).
    One patch row is all zero (the 1e-12 clamp).  Nothing is written outside the outputs and the workspace."""
    errs = _mask_alone(dev, B, n, K, E)
    print("mask kernel B=%d n=%d K=%d E=%d: %s" % (B, n, K, E, {k: "%.1e" % v for k, v in errs.items()}))
    assert errs["fwd"] < 1e-4 and errs["dgamma"] < 1e-4 and errs["dbeta"] < 1e-5, errs
    assert errs["dP"] < 4e-3 and errs["dC"] < 4e-3, errs


def test_zero_patch_features(dev):
    """patch_proj.weight = 0: every patch feature is zero, the cosine is 0 / 1e-12 = 0 and the class map is mask_norm.bias."""
    ad, p = _head(13, dev, 5, depth=1, E=128, heads=4)
    with torch.no_grad():
        ad.patch_proj.weight.zero_()
    info = _info(64, 96, ("rgb",))
    out = ad.train()(torch.randn(2, 25, 768, device=dev, requires_grad=True), info)
    out.sum().backward()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())
    torch.testing.assert_close(out, ad.mask_norm.bias.view(1, 13, 1, 1).expand_as(out), rtol=0, atol=1e-5)
    assert all(bool(torch.isfinite(q.grad).all()) for q in ad.parameters())


def test_repeatable_and_eval_bitwise(dev):
    """Two forward + backward passes give bitwise-equal outputs, encoder-token gradients, dcls_emb and mask_norm
    gradients; the torch.no_grad() eval forward equals the training forward (no stochastic depth, no dropout)."""
    ad, _ = _head(151, dev, 3)
    info = _info(512, 512, ("rgb",))
    enc = torch.randn(4, 1025, 768, device=dev)
    dout = torch.randn(4, 151, 512, 512, device=dev)
    runs = []
    for _ in range(2):
        ad.zero_grad(set_to_none=True)
        e = enc.clone().requires_grad_(True)
        out = ad.train()(e, info)
        out.backward(dout)
        torch.cuda.synchronize()
        runs.append((out.detach().clone(), e.grad.clone(),
                     {k: v.grad.clone() for k, v in ad.named_parameters() if k == "cls_emb" or k.startswith("mask_norm")}))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    for k in runs[0][2]:
        assert torch.equal(runs[0][2][k], runs[1][2][k]), k
    with torch.no_grad():
        ev = ad.eval()(enc, info)
    torch.cuda.synchronize()
    assert ev.grad_fn is None and torch.equal(ev, runs[0][0])


def test_drop_path_pinned_and_dropout_reproducible(dev, monkeypatch):
    """drop_path_rate > 0 in training with the per-sample factors pinned: equality with the oracle under the same factors.
    Dropout rates > 0 run, differ from eval, and repeat for a fixed seed."""
    B, K = 4, 41
    ad, p = _head(K, dev, 11, depth=2, drop_path_rate=0.3)
    info = _info(256, 256, ("rgb",))
    enc = torch.randn(B, 257, 768, device=dev)
    g = torch.Generator().manual_seed(1)
    keep = lambda: ((torch.rand(B, generator=g) < 0.7).float() / 0.7).to(dev)        # noqa: E731
    pinned = [None, (keep(), keep())]

    def fake(blocks, batch, device):
        assert batch == B and [Fn.drop_path_prob(b) > 0 for b in blocks] == [False, True]
        return pinned
    monkeypatch.setattr(Fn, "drop_path_scales", fake)
    errs, _ = _compare(ad.train(), p, enc, info, ("rgb",), 2, 12, scales=pinned)
    worst = max(errs, key=errs.get)
    print("pinned drop path: worst %s %.2e" % (worst, errs[worst]))
    assert errs[worst] < BF16_TOL, (worst, errs[worst])
    monkeypatch.undo()
    ad, _ = _head(K, dev, 12, depth=2, drop_rate=0.1, attn_drop_rate=0.1)
    outs = []
    for _ in range(2):
        torch.manual_seed(99)
        outs.append(ad.train()(enc, info).detach().clone())
    with torch.no_grad():
        ev = ad.eval()(enc, info)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], ev) and bool(torch.isfinite(outs[0]).all())


def _small_semseg(K=13, size=64):
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.output_adapters import SegmenterMaskTransformerAdapter
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=size)}
    outs = {"semseg": SegmenterMaskTransformerAdapter(K, embed_dim=128, num_heads=4, depth=2, drop_path_rate=0.1)}
    return MultiViT(ins, outs, num_global_tokens=1, dim_tokens=128, depth=2, num_heads=2, mlp_ratio=4, qkv_bias=True,
                    drop_path_rate=0.0, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))


def test_finetune_semseg_train_one_epoch_sequence(dev):
    """run_finetuning_semseg.py's train_one_epoch step restated over the overlay classes with the real library, two steps
    on a fixed batch: autocast, CrossEntropyLoss(ignore_index=255), NativeScalerWithGradNormCount with loss scaling,
    layer-decay parameter groups on the stock torch.optim.AdamW, arena-owned gradients.  The loss is finite and falls."""
    from multimae_b200 import multimae as mm
    from multimae_b200 import overlay
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True
    try:
        torch.manual_seed(0)
        K, B = 13, 4
        model = overlay._IdentityDDP(_small_semseg(K).to(dev), device_ids=[0])
        optimizer = torch.optim.AdamW(_param_groups(model.module, 0.05, 0.75), lr=1e-3)
        loss_scaler = NativeScalerWithGradNormCount()
        criterion = torch.nn.CrossEntropyLoss(ignore_index=255)
        g = torch.Generator().manual_seed(7)
        x = torch.randn(B, 3, 64, 64, generator=g).to(dev)
        target = torch.randint(0, K, (B, 64, 64), generator=g)
        target[torch.rand(target.shape, generator=g) < 0.1] = 255
        target = target.to(dev)
        model.train(True)
        losses = []
        for step in range(3):
            for group in optimizer.param_groups:
                group["lr"] = 1e-3 * group["lr_scale"]
            with torch.autocast("cuda", dtype=torch.float16):
                loss = criterion(model({"rgb": x})["semseg"], target)
            losses.append(loss.item())
            assert math.isfinite(losses[-1])
            optimizer.zero_grad()
            grad_norm = loss_scaler(loss, optimizer, clip_grad=None, parameters=model.parameters(), create_graph=False,
                                    update_grad=True)
            torch.cuda.synchronize()
            assert model.module.grad_arena().owned and math.isfinite(float(grad_norm))
        print("losses", losses)
        assert losses[2] < losses[0]
    finally:
        mm.AUTO_OWN_GRADIENTS = old
