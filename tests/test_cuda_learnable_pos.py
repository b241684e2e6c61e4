"""GPU: trainable position tables of the input adapters (learnable_pos_emb=True / sincos_pos_emb=False).

1. The recorded reference steps (tests/golden/make_golden_learnable_pos.py): outputs and every pos_emb gradient.
2. The resize kernels against F.interpolate and its autograd in float64, both modes, up / down / identity / non-square.
3. Masking (a patch masked in every sample gets a zero gradient) and bitwise-repeatable table gradients.
4. A TrainStep-captured step replays the optimizer's latest table values; run_finetuning_semseg.py's train_one_epoch body
   with --learnable_pos_emb over the overlay classes trains the table."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from helpers import formula_fill_, load_fixture, rel_l2
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn

pytestmark = pytest.mark.gpu

TOL = 1e-2            # bf16 tensor-core path against the fp32 reference, relative L2: outputs
GRAD_TOL = 3e-2       # and gradients (as test_cuda_parity)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def fx(golden_dir):
    return load_fixture(golden_dir, "learnable_pos.pt")


def _mae_model(c, tables, dev):
    from test_host_api import _build
    model = _build(tuple(c["in_domains"]), c["dim"], c["depth"], c["heads"], c["dec_dim"], c["dec_depth"], c["dec_heads"],
                   c["image_size"])
    formula_fill_(list(model.named_parameters()))
    with torch.no_grad():
        for k, v in tables.items():
            model.get_parameter(k).copy_(v)
    for ad in model.input_adapters.values():
        ad.pos_emb.requires_grad_(True)
    return model.to(dev).train()


def _losses(preds, x, masks):
    from test_cuda_parity import _loss_modules
    fns = _loss_modules()
    return {t: fns[t](preds[t].float(), x["rgb" if t == "norm_rgb" else t], mask=masks.get("rgb" if t == "norm_rgb" else t))
            for t in preds}


def test_masked_multimae_against_reference(fx, dev):
    m = fx["mae"]
    model = _mae_model(m["config"], m["tables"], dev)
    x = {k: v.to(dev) for k, v in m["inputs"].items()}
    preds, masks = model(x, task_masks={k: v.to(dev) for k, v in m["task_masks"].items()})
    losses = _losses(preds, x, masks)
    sum(losses.values()).backward()
    torch.cuda.synchronize()
    for k, ref in m["preds"].items():
        assert rel_l2(preds[k], ref) < TOL, (k, rel_l2(preds[k], ref))
    for k, ref in m["losses"].items():
        assert abs(float(losses[k]) - float(ref)) <= TOL * abs(float(ref)), (k, float(losses[k]), float(ref))
    # The encoder-input gradient of this step is ~1e-4 against a global gradient norm of 15: at that scale the bf16 path's
    # rounding dominates every embedding gradient, the existing proj.bias ones included.  Each table gradient must be as
    # accurate as its adapter's proj.bias gradient (made from the same dx), and at the tables' own grid the patch sums of
    # the table gradient ARE that bias gradient, which holds to fp32 summation order.
    for k, ref in m["pos_grads"].items():
        d = k.split(".")[1]
        got = model.get_parameter(k).grad
        bias = model.input_adapters[d].proj.bias.grad
        bias_ref = m["grads"]["input_adapters.%s.proj.bias" % d]
        assert bias_ref["step"] == 1 and bias_ref["samples"].numel() == bias.numel()
        bias_err = rel_l2(bias, bias_ref["samples"])
        print(k, rel_l2(got, ref), "proj.bias", bias_err)
        assert rel_l2(got, ref) < max(TOL, 1.5 * bias_err), (k, rel_l2(got, ref), bias_err)
        assert rel_l2(got.flatten(2)[0].sum(1), bias) < 1e-5, k
        # the patches masked in both samples: exactly zero (the tables are at the input's grid)
        always = m["task_masks"][d].bool().all(0)
        assert bool((got.flatten(2)[0][:, always.to(dev)] == 0).all()), k


def test_multivit_resized_tables_against_reference(fx, dev):
    from functools import partial

    from multimae_b200.input_adapters import PatchedInputAdapter, SemSegInputAdapter
    from multimae_b200.multimae import MultiViT
    v = fx["vit"]
    c = v["config"]
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=c["table_size"],
                                      sincos_pos_emb=False),
           "semseg": SemSegInputAdapter(num_classes=133, dim_class_emb=64, stride_level=4, patch_size_full=16,
                                        image_size=c["table_size"], learnable_pos_emb=True)}
    model = MultiViT(ins, None, num_global_tokens=1, dim_tokens=c["dim"], depth=c["depth"], num_heads=c["heads"],
                     mlp_ratio=4, qkv_bias=True, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6))
    formula_fill_(list(model.named_parameters()))
    with torch.no_grad():
        for k, t in v["tables"].items():
            model.get_parameter(k).copy_(t)
    model = model.to(dev).train()
    seq, _ = model.process_input({k: t.to(dev) for k, t in v["inputs"].items()})     # MultiViT.forward, split open
    seq.retain_grad()
    tokens = Fn.block_stack(model.encoder, seq)
    loss = (tokens * v["weights"].to(dev)).sum()
    loss.backward()
    torch.cuda.synchronize()
    assert rel_l2(tokens, v["tokens"]) < TOL
    # a weighted sum with random signs: bound its error by the sum of the magnitudes of its terms
    assert abs(float(loss) - float(v["loss"])) <= TOL * float((v["tokens"] * v["weights"]).abs().sum())
    n = 5 * 6
    for i, (d, mode) in enumerate((("rgb", "bicubic"), ("semseg", "bilinear"))):
        k = "input_adapters.%s.pos_emb" % d
        got = model.get_parameter(k).grad
        # against the reference step: the bf16 path's gradient tolerance (test_cuda_parity.GRAD_TOL)
        print(k, rel_l2(got, v["pos_grads"][k]))
        assert rel_l2(got, v["pos_grads"][k]) < GRAD_TOL, (k, rel_l2(got, v["pos_grads"][k]))
        # against F.interpolate's autograd in float64 on this path's own encoder-input gradient: the kernels exactly
        t64 = v["tables"][k].double().requires_grad_(True)
        F.interpolate(t64, size=(5, 6), mode=mode, align_corners=False).flatten(2).transpose(1, 2)[0].backward(
            seq.grad[:, i * n:(i + 1) * n].sum(0).double().cpu())
        assert rel_l2(got, t64.grad) < 1e-5, (k, rel_l2(got, t64.grad))


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["bicubic", "bilinear"])
@pytest.mark.parametrize("src,dst", [((14, 14), (32, 32)), ((32, 32), (14, 14)), ((14, 14), (14, 14)), ((12, 16), (7, 9))])
def test_resample_forward_and_adjoint_against_interpolate(dev, mode, src, dst):
    lib = L.lib()
    D = 96
    g = torch.Generator(device="cpu").manual_seed(3)
    table = torch.randn(1, D, *src, generator=g, dtype=torch.float64)
    drows = torch.randn(dst[0] * dst[1], D, generator=g, dtype=torch.float64)
    t64 = table.clone().requires_grad_(True)
    ref = F.interpolate(t64, size=dst, mode=mode, align_corners=False).flatten(2).transpose(1, 2)[0]
    ref.backward(drows)
    t32 = table.float().to(dev).contiguous()
    rows = torch.empty(dst[0] * dst[1], D, device=dev)
    L.check(lib.mmae_pos_resample_forward(t32.data_ptr(), D, src[0], src[1], dst[0], dst[1], L.POS_MODES[mode],
                                          rows.data_ptr(), L.current_stream()), "forward")
    dtable = torch.full_like(t32, 0.25)                                        # accumulated onto: += adjoint
    L.check(lib.mmae_pos_resample_backward(drows.float().to(dev).data_ptr(), D, src[0], src[1], dst[0], dst[1],
                                           L.POS_MODES[mode], dtable.data_ptr(), L.current_stream()), "backward")
    torch.cuda.synchronize()
    torch.testing.assert_close(rows.double().cpu(), ref.detach(), rtol=1e-5, atol=1e-5 * float(ref.abs().max()))
    adj = t64.grad + 0.25
    torch.testing.assert_close(dtable.double().cpu(), adj, rtol=1e-5, atol=1e-5 * float(adj.abs().max()))
    if src == dst:                                                              # the identity: a transpose, exactly
        assert torch.equal(rows.cpu(), t32.cpu().flatten(2).transpose(1, 2)[0])


def test_masked_patch_zero_and_bitwise_repeatable(dev):
    """Row gradients from a hand-made dx / ids_restore: a patch masked in every sample gets exactly 0, the others the sum
    of their visible tokens' gradients; two identical calls give bitwise-equal table gradients."""
    lib = L.lib()
    from multimae_b200.multimae import _build_layout
    from multimae_b200.input_adapters import PatchedInputAdapter
    ads = [("rgb", PatchedInputAdapter(3, 1, 16, dim_tokens=128, image_size=64, learnable_pos_emb=True)),
           ("depth", PatchedInputAdapter(1, 1, 16, dim_tokens=128, image_size=64, learnable_pos_emb=True))]
    B, G, D, total, T = 3, 1, 128, 32, 9
    layout = _build_layout(ads, {"rgb": torch.zeros(B, 3, 64, 64), "depth": torch.zeros(B, 1, 64, 64)})
    g = torch.Generator().manual_seed(5)
    shuffle = torch.stack([torch.randperm(total, generator=g) for _ in range(B)])
    never = [0, 5, 17]                                                          # masked in every sample
    for b in range(B):
        rest = [int(i) for i in shuffle[b] if int(i) not in never]
        shuffle[b] = torch.tensor(rest + never)
    ids_restore = torch.argsort(shuffle, dim=1).to(dev)
    dx = torch.randn(B, T + G, D, generator=g).to(dev)
    rows = [torch.empty(16, D, device=dev) for _ in range(2)]

    def run():
        arr = (ctypes.c_void_p * 2)(*[r.data_ptr() for r in rows])
        L.check(lib.mmae_embed_pos_backward(ctypes.byref(layout), ids_restore.data_ptr(), B, T, G, D, dx.data_ptr(), arr,
                                            L.current_stream()), "rows")
        out = []
        for r in rows:
            tb = torch.zeros(1, D, 4, 4, device=dev)
            L.check(lib.mmae_pos_resample_backward(r.data_ptr(), D, 4, 4, 4, 4, 0, tb.data_ptr(), L.current_stream()), "adj")
            out.append(tb)
        torch.cuda.synchronize()
        return [r.clone() for r in rows], out

    rows1, tabs1 = run()
    rows2, tabs2 = run()
    assert all(torch.equal(a, b) for a, b in zip(rows1 + tabs1, rows2 + tabs2))
    full = torch.cat(rows1).cpu()
    ref = torch.zeros(total, D)
    for b in range(B):
        for gi in range(total):
            s = int(ids_restore[b, gi])
            if s < T:
                ref[gi] += dx[b, s].cpu()
    torch.testing.assert_close(full, ref, rtol=1e-6, atol=1e-6)
    assert all(bool((full[i] == 0).all()) for i in never)
    assert torch.equal(tabs1[1].flatten(2)[0].t(), rows1[1])                   # identity adjoint: the transposed rows


def test_model_backward_bitwise_repeatable(fx, dev):
    m = fx["mae"]
    model = _mae_model(m["config"], m["tables"], dev)
    x = {k: v.to(dev) for k, v in m["inputs"].items()}
    tm = {k: v.to(dev) for k, v in m["task_masks"].items()}
    grads = []
    for _ in range(2):
        for p in model.parameters():
            p.grad = None
        preds, masks = model(x, task_masks=tm)
        sum(_losses(preds, x, masks).values()).backward()
        torch.cuda.synchronize()
        grads.append({d: ad.pos_emb.grad.clone() for d, ad in model.input_adapters.items()})
    assert all(torch.equal(grads[0][d], grads[1][d]) for d in grads[0])


def test_cuda_graph_replay_reads_updated_table(fx, dev):
    """TrainStep.capture with trainable tables: 1 eager warm-up + 3 replays equal 4 eager steps (the optimizer moves the
    tables every step); a table written in place between replays changes the next replay's loss."""
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep
    from test_cuda_parity import _loss_modules
    m = fx["mae"]

    def make():
        model = _mae_model(m["config"], m["tables"], dev)
        tm = {k: v.to(dev) for k, v in m["task_masks"].items()}
        triple = (tm, m["ids_keep"].to(dev), m["ids_restore"].to(dev))
        model.generate_random_masks = lambda *a, **k: triple
        opt = FlatAdamW(model, lr=1e-2)
        scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
        step = TrainStep(model, _loss_modules(), opt, scaler, num_encoded_tokens=m["config"]["n_visible"],
                         loss_sources={"norm_rgb": "rgb"})
        return model, step

    x = {k: v.to(dev) for k, v in m["inputs"].items()}

    def run(use_graph):
        model, step = make()
        start = model.input_adapters["rgb"].pos_emb.detach().clone()
        if use_graph:
            step.capture(x, warmup=1)
            assert step.graph is not None
        else:
            step(x)
        losses = [float(step(x)[0]) for _ in range(3)]
        torch.cuda.synchronize()
        tables = torch.cat([ad.pos_emb.detach().flatten() for ad in model.input_adapters.values()])
        assert not torch.equal(model.input_adapters["rgb"].pos_emb.detach(), start)
        return losses, tables, model, step

    l_eager, t_eager, _, _ = run(False)
    l_graph, t_graph, model, step = run(True)
    assert all(abs(a - b) <= 2e-3 * abs(a) for a, b in zip(l_eager, l_graph)), (l_eager, l_graph)
    assert rel_l2(t_graph, t_eager) < 1e-3
    before = float(step(x)[0])
    with torch.no_grad():
        for ad in model.input_adapters.values():
            ad.pos_emb.add_(torch.randn_like(ad.pos_emb))
    after = float(step(x)[0])
    assert math.isfinite(after) and abs(after - before) > 0.05 * abs(before), (before, after)


def test_finetune_semseg_sequence_trains_the_table(dev):
    """run_finetuning_semseg.py's train_one_epoch body with --learnable_pos_emb over the overlay classes, the REAL library:
    autocast, CrossEntropyLoss(ignore_index=255), NativeScalerWithGradNormCount with loss scaling, stock AdamW, arena-owned
    gradients.  The rgb table (3 x 3, resized bicubic to the 4 x 4 grid) receives a finite non-zero gradient and moves."""
    from functools import partial

    from multimae_b200 import multimae as mm
    from multimae_b200 import overlay
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.output_adapters import ConvNeXtAdapter
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True
    try:
        torch.manual_seed(0)
        K, B = 5, 4
        ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=48,
                                          learnable_pos_emb=True)}
        outs = {"semseg": ConvNeXtAdapter(K, embed_dim=2048, preds_per_patch=16, depth=2)}
        net = MultiViT(ins, outs, num_global_tokens=1, dim_tokens=128, depth=2, num_heads=2, mlp_ratio=4, qkv_bias=True,
                       drop_path_rate=0.1, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6)).to(dev)
        model = overlay._IdentityDDP(net, device_ids=[0])
        optimizer = torch.optim.AdamW([p for p in net.parameters() if p.requires_grad], lr=1e-3, weight_decay=0.05)
        loss_scaler = NativeScalerWithGradNormCount()
        criterion = torch.nn.CrossEntropyLoss(ignore_index=255)
        g = torch.Generator().manual_seed(7)
        x = torch.randn(B, 3, 64, 64, generator=g).to(dev)
        target = torch.randint(0, K, (B, 64, 64), generator=g).to(dev)
        table = net.input_adapters["rgb"].pos_emb
        start = table.detach().clone()
        model.train(True)
        for _ in range(2):
            with torch.autocast("cuda", dtype=torch.float16):
                loss = criterion(model({"rgb": x})["semseg"], target)
            assert math.isfinite(loss.item())
            optimizer.zero_grad()
            grad_norm = loss_scaler(loss, optimizer, clip_grad=None, parameters=model.parameters(), create_graph=False,
                                    update_grad=True)
            torch.cuda.synchronize()
            assert math.isfinite(float(grad_norm))
            assert table.grad is not None and table.grad.data_ptr() == net.grad_arena().views["input_adapters.rgb.pos_emb"].data_ptr()
            assert torch.isfinite(table.grad).all() and float(table.grad.abs().sum()) > 0
        assert not torch.equal(table.detach(), start)
    finally:
        mm.AUTO_OWN_GRADIENTS = old
