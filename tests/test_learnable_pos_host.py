"""CPU: trainable position tables of the input adapters (learnable_pos_emb=True / sincos_pos_emb=False) without a GPU.

1. The oracle with trainable tables reproduces the reference's outputs, losses and gradients recorded by
   tests/golden/make_golden_learnable_pos.py (a masked MultiMAE step at the tables' own grid, a MultiViT step on a larger
   grid: bicubic and bilinear resizes).
2. The host layer against a stub of the C library: the tables are in the gradient arena and reported with the adapter's
   other gradients, the new entry points get well-formed arguments, frozen tables make the calls they always made.
3. run_finetuning_semseg.py's model set-up with --learnable_pos_emb through the overlay, with a 14 x 14 table resized
   into the 32 x 32 one as interpolate_pos_embed_multimae does.
4. Data parallelism over gloo (2 ranks): the table gradients are all-reduced with the rest of the arena."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from helpers import formula_fill_, load_fixture
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from oracle import multimae_oracle as O
from test_drop_path_host import _Rec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_CALLS = ("mmae_pos_resample_forward", "mmae_embed_pos_backward", "mmae_pos_resample_backward")


@pytest.fixture(scope="module")
def fx(golden_dir):
    return load_fixture(golden_dir, "learnable_pos.pt")


def oracle_params(c, tables, out_domains):
    """Formula-filled oracle parameters (as the recording's model) with the recorded tables, every entry trainable."""
    cfg = O.make_config(in_domains=tuple(c["in_domains"]), out_domains=out_domains, extra_norm_pix=bool(out_domains))
    cfg.dim, cfg.depth, cfg.heads = c["dim"], c["depth"], c["heads"]
    if out_domains:
        cfg.dec_dim, cfg.dec_depth, cfg.dec_heads = c["dec_dim"], c["dec_depth"], c["dec_heads"]
        cfg.posemb_grid = c["image_size"] // 16
    p = O.init_params(cfg)
    formula_fill_(list(O.trainable(p).items()))
    for k, v in tables.items():
        p[k] = v.clone()
    trained = {k: v for k, v in p.items() if k.startswith("input_adapters.") or k in O.trainable(p)}
    for v in trained.values():
        v.requires_grad_(True)
    return cfg, p, trained


def check_grads(trained, fx_pos, fx_rest):
    for k, ref in fx_pos.items():
        torch.testing.assert_close(trained[k].grad, ref, rtol=2e-4, atol=1e-7, msg=lambda m, k=k: "%s: %s" % (k, m))
    for k, d in fx_rest.items():
        g = trained[k].grad.flatten()
        torch.testing.assert_close(g.norm(), d["norm"], rtol=2e-4, atol=1e-7, msg=lambda m, k=k: "%s norm: %s" % (k, m))
        torch.testing.assert_close(g[::d["step"]][:d["samples"].numel()], d["samples"], rtol=1e-3, atol=2e-5,
                                   msg=lambda m, k=k: "%s samples: %s" % (k, m))


def test_oracle_masked_multimae_against_reference(fx):
    m = fx["mae"]
    c = m["config"]
    cfg, p, trained = oracle_params(c, m["tables"], c["in_domains"])
    losses, preds = O.step_losses(p, m["inputs"], cfg, m["task_masks"], m["ids_keep"], m["ids_restore"])
    for k, ref in m["preds"].items():
        torch.testing.assert_close(preds[k], ref, rtol=2e-4, atol=2e-5)
    for k, ref in m["losses"].items():
        torch.testing.assert_close(losses[k], ref, rtol=1e-5, atol=1e-6)
    sum(losses.values()).backward()
    assert set(m["pos_grads"]) == {"input_adapters.%s.pos_emb" % d for d in c["in_domains"]}
    check_grads(trained, m["pos_grads"], m["grads"])


def test_fixture_masks_patches_in_every_sample(fx):
    """At the tables' own grid row p of the table is patch p: a patch masked in both samples has an exactly zero gradient,
    and the fixture has such patches in every task (and visible ones)."""
    m = fx["mae"]
    for d, mask in m["task_masks"].items():
        g = m["pos_grads"]["input_adapters.%s.pos_emb" % d].flatten(2)[0]         # [D, 16]
        always = mask.bool().all(0)
        assert 0 < int(always.sum()) < always.numel(), d
        assert bool((g[:, always] == 0).all()) and bool((g[:, ~always].abs().sum(0) > 0).all()), d


def test_oracle_multivit_resize_against_reference(fx):
    v = fx["vit"]
    c = v["config"]
    cfg, p, trained = oracle_params(c, v["tables"], [])
    assert tuple(v["tables"]["input_adapters.rgb.pos_emb"].shape[2:]) == (3, 4)
    B, _, H, W = v["inputs"]["rgb"].shape
    total = (H // 16) * (W // 16) * len(c["in_domains"])                    # nothing masked: 2 x 5 x 6 tokens
    ids = torch.arange(total).unsqueeze(0).expand(B, -1)
    _, tokens = O.forward(p, v["inputs"], cfg, ids, ids)
    torch.testing.assert_close(tokens, v["tokens"], rtol=2e-4, atol=2e-5)
    loss = (tokens * v["weights"]).sum()
    torch.testing.assert_close(loss, v["loss"], rtol=1e-5, atol=1e-4)
    loss.backward()
    check_grads(trained, v["pos_grads"], v["grads"])


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(L, "lib", lambda: r)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    return r


def _model(trainable=("rgb", "depth", "semseg")):
    from test_host_api import _build
    model = _build(in_domains=("rgb", "depth", "semseg"), image_size=64).train()
    for d in trainable:
        model.input_adapters[d].pos_emb.requires_grad_(True)
    return model


def _step(model, size=64, B=2, num_encoded=10):
    x = {"rgb": torch.randn(B, 3, size, size), "depth": torch.randn(B, 1, size, size),
         "semseg": torch.randint(0, 133, (B, size // 4, size // 4))}
    preds, _ = model(x, num_encoded_tokens=num_encoded)
    sum(v.sum() for v in preds.values()).backward()


def _struct(arg):
    return arg._obj if hasattr(arg, "_obj") else arg


@pytest.mark.parametrize("trainable", [("rgb", "depth", "semseg"), ("semseg",)])
def test_tables_in_arena_and_reported_with_the_embedding(rec, trainable):
    model = _model(trainable)
    seen = []
    model.set_grad_callback(lambda names: seen.append(list(names)))
    _step(model, size=96)                                                  # 6 x 6 patches against 4 x 4 tables
    arena = model.grad_arena()
    embed = [names for names in seen if any(n.endswith("proj.weight") and n.startswith("input_adapters") for n in names)]
    assert len(embed) == 1
    for d in ("rgb", "depth", "semseg"):
        name = "input_adapters.%s.pos_emb" % d
        assert (name in arena.views) == (d in trainable)
        assert (name in embed[0]) == (d in trainable)
    reported = [n for names in seen for n in names]
    assert sorted(reported) == sorted(n for n, p in model.named_parameters() if p.requires_grad)
    for d in trainable:
        p = model.input_adapters[d].pos_emb
        assert p.grad is not None and torch.equal(p.grad, arena.views["input_adapters.%s.pos_emb" % d])


def test_entry_point_arguments(rec):
    model = _model(("rgb", "semseg"))
    _step(model, size=96, num_encoded=12)
    names = rec.names()
    i_fwd, i_emb = names.index("mmae_pos_resample_forward"), names.index("mmae_embed_forward")
    assert names.count("mmae_pos_resample_forward") == 2 and i_fwd < i_emb
    fwd = [a for n, a in rec.calls if n == "mmae_pos_resample_forward"]
    (emb,) = [a for n, a in rec.calls if n == "mmae_embed_forward"]
    prm = _struct(emb[2])
    cached = model.input_adapters["depth"]._resized_pos(6, 6, "bicubic")
    assert prm.pos[1] == cached.data_ptr()                                  # the frozen table: its cached rows
    for a, (t, d, mode) in zip(fwd, ((0, "rgb", 0), (2, "semseg", 1))):
        tb = model.input_adapters[d].pos_emb
        assert a[0] == tb.data_ptr() and list(a[1:7]) == [128, 4, 4, 6, 6, mode], (d, a)
        assert a[7] == prm.pos[t]                                           # the rows the embedding reads
    # backward: the row gradients in one call (NULL for the frozen depth table), then one adjoint per table into the arena
    (eb,) = [a for n, a in rec.calls if n == "mmae_embed_backward"]
    (pb,) = [a for n, a in rec.calls if n == "mmae_embed_pos_backward"]
    bwd = [a for n, a in rec.calls if n == "mmae_pos_resample_backward"]
    assert names.index("mmae_embed_backward") < names.index("mmae_embed_pos_backward") < names.index("mmae_pos_resample_backward")
    B, T, G, D = 2, 12, 1, 128
    assert list(pb[2:6]) == [B, T, G, D] and pb[6] == eb[9] and _struct(pb[0]).num_tasks == 3
    rows = list(pb[7])
    assert rows[1] is None and rows[0] and rows[2] and len(rows) == 3
    arena = model.grad_arena()
    for a, (t, d, mode) in zip(bwd, ((0, "rgb", 0), (2, "semseg", 1))):
        assert a[0] == rows[t] and list(a[1:7]) == [128, 4, 4, 6, 6, mode]
        assert a[7] == arena.views["input_adapters.%s.pos_emb" % d].data_ptr()


def test_identity_grid_and_direct_adapter_call(rec):
    from multimae_b200.input_adapters import SemSegInputAdapter
    ad = SemSegInputAdapter(num_classes=5, stride_level=4, patch_size_full=16, dim_tokens=128, image_size=64,
                            learnable_pos_emb=True)
    out = ad(torch.randint(0, 5, (2, 16, 16)))
    out.sum().backward()
    (f,) = [a for n, a in rec.calls if n == "mmae_pos_resample_forward"]
    (b,) = [a for n, a in rec.calls if n == "mmae_pos_resample_backward"]
    assert list(f[1:7]) == [128, 4, 4, 4, 4, 1] and list(b[1:7]) == [128, 4, 4, 4, 4, 1]
    assert f[0] == ad.pos_emb.data_ptr() and b[7] and ad.pos_emb.grad is not None    # the call's own arena slot
    (pb,) = [a for n, a in rec.calls if n == "mmae_embed_pos_backward"]
    assert list(pb[2:6]) == [2, 16, 0, 128]


def test_frozen_tables_make_the_plain_calls(rec):
    """Frozen tables: none of the new entry points, and the call sequence is the trainable one without them."""
    torch.manual_seed(0)
    _step(_model(()))
    frozen = rec.names()
    assert not any(n in NEW_CALLS for n in frozen)
    rec.calls.clear()
    torch.manual_seed(0)
    _step(_model())
    trainable = rec.names()
    assert sum(n in NEW_CALLS for n in trainable) == 3 + 1 + 3
    assert [n for n in trainable if n not in NEW_CALLS] == frozen


def test_output_adapter_table_and_class_emb_interpolation_still_refused():
    from multimae_b200.input_adapters import SemSegInputAdapter
    from multimae_b200.output_adapters import SpatialOutputAdapter
    ad = SpatialOutputAdapter(num_channels=3, stride_level=1, patch_size_full=16, dim_tokens=128, task="rgb",
                              context_tasks=["rgb"], learnable_pos_emb=True, image_size=64)
    ad.init(dim_tokens_enc=128)
    info = {"image_size": (64, 64), "num_task_tokens": 16, "num_global_tokens": 1,
            "tasks": {"rgb": {"num_tokens": 16, "start_idx": 0, "end_idx": 16}}}
    ids = torch.arange(16).unsqueeze(0)
    with pytest.raises(NotImplementedError, match="learnable_pos_emb"):
        ad(torch.zeros(1, 5, 128), info, ids[:, :4], ids)
    with pytest.raises(NotImplementedError, match="interpolate_class_emb"):
        SemSegInputAdapter(num_classes=5, stride_level=4, patch_size_full=16, interpolate_class_emb=True)


def test_semseg_script_model_setup_learnable_pos_emb():
    """run_finetuning_semseg.py:374-407 and :428 with --learnable_pos_emb and the ADE config (512 x 512 input, patch 16)
    through the overlay: the rgb table is a trainable 32 x 32 parameter, a pre-trained 14 x 14 table is resized into it
    (F.interpolate(..., (32, 32), mode='bicubic', align_corners=False), what interpolate_pos_embed_multimae does,
    utils/pos_embed.py:44-58) and loaded, and one training step against the stub library resizes it on the device
    (identity: 32 x 32 -> 32 x 32) and writes its gradient into the arena."""
    code = r'''
import sys, types
from functools import partial
import torch
import torch.nn.functional as F
sys.path.insert(0, %r)
sys.path.insert(0, %r)
from multimae_b200 import overlay
overlay.install()
from multimae.input_adapters import PatchedInputAdapter
from multimae.output_adapters import ConvNeXtAdapter
from multimae import multimae as mm
from multimae_b200 import _lib as L, functional as Fn
from test_drop_path_host import _Rec
args = types.SimpleNamespace(in_domains=["rgb"], patch_size=16, input_size=512, learnable_pos_emb=True, model="multivit_base",
                             decoder_depth=4, decoder_preds_per_patch=16, decoder_main_tasks="rgb", num_classes_with_void=151,
                             decoder_dim=6144, drop_path_encoder=0.1)
input_adapters = {d: PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=args.patch_size,
                                         image_size=args.input_size, learnable_pos_emb=args.learnable_pos_emb)
                  for d in args.in_domains}
output_adapters = {"semseg": ConvNeXtAdapter(num_classes=args.num_classes_with_void, embed_dim=args.decoder_dim,
                                             patch_size=args.patch_size, preds_per_patch=args.decoder_preds_per_patch,
                                             depth=args.decoder_depth, interpolate_mode="bilinear",
                                             main_tasks=args.decoder_main_tasks.split("-"))}
model = mm.__dict__[args.model](input_adapters=input_adapters, output_adapters=output_adapters,
                                drop_path_rate=args.drop_path_encoder)
table = model.input_adapters.rgb.pos_emb
assert table.requires_grad and tuple(table.shape) == (1, 768, 32, 32)
ckpt = {"input_adapters.rgb.pos_emb": torch.randn(1, 768, 14, 14)}
key = "input_adapters.rgb.pos_emb"
ckpt[key] = F.interpolate(ckpt[key], size=(32, 32), mode="bicubic", align_corners=False)
msg = model.load_state_dict(ckpt, strict=False)
assert key not in msg.missing_keys and torch.equal(model.input_adapters.rgb.pos_emb.detach(), ckpt[key])
assert model.input_adapters.rgb.pos_emb.requires_grad and "input_adapters.rgb.pos_emb" in model.no_weight_decay()
rec = _Rec()
L.lib = lambda: rec
L.current_stream = lambda: 0
Fn._require_cuda = lambda t, what: None
model.train()
out = model({"rgb": torch.zeros(1, 3, 512, 512)})
out["semseg"].sum().backward()
f = [a for n, a in rec.calls if n == "mmae_pos_resample_forward"]
b = [a for n, a in rec.calls if n == "mmae_pos_resample_backward"]
assert len(f) == 1 and f[0][0] == table.data_ptr() and list(f[0][1:7]) == [768, 32, 32, 32, 32, 0], f
assert len(b) == 1 and b[0][7] == table.grad.data_ptr() == model.grad_arena().views[key].data_ptr(), b
print("ok")
''' % (ROOT, os.path.join(ROOT, "tests"))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout + res.stderr


# ---------------------------------------------------------------------------------------------------------------------
def _dp_worker(rank, world, port, out):
    """The overlay's multi-rank path (see test_parallel_gloo._overlay_worker) with trainable tables: each rank's backward
    writes rank + 1 into every gradient it reports; after the scaler's exchange the tables hold the sum over ranks."""
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from multimae_b200 import overlay
    from multimae_b200.criterion import MaskedMSELoss
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from test_host_api import _build
    rec = _Rec()
    L.lib = lambda: rec
    L.current_stream = lambda: 0
    Fn._require_cuda = lambda t, what: None
    Fn.grad_unscale_norm = lambda flat, inv_scale=1.0, post_scale=1.0, inv_scale_tensor=None: (torch.ones(()), torch.zeros(2))
    torch.manual_seed(rank)
    model = _build(in_domains=("rgb", "depth")).train()
    for ad in model.input_adapters.values():
        ad.pos_emb.requires_grad_(True)
    wrapped = overlay._IdentityDDP(model, device_ids=[0], find_unused_parameters=True)
    reducer, arena = model._mmae_reducer, model.grad_arena()
    assert any("input_adapters.rgb.pos_emb" in b[2] for b in reducer.buckets)
    ready = reducer.on_grads_ready

    def fill_then_report(names):
        for n in names:
            arena.view(n).fill_(float(rank + 1))
        ready(names)
    model.set_grad_callback(fill_then_report)
    optimizer = torch.optim.AdamW(model.parameters(), lr=0.0)
    scaler = NativeScalerWithGradNormCount(enabled=True)
    x = {"rgb": torch.randn(2, 3, 64, 64), "depth": torch.randn(2, 1, 64, 64)}
    preds, masks = wrapped(x, num_encoded_tokens=6)
    loss = sum(MaskedMSELoss(16, 1)(preds[k], x["rgb"], mask=masks["rgb"]) for k in preds)
    optimizer.zero_grad()
    scaler(loss, optimizer, clip_grad=None, skip_grad=None, parameters=wrapped.parameters())
    total = float(sum(r + 1 for r in range(world)))
    for d in ("rgb", "depth"):
        p = model.input_adapters[d].pos_emb
        assert p.grad is not None and p.grad.data_ptr() == arena.view("input_adapters.%s.pos_emb" % d).data_ptr()
        assert torch.all(p.grad == total), d
    out.put((rank, "ok"))
    dist.destroy_process_group()


def test_data_parallel_all_reduces_table_gradients():
    import torch.multiprocessing as mp
    from test_parallel_gloo import _free_port
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    assert sorted(out.get(timeout=5) for _ in range(2)) == [(0, "ok"), (1, "ok")]
