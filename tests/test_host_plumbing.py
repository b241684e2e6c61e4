"""CPU: exercise the Python host layer end to end (autograd Functions, struct marshalling, gradient arena, scaler,
flat optimizer bookkeeping) against a STUB of the C library that validates every call's argument count / ctypes
convertibility and returns success without computing.  Numerical results are meaningless here; what is checked is
the plumbing the GPU tests rely on."""
import ctypes

import pytest
import torch

from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from test_host_api import _build


class _StubLib:
    def __init__(self):
        self.calls = []        # names, in call order
        self.log = []          # (name, args) of every call

    def args_of(self, name):
        return [a for n, a in self.log if n == name]

    def __getattr__(self, name):
        if name not in L.SIGNATURES:
            raise AttributeError(name)
        res, argtypes = L.SIGNATURES[name]

        def fn(*args):
            assert len(args) == len(argtypes), "%s: %d args for %d parameters" % (name, len(args), len(argtypes))
            for a, t in zip(args, argtypes):
                if isinstance(a, type(ctypes.byref(ctypes.c_int()))):
                    continue
                t.from_param(a)        # raises on a type the real ctypes call would reject
            self.calls.append(name)
            self.log.append((name, args))
            if name.endswith("_bytes"):
                return 4096
            if name == "mmae_abi_version":
                return L.ABI_VERSION
            if name == "mmae_last_error":
                return b""
            return 0
        return fn


@pytest.fixture()
def stub(monkeypatch):
    s = _StubLib()
    monkeypatch.setattr(L, "lib", lambda: s)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    return s


def _inputs(B=2, size=64):
    return {"rgb": torch.randn(B, 3, size, size), "depth": torch.randn(B, 1, size, size),
            "semseg": torch.randint(0, 133, (B, size // 4, size // 4))}


@pytest.mark.parametrize("shared_ctx", [True, False])
def test_model_forward_backward_plumbing(stub, monkeypatch, shared_ctx):
    """shared_ctx: the four adapters' proj_context Linears as one GEMM (the default) or one per adapter (MMAE_SHARED_CTX=0)."""
    from multimae_b200 import multimae as MM
    from multimae_b200.criterion import MaskedCrossEntropyLoss, MaskedL1Loss, MaskedMSELoss
    monkeypatch.setattr(MM, "SHARED_CONTEXT_PROJECTION", shared_ctx)
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", shared_ctx)          # the same switch position also covers chained / single blocks
    model = _build().train()
    x = _inputs()
    preds, masks = model(x, num_encoded_tokens=12, alphas=1.0)
    assert set(preds) == {"rgb", "depth", "semseg", "norm_rgb"} and set(masks) == {"rgb", "depth", "semseg"}
    assert preds["rgb"].shape == (2, 3, 64, 64) and preds["semseg"].shape == (2, 133, 16, 16)
    assert masks["rgb"].shape == (2, 16) and masks["rgb"].dtype == torch.int64
    fns = {"rgb": MaskedMSELoss(16, 1), "depth": MaskedL1Loss(16, 1), "semseg": MaskedCrossEntropyLoss(16, 4),
           "norm_rgb": MaskedMSELoss(16, 1, norm_pix=True)}
    loss = sum(fns[k](preds[k].float(), x["rgb" if k == "norm_rgb" else k], mask=masks["rgb" if k == "norm_rgb" else k])
               for k in preds)
    loss.backward()
    arena = model.grad_arena()
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and p.grad.shape == p.shape, n
        else:
            assert p.grad is None, n
    # every module-level entry point was reached
    head_f, head_b = ("mmae_dechead_forward_ctx", "mmae_dechead_backward_ctx") if shared_ctx else \
        ("mmae_dechead_forward", "mmae_dechead_backward")
    for name in ("mmae_sample_masks", "mmae_embed_forward", "mmae_embed_backward", "mmae_block_forward",
                 "mmae_block_backward", head_f, head_b, "mmae_dectail_forward",
                 "mmae_dectail_backward", "mmae_masked_loss_forward", "mmae_masked_loss_backward"):
        assert name in stub.calls, name
    # the 2 encoder blocks run chained (one hand-off: x_add / y_out forward, dx_out_bf16 / dx_in_bf16 backward); the 4
    # one-block decoder transformers stay single blocks
    chained = 2 if shared_ctx else 0
    fwd, bwd = stub.args_of("mmae_block_forward"), stub.args_of("mmae_block_backward")
    assert len(fwd) == len(bwd) == 2 + 4 * 1 and stub.calls.count(head_b) == 4
    assert sum(a[1] is not None or a[4] is not None for a in fwd) == chained
    assert sum(a[2] is not None or a[4] is not None for a in bwd) == chained
    assert stub.calls.count("mmae_block_saved_x_mid") == chained // 2
    assert stub.calls.count("mmae_ctxproj_forward") == stub.calls.count("mmae_ctxproj_backward") == (1 if shared_ctx else 0)
    if shared_ctx:      # the shared projection's backward runs after the last head's, before the encoder's
        order = [c for c in stub.calls if c in (head_b, "mmae_ctxproj_backward", "mmae_block_backward")]
        i = order.index("mmae_ctxproj_backward")
        assert order[:i].count(head_b) == 4 and order[i + 1:].count(head_b) == 0
        # the proj_context tensors of the four adapters lie back to back in the arena (used in place as one matrix)
        offs = [arena.offsets["output_adapters.%s.proj_context.weight" % k] for k in preds]
        assert all(o1[0] + o1[1] == o2[0] for o1, o2 in zip(offs, offs[1:])), offs
    assert arena.numel >= sum(p.numel() for p in model.parameters() if p.requires_grad)


def test_owned_gradients_scaler_and_flat_optimizer(stub):
    from multimae_b200.criterion import MaskedMSELoss
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    model = _build(in_domains=("rgb",)).train()
    opt = FlatAdamW(model, lr=1e-3)
    arena = model.grad_arena()
    assert arena.owned and all(p.grad is not None and p.grad.data_ptr() == arena.views[n].data_ptr()
                               for n, p in model.named_parameters() if p.requires_grad)
    ready = []
    model.set_grad_callback(lambda names: ready.extend(names))
    scaler = NativeScalerWithGradNormCount(enabled=True).attach_arena(arena)
    x = {"rgb": torch.randn(2, 3, 64, 64)}
    preds, masks = model(x, num_encoded_tokens=4)
    loss = sum(MaskedMSELoss(16, 1)(preds[k], x["rgb"], mask=masks["rgb"]) for k in preds)
    opt.zero_grad()
    norm = scaler(loss, opt, parameters=model.parameters())
    assert norm is not None and "mmae_grad_unscale_norm" in stub.calls and "mmae_adamw_step" in stub.calls
    assert set(ready) == {n for n, p in model.named_parameters() if p.requires_grad}     # every gradient announced once
    assert len(ready) == len(set(ready))
    sd = scaler.state_dict()
    assert "scale" in sd and sd["scale"] > 0
    # parameters were re-homed into one flat buffer and still expose the reference state_dict schema
    assert all(p.data_ptr() >= opt.flat_params.data_ptr() for p in model.parameters() if p.requires_grad)


def test_fixed_masks_and_no_masking(stub):
    model = _build().train()
    x = _inputs(B=1)
    tm = {k: torch.ones(1, 16, dtype=torch.long) for k in ("rgb", "depth", "semseg")}
    tm["rgb"][0, :5] = 0
    tm["depth"][0, 3] = 0
    preds, masks = model(x, task_masks=tm)
    assert masks is tm and preds["rgb"].shape == (1, 3, 64, 64)
    preds, masks = model(x, mask_inputs=False)
    assert preds["depth"].shape == (1, 1, 64, 64)
    with pytest.raises(ValueError):
        model(_inputs(B=2), task_masks={k: torch.cat([v, torch.ones_like(v)]) for k, v in tm.items()})


def test_mask_token_queries_plumbing(stub):
    """Host side of the mask-token decoder queries (multimae/output_adapters.py:214-221): a context task that is not fed
    rides in the spare task-embedding slot, an output task that is no context task has no embedding, and
    use_task_queries=False keeps the task's own slot; gradients are announced under the reference's parameter names."""
    from multimae_b200.criterion import MaskedL1Loss
    seen = []
    real_apply = Fn.DecoderHeadFunction.apply

    def spy(enc, meta, *rest):
        seen.append((meta["prefix"], meta["query_mode"], meta["own_task"], list(meta["task_names"])))
        return real_apply(enc, meta, *rest)

    Fn.DecoderHeadFunction.apply = staticmethod(spy)
    try:
        # built for rgb+depth+semseg, fed rgb+semseg: 'depth' is decoded from mask-token queries + its own embedding
        model = _build().train()
        ready = []
        model.set_grad_callback(lambda names: ready.extend(names))
        x = _inputs()
        preds, masks = model({"rgb": x["rgb"], "semseg": x["semseg"]}, num_encoded_tokens=10)
        assert set(preds) == {"rgb", "depth", "semseg", "norm_rgb"} and set(masks) == {"rgb", "semseg"}
        by_prefix = {p: (mode, own, names) for p, mode, own, names in seen}
        assert by_prefix["output_adapters.depth."] == (1, 2, ["rgb", "semseg", "depth"])
        assert by_prefix["output_adapters.rgb."] == (0, 0, ["rgb", "semseg"])
        assert by_prefix["output_adapters.semseg."] == (0, 1, ["rgb", "semseg"])
        MaskedL1Loss(16, 1)(preds["depth"], x["depth"], mask=masks.get("depth")).backward()    # no mask: plain mean
        assert "output_adapters.depth.task_embeddings.depth" in ready
        assert "output_adapters.depth.mask_token" in ready
        assert not any(n.startswith("input_adapters.depth.") for n in ready)                   # never embedded
        # an output task that is no context task at all, and use_task_queries=False
        seen.clear()
        model = _build(in_domains=("rgb",), out_domains=("rgb", "depth"), use_task_queries=False).train()
        preds, masks = model({"rgb": x["rgb"]}, num_encoded_tokens=6)
        by_prefix = {p: (mode, own, names) for p, mode, own, names in seen}
        assert by_prefix["output_adapters.depth."] == (1, -1, ["rgb"])
        assert by_prefix["output_adapters.rgb."] == (1, 0, ["rgb"])
        assert preds["depth"].shape == (2, 1, 64, 64)
    finally:
        Fn.DecoderHeadFunction.apply = real_apply


def test_train_step_eager_and_sampling_options(stub):
    """TrainStep._step (the body of train_one_epoch between the H2D copy and the optimizer step) through the stub: depth
    standardisation first, `loss_sources` routing of norm_rgb, per-task alphas and uniform task sampling
    (multimae/multimae.py:148-162,182-187)."""
    from multimae_b200.criterion import MaskedCrossEntropyLoss, MaskedL1Loss, MaskedMSELoss
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep
    model = _build().train()
    opt = FlatAdamW(model, lr=1e-3)
    scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
    fns = {"rgb": MaskedMSELoss(16, 1), "depth": MaskedL1Loss(16, 1), "semseg": MaskedCrossEntropyLoss(16, 4),
           "norm_rgb": MaskedMSELoss(16, 1, norm_pix=True)}
    x = _inputs()
    step = TrainStep(model, fns, opt, scaler, num_encoded_tokens=12, alphas=[0.5, 1.0, 2.0], loss_sources={"norm_rgb": "rgb"},
                     standardize_depth=True)
    loss, norm = step(x, use_graph=False)
    assert loss.shape == () and norm is not None
    assert stub.calls.count("mmae_standardize_depth") == 1 and stub.calls.index("mmae_standardize_depth") < stub.calls.index("mmae_embed_forward")
    assert stub.calls.count("mmae_masked_loss_forward") == 4 and "mmae_adamw_step" in stub.calls
    assert x["depth"].shape == (2, 1, 64, 64)               # the caller's batch dict still holds its own depth tensor
    stub.calls.clear()
    uniform = TrainStep(model, fns, opt, scaler, num_encoded_tokens=12, sample_tasks_uniformly=True,
                        loss_sources={"norm_rgb": "rgb"})
    torch.manual_seed(0)
    uniform(x, use_graph=False)
    assert "mmae_sample_masks" in stub.calls and "mmae_standardize_depth" not in stub.calls
    a = model.sample_alphas(64, 3, alphas=[1.0, 1.0, 1.0])
    assert a.shape == (64, 3) and bool(((a > 0.5).sum(1) >= 1).all())      # never the all-zero task subset (:150)


def test_block_stack_hand_off_call_arguments(monkeypatch):
    """BlockFunction wires consecutive blocks through raw pointers: block i+1 must receive block i's x_mid (inside
    block i's `saved` buffer) as x_in and the shared MLP-output buffer as x_add; only the last block writes x_out; in backward
    block i+1 writes bf16(dx) into the buffer block i then reads, and its column sums into block i's fc2 bias gradient."""
    from multimae_b200.multimae_utils import Block
    calls = []

    class Rec:
        def __getattr__(self, name):
            res, argtypes = L.SIGNATURES[name]

            def fn(*args):
                assert len(args) == len(argtypes), name
                calls.append((name, args))
                if name.endswith("_bytes"):
                    return 4096
                if name == "mmae_block_saved_x_mid":
                    return args[0] + 64                     # "x_mid lives 64 bytes into the saved buffer"
                return 0
            return fn

    rec = Rec()
    monkeypatch.setattr(L, "lib", lambda: rec)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", True)
    blocks = torch.nn.Sequential(*[Block(128, 2, qkv_bias=True) for _ in range(4)])
    named = [(n, p) for n, p in blocks.named_parameters()]
    arena = Fn.GradArena(named, torch.device("cpu"))
    ready = []
    for i, b in enumerate(blocks):
        b.bind(arena, "%d." % i, lambda names: ready.append(list(names)))
    x = torch.randn(2, 5, 128, requires_grad=True)
    out = Fn.block_stack(blocks, x)
    fwd = [a for n, a in calls if n == "mmae_block_forward"]
    mids = [a for n, a in calls if n == "mmae_block_saved_x_mid"]
    assert len(fwd) == 4 and len(mids) == 3
    # args: x_in, x_add, x_sum, x_out, y_out, ..., saved (index 16)
    assert fwd[0][0] == x.data_ptr() and fwd[0][1] is None and fwd[0][2] is None        # first block: plain input
    y_buf = fwd[0][4]
    assert y_buf is not None and fwd[0][3] is None                                       # not the last: y_out, no x_out
    for i in (1, 2, 3):
        assert fwd[i][0] == fwd[i - 1][16] + 64                  # x_in = x_mid of the block before (inside ITS saved buffer)
        assert fwd[i][1] == y_buf and fwd[i][2] is not None      # x_add = the MLP branch output; the sum is materialised
    assert fwd[3][3] == out.data_ptr() and fwd[3][4] is None    # the last block adds by itself
    assert len({a[16] for a in fwd}) == 4 and len({a[2] for a in fwd[1:]}) == 3          # own saved / x_sum buffers
    out.sum().backward()
    bwd = [a for n, a in calls if n == "mmae_block_backward"]
    assert len(bwd) == 4
    # args: x_in, dx_out, dx_out_bf16, dx_in, dx_in_bf16, dx_in_colsum, ...; issued for blocks 3, 2, 1, 0
    assert bwd[0][2] is None and bwd[3][4] is None and bwd[3][5] is None
    for k in (1, 2, 3):
        assert bwd[k][1] == bwd[k - 1][3]                        # dx_out = the dx_in the block above produced
        assert bwd[k][2] == bwd[k - 1][4] is not None            # ... and its bf16 copy
        blk = 3 - k                                              # this call's block; the one above added into ITS fc2 bias slot
        assert bwd[k - 1][5] == arena.views["%d.mlp.fc2.bias" % blk].data_ptr()
        assert bwd[k][4] != bwd[k][2] or bwd[k][4] is None       # never reads and writes the same hand-off buffer
    # the saved x_in of backward is what forward used: x for block 0, the materialised sums above
    assert bwd[3][0] == x.data_ptr() and [b[0] for b in bwd[:3]] == [fwd[3][2], fwd[2][2], fwd[1][2]]
    assert [r[0].split(".")[0] for r in ready] == ["3", "2", "1", "0"] and all(len(r) == 12 for r in ready)
    assert x.grad is not None and x.grad.shape == x.shape


def test_shared_context_projection_pointers(monkeypatch):
    """SharedContextFunction / DecoderHeadFunction wiring: every head reads its column segment of the ONE projection output and
    writes its bf16 context gradient into the matching segment of the ONE gradient matrix that mmae_ctxproj_backward consumes;
    the four proj_context weights (and their gradient slots) are handed over in adapter order and lie back to back."""
    from multimae_b200 import multimae as MM
    from multimae_b200.criterion import MaskedMSELoss
    calls = []

    class Rec:
        def __getattr__(self, name):
            res, argtypes = L.SIGNATURES[name]

            def fn(*args):
                assert len(args) == len(argtypes), name
                calls.append((name, args))
                return 4096 if name.endswith("_bytes") else 0
            return fn

    rec = Rec()
    monkeypatch.setattr(L, "lib", lambda: rec)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(MM, "SHARED_CONTEXT_PROJECTION", True)
    model = _build().train()
    x = _inputs()
    preds, masks = model(x, num_encoded_tokens=12, alphas=1.0)
    order = list(preds)                                              # adapter order = column-segment order
    dims = [model.output_adapters[k].dim_tokens for k in order]
    offs = [sum(dims[:i]) for i in range(len(dims))]
    (pf,) = [a for n, a in calls if n == "mmae_ctxproj_forward"]
    prm = pf[3]._obj
    arena = model.grad_arena()
    assert prm.num == len(order) and list(prm.dim)[:len(order)] == dims
    for i, k in enumerate(order):
        ad = model.output_adapters[k]
        assert prm.weight[i] == ad.proj_context.weight.data_ptr() and prm.bias[i] == ad.proj_context.bias.data_ptr()
    ctx_ptr = pf[4]
    heads = [a for n, a in calls if n == "mmae_dechead_forward_ctx"]
    assert [h[0] for h in heads] == [ctx_ptr + 4 * o for o in offs] and all(h[1] == sum(dims) for h in heads)
    assert all(h[6]._obj.proj_context_w is None for h in heads)       # the weight belongs to the shared GEMM
    loss = sum(MaskedMSELoss(16, 1)(preds[k].float(), torch.zeros_like(preds[k]), mask=None) for k in preds)
    loss.backward()
    (pb,) = [a for n, a in calls if n == "mmae_ctxproj_backward"]
    dctx_ptr = pb[4]
    hb = {a[6]: a for n, a in calls if n == "mmae_dechead_backward_ctx"}
    assert sorted(hb) == [dctx_ptr + 2 * o for o in offs] and all(a[7] == sum(dims) for a in hb.values())
    grd = pb[3]._obj
    for i, k in enumerate(order):
        assert grd.weight[i] == arena.views["output_adapters.%s.proj_context.weight" % k].data_ptr()
        seg = hb[dctx_ptr + 2 * offs[i]]
        assert seg[4]._obj.proj_context_b == arena.views["output_adapters.%s.proj_context.bias" % k].data_ptr()
        assert seg[4]._obj.proj_context_w is None
    assert all(grd.weight[i + 1] == grd.weight[i] + 4 * dims[i] * pf[2] for i in range(len(order) - 1))   # back to back
