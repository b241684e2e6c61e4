"""GPU: deterministic mode (torch.use_deterministic_algorithms on; warn_only, so torch's own ops in the steps below warn
instead of raising where they have no deterministic form - the library's switch is on either way).

1. Exact order: the ordered split-K GEMM equals, bit for bit, the per-split GEMMs (each unsplit on its K slice) added on
   the device in split order in fp32 and then onto the destination, at the bench's weight-gradient shapes, with and
   without accumulate (a split-K GEMM adds onto out_f32 either way, as in the unordered form).
2. Whole steps repeat bit for bit from identical state and seeds - losses, every gradient, the parameters after the
   optimizer step - and give the same bits under mmae_set_sm_budget(66) as on the full card: pre-training at the bench
   config with a reduced batch (eager and graph-replayed, FlatAdamW), classification, ConvNeXt semseg and Segmenter
   fine-tuning and ConvNeXt depth fine-tuning (stock AdamW and GroupedFlatAdamW).  With the mode off, some weight-gradient shape differs between the
   two budgets, because the automatic split count follows the SM count.
3. Flag-on results stay close to flag-off ones (the same arithmetic in another summation order).
"""
import ctypes
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TOKENS = 128 * 99              # the bench's encoder rows: batch 128 x (98 visible + 1 global token)
DET_KB_PER_SPLIT = 32          # gemm_wgmma.cu: most k-blocks of 64 per split of the automatic split in deterministic mode


@pytest.fixture()
def det():
    """Deterministic mode on for the test; torch's flag, the library's switch and the SM budget restored afterwards."""
    from multimae_b200 import _lib as L
    from multimae_b200 import functional as Fn
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    Fn.sync_deterministic()
    yield L.lib()
    torch.use_deterministic_algorithms(was, warn_only=warn)
    Fn.sync_deterministic()
    L.lib().mmae_set_sm_budget(0)


def _wgrad(lib, dy, x, out, accumulate, split_k=0):
    """out[Nout, Kin] (+)= dy[T, Nout]^T x[T, Kin]: the weight-gradient GEMM form of modules.cu (both operands MN-major)."""
    from multimae_b200 import _lib as L
    T, Nout = dy.shape
    Kin = x.shape[1]
    ep = L.GemmEpilogue()
    ep.alpha = 1.0
    ep.accumulate = int(accumulate)
    ep.out_f32 = out.data_ptr()
    ep.ld_out_f32 = Kin
    L.check(lib.mmae_gemm_bf16(dy.data_ptr(), Nout, 1, x.data_ptr(), Kin, 1, Nout, Kin, T, split_k, ctypes.byref(ep),
                               L.current_stream()), "mmae_gemm_bf16")


SHAPES = [(2304, 768), (768, 768), (3072, 768), (768, 3072)]     # qkv, proj, fc1, fc2 weights: (Nout, Kin)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("nout,kin", SHAPES)
def test_ordered_split_k_is_the_per_split_sum_in_split_order(det, nout, kin, accumulate):
    lib = det
    g = torch.Generator(device="cuda").manual_seed(nout * 7 + kin)
    dy = torch.randn(TOKENS, nout, device="cuda", generator=g).bfloat16()
    x = torch.randn(TOKENS, kin, device="cuda", generator=g).bfloat16()
    init = torch.randn(nout, kin, device="cuda", generator=g)
    out = init.clone()
    _wgrad(lib, dy, x, out, accumulate)
    kblocks = math.ceil(TOKENS / 64)
    splits = math.ceil(kblocks / DET_KB_PER_SPLIT)          # the split count follows K alone ...
    rows = math.ceil(kblocks / splits) * 64                  # ... and the k-blocks are spread evenly over the splits
    assert splits > 1 and math.ceil(TOKENS / rows) == splits
    total = None
    for s in range(splits):
        part = torch.zeros(nout, kin, device="cuda")
        _wgrad(lib, dy[s * rows:(s + 1) * rows], x[s * rows:(s + 1) * rows], part, False, split_k=1)
        total = part if total is None else total + part
    ref = init + total
    torch.cuda.synchronize()
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    # and the sum itself is right
    exact = dy.double().t() @ x.double() + init.double()
    assert ((out.double() - exact).norm() / exact.norm()).item() < 1e-5


def test_sm_budget_changes_flag_off_bits_but_not_flag_on(det):
    lib = det
    from multimae_b200 import functional as Fn
    g = torch.Generator(device="cuda").manual_seed(3)
    data = [(torch.randn(TOKENS, n, device="cuda", generator=g).bfloat16(),
             torch.randn(TOKENS, k, device="cuda", generator=g).bfloat16()) for n, k in SHAPES]

    def run(budget):
        lib.mmae_set_sm_budget(budget)
        outs = []
        for dy, x in data:
            out = torch.zeros(dy.shape[1], x.shape[1], device="cuda")
            _wgrad(lib, dy, x, out, True)
            outs.append(out)
        torch.cuda.synchronize()
        lib.mmae_set_sm_budget(0)
        return outs

    on_full, on_half = run(0), run(66)
    assert all(torch.equal(a, b) for a, b in zip(on_full, on_half))
    torch.use_deterministic_algorithms(False)
    Fn.sync_deterministic()
    off_full, off_half = run(0), run(66)
    assert any(not torch.equal(a, b) for a, b in zip(off_full, off_half))   # the test has teeth
    for a, b in zip(on_full, off_full):
        assert ((a - b).norm() / b.norm()).item() < 1e-5


# ---- whole steps -------------------------------------------------------------------------------------------------------
def _trainable(model):
    return [(n, p) for n, p in model.named_parameters() if p.requires_grad]


def _state(model, loss):
    torch.cuda.synchronize()
    return ([loss.detach().float().clone()] + [p.grad.detach().clone() for _, p in _trainable(model)] +
            [p.detach().clone() for _, p in _trainable(model)])


def _pretrain(graph):
    def run():
        import bench
        from multimae_b200.native_scaler import NativeScalerWithGradNormCount
        from multimae_b200.optim import FlatAdamW
        from multimae_b200.train_step import TrainStep
        dev = torch.device("cuda")
        torch.manual_seed(0)
        model, loss_fns = bench.build_model_and_losses(dev, "base", 224)
        opt = FlatAdamW(model, lr=1e-4, betas=(0.9, 0.95), weight_decay=0.05)
        scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
        torch.manual_seed(1234)
        x = {k: v.to(dev) for k, v in bench.synthetic_batch(32, 7).items()}
        step = TrainStep(model, loss_fns, opt, scaler, num_encoded_tokens=98, alphas=1.0, loss_sources={"norm_rgb": "rgb"})
        if graph:
            step.capture(x, warmup=1)
        loss, _ = step(x)
        return _state(model, loss)
    return run


def _finetune(head, optim):
    def run():
        from multimae_b200 import multimae as mm
        S, B = (224, 8) if head == "cls" else (256, 4)
        torch.manual_seed(0)
        own, mm.AUTO_OWN_GRADIENTS = mm.AUTO_OWN_GRADIENTS, True     # p.grad aliases the arena, as under the overlay
        try:
            return _finetune_step(mm, head, optim, S, B)
        finally:
            mm.AUTO_OWN_GRADIENTS = own
    return run


def _finetune_step(mm, head, optim, S, B):
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import GroupedFlatAdamW
    from multimae_b200.output_adapters import ConvNeXtAdapter, LinearOutputAdapter, SegmenterMaskTransformerAdapter
    dev = torch.device("cuda")
    out = {"cls": lambda: LinearOutputAdapter(100),
           "convnext": lambda: ConvNeXtAdapter(41, embed_dim=6144, preds_per_patch=16, depth=4),
           "segmenter": lambda: SegmenterMaskTransformerAdapter(41, embed_dim=768, depth=2),
           "depth": lambda: ConvNeXtAdapter(1, preds_per_patch=64, main_tasks=["rgb"])}[head]()
    key = {"cls": "cls", "depth": "depth"}.get(head, "semseg")
    model = mm.multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16,
                                                         image_size=S)}, {key: out}, drop_path_rate=0.1).to(dev)
    params = [p for p in model.parameters() if p.requires_grad]
    opt = (GroupedFlatAdamW(params, lr=1e-4, weight_decay=0.05) if optim == "grouped"
           else torch.optim.AdamW(params, lr=1e-4, weight_decay=0.05))
    scaler = NativeScalerWithGradNormCount()
    torch.manual_seed(5)
    x = torch.randn(B, 3, S, S, device=dev)
    if head == "cls":
        target = torch.randint(0, 100, (B,), device=dev)
    elif head == "depth":
        target = 0.5 + 4.0 * torch.rand(B, 1, S, S, device=dev)
    else:
        target = torch.randint(0, 41, (B, S, S), device=dev)
    model.train()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        pred = model({"rgb": x})[key].float()
        loss = (torch.nn.functional.l1_loss(pred, target) if head == "depth"
                else torch.nn.functional.cross_entropy(pred, target))
    scaler(loss, opt, clip_grad=None, parameters=model.parameters())
    return _state(model, loss)


STEPS = {
    "pretrain-eager": _pretrain(False),
    "pretrain-graph": _pretrain(True),
    "cls-adamw": _finetune("cls", "stock"),
    "cls-grouped": _finetune("cls", "grouped"),
    "convnext-adamw": _finetune("convnext", "stock"),
    "convnext-grouped": _finetune("convnext", "grouped"),
    "segmenter-adamw": _finetune("segmenter", "stock"),
    "segmenter-grouped": _finetune("segmenter", "grouped"),
    "convnext-depth-adamw": _finetune("depth", "stock"),
    "convnext-depth-grouped": _finetune("depth", "grouped"),
}


def _first_difference(a, b):
    for i, (u, v) in enumerate(zip(a, b)):
        if not torch.equal(u, v):
            return i, (u.double() - v.double()).abs().max().item()
    return None


@pytest.mark.parametrize("name", list(STEPS))
def test_step_repeats_bitwise_on_any_sm_budget(det, name):
    lib = det
    run = STEPS[name]
    first = run()
    second = run()
    assert len(first) == len(second) and len(first) > 3
    assert _first_difference(first, second) is None, _first_difference(first, second)
    lib.mmae_set_sm_budget(66)
    try:
        half = run()
    finally:
        lib.mmae_set_sm_budget(0)
    assert _first_difference(first, half) is None, _first_difference(first, half)
    assert all(torch.isfinite(t).all() for t in first)


@pytest.mark.parametrize("name", ["pretrain-eager", "cls-grouped", "convnext-grouped", "segmenter-grouped",
                                  "convnext-depth-grouped"])
def test_flag_on_stays_close_to_flag_off(det, name):
    from multimae_b200 import functional as Fn
    on = STEPS[name]()
    torch.use_deterministic_algorithms(False)
    Fn.sync_deterministic()
    off = STEPS[name]()
    assert abs(on[0].item() - off[0].item()) <= 1e-3 * abs(off[0].item())
    n = (len(on) - 1) // 2
    g_on = torch.cat([t.flatten().double() for t in on[1:1 + n]])
    g_off = torch.cat([t.flatten().double() for t in off[1:1 + n]])
    assert ((g_on - g_off).norm() / g_off.norm()).item() < 2e-2


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 CUDA devices (NCCL data-parallel repeat)")
def test_data_parallel_step_repeats_bitwise(tmp_path):
    import subprocess
    saved = []
    for i in range(2):
        out = str(tmp_path / ("run%d.pt" % i))
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
               "127.0.0.1", "--master-port", "29534", os.path.join(ROOT, "scripts", "gpu_check_dp_deterministic.py"), out]
        res = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
        assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
        saved.append(torch.load(out))
    for k in ("loss", "norm", "grad", "params"):
        assert torch.equal(saved[0][k], saved[1][k]), k
