"""GPU: parity of the CUDA path (through the C ABI) against the oracle and the golden fixtures.

Tolerances (BASELINE.json north_star): indices bit-exact; floating point within 1e-2 relative L2 for the bf16 tensor-core
path against the fp32 oracle (per tensor: ||a-b|| / ||b||); fp32-only kernels (LayerNorm, losses, index kernels) 1e-5.
Nothing here reads /root/reference."""
import os

import pytest
import torch

from helpers import formula_fill_, load_fixture, rel_l2
from multimae_b200 import _lib as L
from oracle import multimae_oracle as O

pytestmark = pytest.mark.gpu

BF16_TOL = 1e-2          # activations / predictions / losses, relative L2
GRAD_TOL = 3e-2          # parameter gradients: global / median relative L2 (bf16 operands in dgrad and wgrad)
PER_TENSOR_TOL = 5e-2    # any single gradient tensor, error scaled as described in _check_grads


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _load(golden_dir, name):
    return load_fixture(golden_dir, name)


def _build_model(c):
    from test_host_api import _build
    return _build(tuple(c["in_domains"]), c["dim"], c["depth"], c["heads"], c["dec_dim"], c["dec_depth"], c["dec_heads"],
                  c["image_size"], out_domains=c.get("out_domains"), use_task_queries=c.get("use_task_queries", True))


def _oracle_cfg(c):
    cfg = O.make_config(in_domains=tuple(c["in_domains"]), out_domains=c.get("out_domains"))
    cfg.use_task_queries = c.get("use_task_queries", True)
    cfg.dim, cfg.depth, cfg.heads = c["dim"], c["depth"], c["heads"]
    cfg.dec_dim, cfg.dec_depth, cfg.dec_heads = c["dec_dim"], c["dec_depth"], c["dec_heads"]
    cfg.posemb_grid = c["image_size"] // 16
    return cfg


def _check_grads(got, ref):
    """Parameter gradients of the bf16 path against the fp32 oracle.

    G = global gradient norm, fair_t = G * sqrt(numel_t / N) = the norm tensor t would have at the global RMS.
      * global relative L2 over the concatenation of all gradients          < GRAD_TOL
      * every tensor:  ||got - ref|| <= PER_TENSOR_TOL * max(||ref||, fair_t)
        (tensors far below the global RMS are rounding-noise dominated: bound their absolute error by the scale that
         matters for the update instead of their own vanishing norm)
      * tensors carrying real signal (||ref|| >= 0.05 fair_t): median relative error < GRAD_TOL"""
    names = list(ref)
    for k in names:
        assert got[k] is not None and torch.isfinite(got[k]).all(), k
    flat_g = torch.cat([got[k].detach().float().cpu().flatten() for k in names])
    flat_r = torch.cat([ref[k].detach().float().cpu().flatten() for k in names])
    G, N = float(flat_r.norm()), flat_r.numel()
    glob = rel_l2(flat_g, flat_r)
    rows, signal = [], []
    for k in names:
        r = ref[k].detach().float().cpu()
        g = got[k].detach().float().cpu()
        fair = G * (r.numel() / N) ** 0.5
        err = float((g - r).norm())
        rows.append((err / max(float(r.norm()), fair), err / (float(r.norm()) + 1e-30), float(r.norm()) / fair, k))
        if float(r.norm()) >= 0.05 * fair:
            signal.append(err / float(r.norm()))
    rows.sort(reverse=True)
    signal.sort()
    median = signal[len(signal) // 2]
    print("global rel-l2 %.4f; median rel over %d signal tensors %.4f (max %.4f); worst scaled error %.4f (%s)" %
          (glob, len(signal), median, signal[-1], rows[0][0], rows[0][3]))
    print("worst tensors (scaled err, rel err, share):", [(round(a, 4), round(b, 3), round(c, 4), k) for a, b, c, k in rows[:5]])
    assert glob < GRAD_TOL, glob
    assert median < GRAD_TOL, median
    assert rows[0][0] < PER_TENSOR_TOL, rows[0]


def _loss_modules():
    from multimae_b200.criterion import MaskedCrossEntropyLoss, MaskedL1Loss, MaskedMSELoss
    return {"rgb": MaskedMSELoss(16, 1), "depth": MaskedL1Loss(16, 1), "semseg": MaskedCrossEntropyLoss(16, 4),
            "norm_rgb": MaskedMSELoss(16, 1, norm_pix=True)}


def _run_cuda_step(model, x, triple, dev, feed=None):
    """`x` holds the targets of every output task; `feed` names the entries handed to the model (default: all of x that
    have an input adapter), like train_one_epoch's input_dict / tasks_dict (run_pretraining_multimae.py:482-498)."""
    model.generate_random_masks = lambda *a, **k: triple
    fed = {k: v.to(dev) for k, v in x.items() if (feed is None or k in feed)}
    preds, masks = model(fed, num_encoded_tokens=triple[1].shape[1], alphas=1.0)
    fns = _loss_modules()
    losses = {}
    for task in preds:
        src = "rgb" if task == "norm_rgb" else task
        losses[task] = fns[task](preds[task].float(), x[src].to(dev), mask=masks.get(src))
    sum(losses.values()).backward()
    torch.cuda.synchronize()
    return preds, masks, losses


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sampler_small.pt", "sampler_cfg2.pt", "sampler_alpha.pt"])
def test_mask_sampler_bit_exact(golden_dir, dev, name):
    from multimae_b200 import functional as Fn
    fx = _load(golden_dir, name)
    counts = [n.shape[1] for n in fx["noises"]]
    masks, ids_keep, ids_restore = Fn.sample_masks(fx["shares"].to(dev), torch.cat(fx["noises"], 1).to(dev),
                                                   fx["noise_all"].to(dev), counts, fx["num_encoded"])
    assert torch.equal(ids_keep.cpu(), fx["ids_keep"])
    assert torch.equal(ids_restore.cpu(), fx["ids_restore"])
    assert torch.equal(masks.cpu(), torch.cat(fx["task_masks"], 1))
    assert masks.dtype == torch.int64 and ids_keep.dtype == torch.int64


def test_mask_sampler_large_and_properties(dev):
    """448^2-sized problem (3 x 784 tokens, 392 kept) against the oracle + structural properties."""
    from multimae_b200 import functional as Fn
    g = torch.Generator().manual_seed(5)
    B, counts, T = 32, [784, 784, 784], 392
    shares = torch.distributions.Dirichlet(torch.ones(3)).sample((B,))
    noises = [torch.rand(B, n, generator=g) for n in counts]
    noise_all = torch.rand(B, sum(counts), generator=g)
    ref_masks, ref_keep, ref_restore = O.sample_masks(shares, noises, noise_all, T)
    masks, ids_keep, ids_restore = Fn.sample_masks(shares.to(dev), torch.cat(noises, 1).to(dev), noise_all.to(dev), counts, T)
    assert torch.equal(ids_keep.cpu(), ref_keep) and torch.equal(ids_restore.cpu(), ref_restore)
    assert torch.equal(masks.cpu(), torch.cat(ref_masks, 1))
    assert bool(((masks == 0).sum(1) == T).all())                                   # exactly T visible per row
    assert bool((torch.sort(ids_restore, 1).values == torch.arange(sum(counts), device=dev)).all())   # a permutation


# cuda_xtask / cuda_noq: mask-token decoder queries (multimae/output_adapters.py:214-221) — a context task that is not fed
# in this call (its embedding rides in the spare task slot), --decoder_use_task_queries False, and an output task that is
# no context task at all (no embedding); their losses run without a mask (run_pretraining_multimae.py:520)
@pytest.mark.parametrize("name", ["cuda_small.pt", "cuda_interp.pt", "cuda_xtask.pt", "cuda_noq.pt"])
def test_model_against_golden_and_oracle(golden_dir, dev, name):
    fx = _load(golden_dir, name)
    c = fx["config"]
    feed = c.get("feed") or c["in_domains"]
    model = _build_model(c)
    formula_fill_(list(model.named_parameters()))
    model = model.to(dev).train()
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))
    preds, masks, losses = _run_cuda_step(model, fx["inputs"], triple, dev, feed=feed)
    assert set(preds) == set(fx["preds"])

    for k, ref in fx["preds"].items():
        assert rel_l2(preds[k], ref) < BF16_TOL, (k, rel_l2(preds[k], ref))
    for k, ref in fx["losses"].items():
        assert abs(float(losses[k]) - float(ref)) < BF16_TOL * abs(float(ref)), (k, float(losses[k]), float(ref))
    for k in masks:
        assert torch.equal(masks[k].cpu(), fx["task_masks"][k])

    # gradients: full tensors against the oracle (run here on CPU, fp32), digests against the reference fixture
    cfg = _oracle_cfg(c)
    p = O.init_params(cfg)
    train = O.trainable(p)
    formula_fill_(list(train.items()))
    for v in train.values():
        v.requires_grad_(True)
    o_losses, _ = O.step_losses(p, {d: fx["inputs"][d] for d in feed}, cfg, fx["task_masks"], fx["ids_keep"],
                                fx["ids_restore"], targets=fx["inputs"])
    sum(o_losses.values()).backward()
    named = dict(model.named_parameters())
    used = [k for k in train if train[k].grad is not None]      # e.g. the input adapter of a domain that was not fed
    assert set(used) == set(fx["grads"])
    for k in train:
        if k not in used:
            assert named[k].grad is None or float(named[k].grad.abs().sum()) == 0.0, k
    _check_grads({k: named[k].grad for k in used}, {k: train[k].grad for k in used})
    for k in used:                                         # and the reference's own digests
        d = fx["grads"][k]
        fair = float(fx["grad_norm"]) * (named[k].numel() / sum(v.numel() for v in train.values())) ** 0.5
        assert abs(float(named[k].grad.float().norm()) - float(d["norm"])) < PER_TENSOR_TOL * max(float(d["norm"]), fair), k


@pytest.mark.parametrize("flat_optimizer", [False, True])
@pytest.mark.parametrize("leave_out", [None, "depth"])
def test_shared_context_projection_matches_per_adapter(golden_dir, dev, monkeypatch, flat_optimizer, leave_out):
    """The proj_context Linears of the four output adapters as ONE GEMM on the shared encoder output (the default,
    mmae_ctxproj_* + mmae_dechead_*_ctx) against one GEMM per adapter (MMAE_SHARED_CTX=0, multimae/output_adapters.py:258 as
    the reference runs it): same bf16 operands and K order forward -> equal predictions; backward sums the four context
    gradients inside one K = sum Dd GEMM instead of four accumulated passes -> gradients equal to fp32 reassociation carried
    through the bf16 encoder backward.  `flat_optimizer`: parameters / bf16 mirror / gradient slots of the four Linears lie
    back to back and are used in place (FlatAdamW) vs gathered.  `leave_out`: a prediction that does not reach the loss -
    its head's backward never runs, its segment of the shared gradient matrix must count as zero."""
    from multimae_b200 import multimae as MM
    from multimae_b200.optim import FlatAdamW
    fx = _load(golden_dir, "cuda_small.pt")
    c = fx["config"]
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))

    def run(shared):
        monkeypatch.setattr(MM, "SHARED_CONTEXT_PROJECTION", shared)
        model = _build_model(c)
        formula_fill_(list(model.named_parameters()))
        model = model.to(dev).train()
        model.generate_random_masks = lambda *a, **k: triple
        if flat_optimizer:
            opt = FlatAdamW(model, lr=1e-3)      # noqa: F841  (keeps the bf16 mirror registered)
        before = L.lib().mmae_launch_count()
        preds, masks = model({k: v.to(dev) for k, v in fx["inputs"].items()}, num_encoded_tokens=12, alphas=1.0)
        fns = _loss_modules()
        loss = sum(fns[t](preds[t].float(), fx["inputs"]["rgb" if t == "norm_rgb" else t].to(dev),
                          mask=masks.get("rgb" if t == "norm_rgb" else t)) for t in preds if t != leave_out)
        loss.backward()
        torch.cuda.synchronize()
        grads = {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in model.named_parameters() if p.requires_grad}
        return {k: v.detach().clone() for k, v in preds.items()}, grads, L.lib().mmae_launch_count() - before

    p_shared, g_shared, n_shared = run(True)
    p_each, g_each, n_each = run(False)
    assert n_shared < n_each                       # 3 casts of the encoder output, 3 forward and >= 6 backward GEMMs fewer
    for k in p_each:
        assert rel_l2(p_shared[k], p_each[k]) < 1e-5, (k, rel_l2(p_shared[k], p_each[k]))
    names = [n for n in g_each if g_each[n] is not None and float(g_each[n].abs().sum()) > 0]
    for n in g_each:
        if n not in names:                         # e.g. the left-out adapter: no gradient either way
            assert g_shared[n] is None or float(g_shared[n].abs().sum()) == 0.0, n
    flat_s = torch.cat([g_shared[n].flatten() for n in names])
    flat_e = torch.cat([g_each[n].flatten() for n in names])
    assert rel_l2(flat_s, flat_e) < 5e-3, rel_l2(flat_s, flat_e)
    for n in names:
        if ".proj_context." in n:                  # same bf16 operands on both paths: fp32 summation order only
            assert rel_l2(g_shared[n], g_each[n]) < 1e-4, (n, rel_l2(g_shared[n], g_each[n]))


def test_block_chain_matches_single_blocks(golden_dir, dev, monkeypatch):
    """Consecutive Blocks with the hand-offs fused (BlockStackFunction / mmae_block_*_chain, the default) against one
    BlockFunction per block (MMAE_BLOCK_CHAIN=0): the residual add moves into the next block's first LayerNorm kernel and the
    gradient cast + fc2 bias gradient into its backward - the same fp32 operations on the same values, so predictions and
    gradients must agree to fp32 summation order (split-K reduce-adds, the fc2 bias column sums).  4 encoder blocks and
    2-block decoder transformers: both alternating hand-off buffers are in use."""
    from multimae_b200 import functional as Fn
    fx = _load(golden_dir, "cuda_small.pt")
    c = dict(fx["config"], depth=4, dec_depth=2)
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))

    def run(chain):
        monkeypatch.setattr(Fn, "BLOCK_CHAIN", chain)
        model = _build_model(c)
        formula_fill_(list(model.named_parameters()))
        model = model.to(dev).train()
        before = L.lib().mmae_launch_count()
        preds, _, losses = _run_cuda_step(model, fx["inputs"], triple, dev)
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.requires_grad}
        return {k: v.detach().clone() for k, v in preds.items()}, grads, L.lib().mmae_launch_count() - before

    p_chain, g_chain, n_chain = run(True)
    p_single, g_single, n_single = run(False)
    assert n_chain < n_single
    for k in p_single:
        assert rel_l2(p_chain[k], p_single[k]) < 1e-6, (k, rel_l2(p_chain[k], p_single[k]))
    for n in g_single:
        if n.endswith("mlp.fc2.bias"):
            assert rel_l2(g_chain[n], g_single[n]) < 1e-5, (n, rel_l2(g_chain[n], g_single[n]))
        elif "norm" in n or n.endswith(".bias") or "token" in n or "emb" in n:
            # column / row reductions that follow the hand-off read identical inputs; their own summation is deterministic
            assert rel_l2(g_chain[n], g_single[n]) < 1e-5, (n, rel_l2(g_chain[n], g_single[n]))
        else:
            assert rel_l2(g_chain[n], g_single[n]) < 1e-4, (n, rel_l2(g_chain[n], g_single[n]))   # split-K reduce-add order


FP32_TOL = 1e-3          # north_star "1e-3 rel fp32": the fp32 tier of fp32_output_adapters against the fp32 oracle


@pytest.mark.parametrize("task", ["semseg", "rgb"])
def test_fp32_output_adapter_tier(golden_dir, dev, task):
    """fp32_output_adapters (multimae/multimae.py:367-377): an adapter run in the fp32 tier - 3 x bf16 split wgmma GEMMs,
    fp32 attention / GELU / LayerNorm - against the fp32 oracle's decode_task on the SAME encoder tokens: prediction, the
    gradient w.r.t. the encoder tokens and every parameter gradient of the adapter to 1e-3."""
    fx = _load(golden_dir, "cuda_small.pt")
    c = fx["config"]
    model = _build_model(c)
    formula_fill_(list(model.named_parameters()))
    model = model.to(dev).train()
    cfg = _oracle_cfg(c)
    p = O.init_params(cfg)
    train = O.trainable(p)
    formula_fill_(list(train.items()))
    prefix = "output_adapters.%s." % task
    keys = [k for k in train if k.startswith(prefix)]
    for k in keys:
        train[k].requires_grad_(True)
    B, n_tok = c["B"], (c["image_size"] // 16) ** 2
    g = torch.Generator().manual_seed(5)
    enc = torch.randn(B, c["num_encoded"] + 1, c["dim"], generator=g) * 0.5
    enc_o = enc.clone().requires_grad_(True)
    counts = {d: n_tok for d in c["in_domains"]}
    hw = (c["image_size"], c["image_size"])
    ref = O.decode_task(enc_o, p, task, O.DOMAINS[task], cfg, counts, hw, fx["ids_keep"], fx["ids_restore"])
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()

    info = model.generate_input_info({d: torch.empty(B, n_tok, 0) for d in c["in_domains"]}, hw)
    model.grad_arena(dev).zero_()
    enc_d = enc.to(dev).requires_grad_(True)
    pred = model.output_adapters[task](enc_d, info, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev), fp32=True)
    (pred * w.to(dev)).sum().backward()
    torch.cuda.synchronize()
    assert pred.shape == ref.shape
    named = dict(model.named_parameters())
    total = sum(float(train[k].grad.norm()) ** 2 for k in keys) ** 0.5
    numel = sum(train[k].numel() for k in keys)
    worst = (0.0, None)
    for k in keys:
        r, got = train[k].grad, named[k].grad.detach().float().cpu()
        fair = total * (r.numel() / numel) ** 0.5
        e = float((got - r).norm()) / max(float(r.norm()), 0.05 * fair)
        worst = max(worst, (e, k))
        if e >= FP32_TOL:
            print("  gradient off: %-60s %.3e (||ref|| %.3e)" % (k, e, float(r.norm())))
    print("fp32 tier %s: pred %.2e, d_enc %.2e, worst parameter gradient %.2e (%s)" %
          (task, rel_l2(pred, ref), rel_l2(enc_d.grad, enc_o.grad), worst[0], worst[1]))
    assert rel_l2(pred, ref) < FP32_TOL, rel_l2(pred, ref)
    assert rel_l2(enc_d.grad, enc_o.grad) < FP32_TOL, rel_l2(enc_d.grad, enc_o.grad)
    assert worst[0] < FP32_TOL, worst


def test_fp32_output_adapters_flag_in_model(golden_dir, dev):
    """MultiMAE.forward(fp32_output_adapters=['semseg']) routes that adapter through the fp32 tier (no warning, no
    downgrade) and the step still matches the fixture."""
    import warnings
    fx = _load(golden_dir, "cuda_small.pt")
    c = fx["config"]
    model = _build_model(c)
    formula_fill_(list(model.named_parameters()))
    model = model.to(dev).train()
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))
    model.generate_random_masks = lambda *a, **k: triple
    fed = {k: v.to(dev) for k, v in fx["inputs"].items()}
    lib = L.lib()
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        before = lib.mmae_launch_count()
        preds, _ = model(fed, num_encoded_tokens=c["num_encoded"], fp32_output_adapters=["semseg"])
        n_fp32 = lib.mmae_launch_count() - before
        before = lib.mmae_launch_count()
        preds_b, _ = model(fed, num_encoded_tokens=c["num_encoded"])
        n_bf16 = lib.mmae_launch_count() - before
    assert n_fp32 > n_bf16                        # the split kernels of the fp32 tier ran
    for k, ref in fx["preds"].items():
        assert rel_l2(preds[k], ref) < BF16_TOL, (k, rel_l2(preds[k], ref))
    assert rel_l2(preds["semseg"], fx["preds"]["semseg"]) <= rel_l2(preds_b["semseg"], fx["preds"]["semseg"]) * 1.05
    sum(p.float().sum() for p in preds.values()).backward()
    torch.cuda.synchronize()
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)


def _full_model_case(dev, size, image_size, n_visible, B, oracle_on=None, global_tol=None):
    """One full-size step (forward, 4 losses, backward) of the CUDA path against the fp32 oracle on the same weights,
    synthetic inputs (SURVEY.md §8d generator) and oracle-sampled masks.  `oracle_on`: device the oracle runs on (fp32, TF32
    off; default CPU) - the bench-sized batch needs the GPU to finish in seconds."""
    from test_host_api import _build
    dim, depth, heads = (768, 12, 12) if size == "base" else (1024, 24, 16)     # multimae/multimae.py:387-397, 405-415
    model = _build(("rgb", "depth", "semseg"), dim, depth, heads, 256, 2, 8, image_size)
    torch.manual_seed(0)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():                                   # non-zero biases / mask tokens so every term is live
        for k, v in sd.items():
            if k.endswith(".bias") or k.endswith("mask_token"):
                v.add_(torch.randn(v.shape, generator=g) * 0.05)
    model.load_state_dict(sd)
    cfg = O.make_config(size=size)
    cfg.posemb_grid = image_size // 16
    x = O.synthetic_inputs(cfg, B, image_size, seed=0)
    shares, noises, noise_all = O.synthetic_mask_draws(cfg, B, image_size, seed=1)
    m, ids_keep, ids_restore = O.sample_masks(shares, noises, noise_all, n_visible)
    tmask = {d.name: mm for d, mm in zip(cfg.in_domains, m)}

    od = torch.device("cpu") if oracle_on is None else oracle_on
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False        # the oracle is fp32
    try:
        p = {k: v.clone().to(od) for k, v in sd.items()}
        train = O.trainable(p)
        for v in train.values():
            v.requires_grad_(True)
        o_losses, o_preds = O.step_losses(p, {k: v.to(od) for k, v in x.items()}, cfg, {k: v.to(od) for k, v in tmask.items()},
                                          ids_keep.to(od), ids_restore.to(od))
        sum(o_losses.values()).backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    o_preds = {k: v.detach().cpu() for k, v in o_preds.items()}
    o_losses = {k: v.detach().cpu() for k, v in o_losses.items()}

    model = model.to(dev).train()
    triple = ({k: v.to(dev) for k, v in tmask.items()}, ids_keep.to(dev), ids_restore.to(dev))
    preds, masks, losses = _run_cuda_step(model, x, triple, dev)
    for k in o_preds:
        assert preds[k].shape == o_preds[k].shape, k
        assert rel_l2(preds[k], o_preds[k]) < BF16_TOL, (k, rel_l2(preds[k], o_preds[k]))
        assert abs(float(losses[k]) - float(o_losses[k])) < BF16_TOL * abs(float(o_losses[k])), k
    named = dict(model.named_parameters())
    _check_grads({k: named[k].grad for k in train}, {k: v.grad for k, v in train.items()})
    if global_tol is not None:
        got = torch.cat([named[k].grad.detach().float().cpu().flatten() for k in train])
        ref = torch.cat([v.grad.detach().float().cpu().flatten() for v in train.values()])
        assert rel_l2(got, ref) < global_tol, rel_l2(got, ref)


def test_bench_batch_model_against_oracle_on_cuda(dev):
    """BASELINE config 2 at a bench-sized batch (B = 64: encoder M = 6336 rows, decoder M = 12544 - the persistent / CTA-pair
    GEMM variants, BN = 192 / 256 tiles, automatic split-K and the warp-specialised attention kernels run as in bench.py)
    against the fp32 oracle evaluated on the same GPU in plain fp32 (TF32 off).  Global gradient error < 1e-2."""
    _full_model_case(dev, "base", 224, 98, B=64, oracle_on=dev, global_tol=1e-2)


def test_full_size_model_against_oracle(dev):
    """MultiMAE-B, rgb+depth+semseg, 224^2, 98 visible tokens (BASELINE config 2 at B=2) against the fp32 oracle."""
    _full_model_case(dev, "base", 224, 98, B=2)


def test_large_model_against_oracle(dev):
    """MultiMAE-L (24 layers, d=1024, 16 heads), rgb+depth+semseg, 224^2, 98 visible tokens: BASELINE config 4 at B=1."""
    _full_model_case(dev, "large", 224, 98, B=1)


def test_448_model_against_oracle(dev):
    """MultiMAE-B at 448^2: 3 x 784 patches, 392 visible tokens (393-token encoder sequence, 784-query decoders):
    BASELINE config 5 at B=1."""
    _full_model_case(dev, "base", 448, 392, B=1)


def test_multivit_encoder_against_oracle(dev):
    """MultiViT (multimae/multimae.py:419-502): no masking, every token of every given modality encoded; encoder tokens of
    the last layer and of every layer (return_all_layers) against the oracle run with ids_keep = all tokens."""
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    B, S = 2, 224
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=S),
           "depth": PatchedInputAdapter(num_channels=1, stride_level=1, patch_size_full=16, image_size=S)}
    torch.manual_seed(0)
    model = multivit_base(ins, None)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for k, v in sd.items():
            if k.endswith(".bias"):
                v.add_(torch.randn(v.shape, generator=g) * 0.05)
    model.load_state_dict(sd)
    cfg = O.make_config(in_domains=("rgb", "depth"), out_domains=[], extra_norm_pix=False)
    x = O.synthetic_inputs(cfg, B, S, seed=0)
    n_tok = 2 * (S // 16) ** 2
    ids = torch.arange(n_tok).unsqueeze(0).expand(B, -1).contiguous()
    p = {k: v.clone() for k, v in sd.items()}
    _, o_tokens = O.forward(p, x, cfg, ids, ids)

    model = model.to(dev).eval()
    xd = {k: v.to(dev) for k, v in x.items()}
    with torch.no_grad():
        got = model(xd)
        layers = model(xd, return_all_layers=True)
    assert got.shape == (B, n_tok + 1, 768) and len(layers) == 12
    assert rel_l2(got, o_tokens) < BF16_TOL, rel_l2(got, o_tokens)
    assert rel_l2(layers[-1], o_tokens) < BF16_TOL
    # a Tensor input is taken as RGB (multimae/multimae.py:441-442)
    model_rgb = multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=S)},
                              None).to(dev).eval()
    with torch.no_grad():
        assert model_rgb(xd["rgb"]).shape == (B, (S // 16) ** 2 + 1, 768)


def test_losses_against_oracle(dev):
    from multimae_b200.criterion import MaskedCrossEntropyLoss, MaskedL1Loss, MaskedMSELoss
    g = torch.Generator().manual_seed(0)
    B = 5
    mask = (torch.rand(B, 196, generator=g) > 0.3).long()
    mask[1] = 0                                               # a sample with no masked patch -> skipped by nanmean
    cases = [
        (MaskedMSELoss(16, 1), lambda p_, t, m: O.masked_mse(p_, t, m, 16, 1), torch.randn(B, 3, 224, 224, generator=g),
         torch.randn(B, 3, 224, 224, generator=g)),
        (MaskedMSELoss(16, 1, norm_pix=True), lambda p_, t, m: O.masked_mse(p_, t, m, 16, 1, norm_pix=True),
         torch.randn(B, 3, 224, 224, generator=g), torch.randn(B, 3, 224, 224, generator=g) * 3 + 1),
        (MaskedL1Loss(16, 1), lambda p_, t, m: O.masked_l1(p_, t, m, 16, 1), torch.randn(B, 1, 224, 224, generator=g),
         torch.randn(B, 1, 224, 224, generator=g)),
        (MaskedCrossEntropyLoss(16, 4), lambda p_, t, m: O.masked_ce(p_, t, m, 16, 4),
         torch.randn(B, 133, 56, 56, generator=g) * 2, torch.randint(0, 133, (B, 56, 56), generator=g)),
    ]
    for mod, ofn, pred, tgt in cases:
        for mk in (mask, None, torch.zeros_like(mask)):
            pr = pred.clone().requires_grad_(True)
            ref = ofn(pr, tgt, mk)
            pc = pred.to(dev).requires_grad_(True)
            got = mod(pc, tgt.to(dev), mask=None if mk is None else mk.to(dev))
            assert abs(float(got) - float(ref)) <= 2e-5 * max(1.0, abs(float(ref))), (type(mod).__name__, float(got), float(ref))
            if ref.requires_grad:
                ref.backward()
                got.backward()
                # a sample WITHOUT masked patches is skipped by nanmean in forward, but the reference's autograd turns
                # its 0/0 into NaN gradients (0 * inf); the fused kernel writes exact zeros there (documented divergence;
                # unreachable in pre-training: every task keeps >= 98 of its 196 patches masked)
                live = torch.ones(B, dtype=torch.bool) if mk is None else (mk.sum(1) > 0)
                assert torch.isnan(pr.grad[~live]).all() or (~live).sum() == 0
                assert float(pc.grad[(~live).to(dev)].abs().sum()) == 0.0
                assert rel_l2(pc.grad[live.to(dev)], pr.grad[live]) < 1e-5, type(mod).__name__
            else:                                             # all-zero mask: constant 0 (criterion.py:42,100,157)
                assert float(got) == 0.0


def test_flat_adamw_matches_torch(dev):
    from multimae_b200 import functional as Fn
    torch.manual_seed(0)
    n = 10007
    p0 = torch.randn(n, device=dev)
    g0 = torch.randn(n, device=dev)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref], lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.05)
    flat, m, v = p0.clone(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    for step in range(1, 4):
        ref.grad = g0 * step
        opt.step()
        Fn.adamw_step(flat, g0 * step, m, v, 1e-3, (0.9, 0.95), 1e-8, 0.05, step)
    assert rel_l2(flat, ref.data) < 1e-6
    # grad norm / unscale
    gflat = torch.randn(100003, device=dev)
    ref_norm = (gflat * 0.5).norm()
    norm, out2 = Fn.grad_unscale_norm(gflat, inv_scale=0.5)
    assert abs(float(norm) - float(ref_norm)) < 1e-4 * float(ref_norm) and float(out2[1]) == 0.0
    gflat[17] = float("inf")
    _, out2 = Fn.grad_unscale_norm(gflat)
    assert float(out2[1]) == 1.0


def test_cuda_graph_step_matches_eager(dev, golden_dir):
    """The whole train step captured as one CUDA graph (train_step.TrainStep) reproduces the eager step: with the mask
    triple pinned, 1 eager warm-up + 3 replays equals 4 eager steps (same kernels in the same order; only fp32 atomics
    reorder)."""
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep
    fx = _load(golden_dir, "cuda_small.pt")
    c = fx["config"]
    x = {k: v.to(dev) for k, v in fx["inputs"].items()}
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))

    def run(use_graph):
        model = _build_model(c)
        formula_fill_(list(model.named_parameters()))
        model = model.to(dev).train()
        model.generate_random_masks = lambda *a, **k: triple
        opt = FlatAdamW(model, lr=1e-3)
        scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
        step = TrainStep(model, _loss_modules(), opt, scaler, num_encoded_tokens=12, loss_sources={"norm_rgb": "rgb"})
        losses = []
        if use_graph:
            step.capture(x, warmup=1)
            assert step.graph is not None
        else:
            step(x)
        for _ in range(3):
            loss, norm = step(x)
            losses.append(float(loss))
        torch.cuda.synchronize()
        return losses, opt.flat_params.clone(), float(opt._dyn[1])

    l_eager, p_eager, n_eager = run(False)
    l_graph, p_graph, n_graph = run(True)
    assert n_eager == n_graph == 4.0                      # device-side step counter advanced by the replays
    assert all(abs(a - b) <= 2e-3 * abs(a) for a, b in zip(l_eager, l_graph)), (l_eager, l_graph)
    assert l_eager[-1] < l_eager[0]
    assert rel_l2(p_graph, p_eager) < 1e-3


def test_bf16_weight_mirror_tracks_parameters(dev, golden_dir):
    """FlatAdamW registers a bf16 twin of the flat parameter buffer: the update kernel keeps it equal to bf16(params), a
    change made through torch is picked up before the next launch, and a step that reads its weights from the twin gives
    the same loss as one that casts them per call (twin unregistered)."""
    from multimae_b200 import _lib as L
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep
    fx = _load(golden_dir, "cuda_small.pt")
    c = fx["config"]
    x = {k: v.to(dev) for k, v in fx["inputs"].items()}
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))

    def run(with_mirror):
        model = _build_model(c)
        formula_fill_(list(model.named_parameters()))
        model = model.to(dev).train()
        model.generate_random_masks = lambda *a, **k: triple
        opt = FlatAdamW(model, lr=1e-3)
        if not with_mirror:
            opt.release_mirror()
        scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
        step = TrainStep(model, _loss_modules(), opt, scaler, num_encoded_tokens=12, loss_sources={"norm_rgb": "rgb"})
        losses = [float(step(x)[0]) for _ in range(3)]
        if with_mirror:
            torch.cuda.synchronize()
            assert torch.equal(opt.flat_bf16, opt.flat_params.to(torch.bfloat16))      # written by the update kernel
            with torch.no_grad():
                next(model.parameters()).mul_(1.5)                                     # bumps the version counter
            assert opt._mirror_version != opt._params_version()
            step(x)
            torch.cuda.synchronize()
            assert torch.equal(opt.flat_bf16, opt.flat_params.to(torch.bfloat16))
        return losses

    launches0 = L.lib().mmae_launch_count()
    l_mirror = run(True)
    l_cast = run(False)
    assert L.lib().mmae_launch_count() > launches0
    assert abs(l_mirror[0] - l_cast[0]) <= 1e-6 * abs(l_cast[0]), (l_mirror, l_cast)   # same bf16 operand bits
    assert all(abs(a - b) <= 1e-3 * abs(a) for a, b in zip(l_mirror, l_cast)), (l_mirror, l_cast)   # atomics reorder
