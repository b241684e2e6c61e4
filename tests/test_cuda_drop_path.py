"""GPU: stochastic depth (drop path) inside the fused block kernels (the scale arguments of mmae_block_*).

The per-sample factors are pinned by substituting functional.drop_path_scales (as other tests substitute
generate_random_masks); the oracle runs with the same factors (tests/drop_path_oracle.py).  Nothing here reads the reference checkout."""
import pytest
import torch

from drop_path_oracle import applied
from helpers import formula_fill_, load_fixture, rel_l2
from multimae_b200 import functional as Fn
from oracle import multimae_oracle as O

pytestmark = pytest.mark.gpu

BF16_TOL = 1e-2
GRAD_TOL = 3e-2
PER_TENSOR_TOL = 5e-2
FP32_TOL = 1e-3


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _check_grads(got, ref):
    """Parameter gradients of the bf16 path against the fp32 oracle (the criteria of test_cuda_parity._check_grads)."""
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
    print("global rel-l2 %.4f; median rel over %d signal tensors %.4f; worst scaled error %.4f (%s)" %
          (glob, len(signal), median, rows[0][0], rows[0][3]))
    assert glob < GRAD_TOL, glob
    assert median < GRAD_TOL, median
    assert rows[0][0] < PER_TENSOR_TOL, rows[0]


# ------------------------------------------------------------------------------------------------------------- helpers
def _set_drop_path(blocks, rate):
    """drop_path = linspace(0, rate, depth)[i] on block i, as the model constructors do."""
    from multimae_b200.multimae_utils import DropPath
    dpr = [v.item() for v in torch.linspace(0, rate, len(blocks))]
    for b, p in zip(blocks, dpr):
        b.drop_path = DropPath(p) if p > 0 else torch.nn.Identity()


def _model_stacks(model):
    """(prefix, nn.Sequential of Blocks) of the encoder and of every output adapter's decoder_transformer."""
    out = [("encoder", model.encoder)]
    for k, ad in (model.output_adapters or {}).items():
        if isinstance(ad.decoder_transformer, torch.nn.Sequential):
            out.append(("output_adapters.%s.decoder_transformer" % k, ad.decoder_transformer))
    return out


def _pattern_scales(model, B, dev):
    """{block prefix: (s_attn, s_mlp)} on `dev` for every block with p > 0: a different sample dropped per branch and block,
    the others kept (1/keep)."""
    table, k = {}, 0
    for prefix, blocks in _model_stacks(model):
        for i, b in enumerate(blocks):
            p = Fn.drop_path_prob(b)
            if p == 0.0:
                continue
            inv = float(torch.tensor(1.0) / (1.0 - p))
            a = torch.tensor([0.0 if (s + k) % 3 == 0 else inv for s in range(B)])
            m = torch.tensor([0.0 if (s + k) % 3 == 1 else inv for s in range(B)])
            table["%s.%d" % (prefix, i)] = (a.to(dev), m.to(dev))
            k += 1
    return table


def _pin_by_prefix(monkeypatch, table):
    def fake(blocks, batch, device):
        out = []
        for b in blocks:
            if Fn.drop_path_prob(b) == 0.0:
                out.append(None)
            else:
                out.append(table[b._meta["prefix"].rstrip(".")])
        return out
    monkeypatch.setattr(Fn, "drop_path_scales", fake)


def _pin_by_block(monkeypatch, table):
    monkeypatch.setattr(Fn, "drop_path_scales",
                        lambda blocks, batch, device: [table.get(id(b)) if Fn.drop_path_prob(b) > 0 else None
                                                       for b in blocks])


def _block_stack(dev, n=4, dim=128, heads=2, seed=0):
    from multimae_b200.multimae_utils import Block
    torch.manual_seed(seed)
    blocks = torch.nn.Sequential(*[Block(dim, heads, qkv_bias=True) for _ in range(n)])
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in blocks.named_parameters():
            if name.endswith(".bias") or "norm" in name:
                p.add_(torch.randn(p.shape, generator=g) * 0.05)
    blocks = blocks.to(dev).train()
    arena = Fn.GradArena(list(blocks.named_parameters()), dev)
    for i, b in enumerate(blocks):
        b.bind(arena, "%d." % i)
    return blocks, arena


def _run_stack(blocks, arena, x, dout, fp32=False):
    arena.zero_()
    xi = x.clone().requires_grad_(True)
    out = Fn.block_stack(blocks, xi, fp32=fp32)
    out.backward(dout)
    torch.cuda.synchronize()
    return out.detach().clone(), xi.grad.clone(), {k: v.clone() for k, v in arena.views.items()}


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("chain", [True, False])
def test_all_keep_equals_no_drop_path_bf16(dev, monkeypatch, chain):
    """Every factor 1.0: x + 1.0f * y == x + y exactly (with or without FMA contraction), so outputs, dx and the LayerNorm /
    bias gradients equal the p = 0 call bit for bit; weight gradients agree to split-K reduce-add order."""
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", chain)
    B, N, D = 3, 37, 128
    blocks, arena = _block_stack(dev)
    g = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(B, N, D, device=dev, generator=g)
    dout = torch.randn(B, N, D, device=dev, generator=g)
    ref = _run_stack(blocks, arena, x, dout)
    _set_drop_path(blocks, 0.5)
    ones = {id(b): (torch.ones(B, device=dev), torch.ones(B, device=dev)) for b in blocks}
    _pin_by_block(monkeypatch, ones)
    from multimae_b200 import _lib as L
    calls = L.lib().mmae_launch_count()
    got = _run_stack(blocks, arena, x, dout)
    assert L.lib().mmae_launch_count() > calls
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    for k in ref[2]:
        if "norm" in k or k.endswith(".bias"):
            assert torch.equal(got[2][k], ref[2][k]), k
        else:
            assert rel_l2(got[2][k], ref[2][k]) < 1e-5, (k, rel_l2(got[2][k], ref[2][k]))


def test_all_keep_equals_no_drop_path_fp32(dev, monkeypatch):
    B, N, D = 2, 37, 128
    blocks, arena = _block_stack(dev, n=2, heads=4)           # the fp32 tier runs head_dim 32 (the decoders')
    g = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(B, N, D, device=dev, generator=g)
    dout = torch.randn(B, N, D, device=dev, generator=g)
    ref = _run_stack(blocks, arena, x, dout, fp32=True)
    _set_drop_path(blocks, 0.5)
    _pin_by_block(monkeypatch, {id(b): (torch.ones(B, device=dev), torch.ones(B, device=dev)) for b in blocks})
    got = _run_stack(blocks, arena, x, dout, fp32=True)
    assert rel_l2(got[0], ref[0]) < 1e-6 and rel_l2(got[1], ref[1]) < 1e-6
    for k in ref[2]:
        assert rel_l2(got[2][k], ref[2][k]) < 1e-6, (k, rel_l2(got[2][k], ref[2][k]))


@pytest.mark.parametrize("fp32", [False, True])
def test_dropped_sample_is_identity(dev, monkeypatch, fp32):
    """Stand-alone Blocks, each built with drop_path > 0 (block 0 included): a sample whose factors are 0 in every block
    leaves the stack unchanged (out rows == in rows, dx rows == dout rows, bit for bit), and contributes nothing to the
    parameter gradients (== the same call with its dout zeroed)."""
    from multimae_b200.multimae_utils import Block
    torch.manual_seed(4)
    blocks = [Block(128, 4, qkv_bias=True, drop_path=0.3).to(dev).train() for _ in range(3)]
    B, N, D = 3, 37, 128
    inv = float(torch.tensor(1.0) / 0.7)
    table = {}
    for i, b in enumerate(blocks):
        a = torch.tensor([inv, 0.0, 0.0 if i == 1 else inv], device=dev)
        m = torch.tensor([inv if i != 2 else 0.0, 0.0, inv], device=dev)
        table[id(b)] = (a, m)
    _pin_by_block(monkeypatch, table)
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.randn(B, N, D, device=dev, generator=g)
    dout = torch.randn(B, N, D, device=dev, generator=g)

    def run(d):
        xi = x.clone().requires_grad_(True)
        h = xi
        for b in blocks:
            h = b(h, fp32=fp32)
        h.backward(d)
        torch.cuda.synchronize()
        grads = {"%d.%s" % (i, k): v.clone() for i, b in enumerate(blocks) for k, v in b._meta["arena"].views.items()}
        return h.detach().clone(), xi.grad.clone(), grads

    out, dx, grads = run(dout)
    assert torch.equal(out[1], x[1]) and torch.equal(dx[1], dout[1])
    assert not torch.equal(out[0], x[0]) and not torch.equal(out[2], x[2])
    d0 = dout.clone()
    d0[1] = 0
    _, _, grads0 = run(d0)
    for k in grads:
        assert rel_l2(grads[k], grads0[k]) < 1e-5, (k, rel_l2(grads[k], grads0[k]))


def _cuda_small(golden_dir, dev, rate):
    from test_host_api import _build
    fx = load_fixture(golden_dir, "cuda_small.pt")
    c = dict(fx["config"], depth=4, dec_depth=2)
    model = _build(tuple(c["in_domains"]), c["dim"], c["depth"], c["heads"], c["dec_dim"], c["dec_depth"], c["dec_heads"],
                   c["image_size"])
    formula_fill_(list(model.named_parameters()))
    for _, blocks in _model_stacks(model):
        _set_drop_path(blocks, rate)
    return fx, c, model.to(dev).train()


def _oracle(c):
    cfg = O.make_config(in_domains=tuple(c["in_domains"]))
    cfg.dim, cfg.depth, cfg.heads = c["dim"], c["depth"], c["heads"]
    cfg.dec_dim, cfg.dec_depth, cfg.dec_heads = c["dec_dim"], c["dec_depth"], c["dec_heads"]
    cfg.posemb_grid = c["image_size"] // 16
    p = O.init_params(cfg)
    train = O.trainable(p)
    formula_fill_(list(train.items()))
    for v in train.values():
        v.requires_grad_(True)
    return cfg, p, train


def _loss_modules():
    from multimae_b200.criterion import MaskedCrossEntropyLoss, MaskedL1Loss, MaskedMSELoss
    return {"rgb": MaskedMSELoss(16, 1), "depth": MaskedL1Loss(16, 1), "semseg": MaskedCrossEntropyLoss(16, 4),
            "norm_rgb": MaskedMSELoss(16, 1, norm_pix=True)}


@pytest.mark.parametrize("chain", [True, False])
def test_model_against_oracle_mixed_scales(golden_dir, dev, monkeypatch, chain):
    """cuda_small with encoder depth 4, decoder depth 2 and drop_path_rate 0.5 everywhere, in training, mask triple and
    factors pinned (a dropped and a kept sample in every branch): predictions, losses and gradients against the oracle."""
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", chain)
    fx, c, model = _cuda_small(golden_dir, dev, 0.5)
    table = _pattern_scales(model, c["B"], dev)
    assert len(table) == 3 + 4 * 1
    _pin_by_prefix(monkeypatch, table)
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))
    model.generate_random_masks = lambda *a, **k: triple
    preds, masks = model({k: v.to(dev) for k, v in fx["inputs"].items()}, num_encoded_tokens=triple[1].shape[1], alphas=1.0)
    fns = _loss_modules()
    losses = {t: fns[t](preds[t].float(), fx["inputs"]["rgb" if t == "norm_rgb" else t].to(dev),
                        mask=masks.get("rgb" if t == "norm_rgb" else t)) for t in preds}
    sum(losses.values()).backward()
    torch.cuda.synchronize()

    cfg, p, train = _oracle(c)
    cpu_table = {k: (a.cpu(), m.cpu()) for k, (a, m) in table.items()}
    with applied(cpu_table):
        o_losses, o_preds = O.step_losses(p, fx["inputs"], cfg, fx["task_masks"], fx["ids_keep"], fx["ids_restore"])
    sum(o_losses.values()).backward()
    plain, _ = O.forward({k: v.detach() for k, v in p.items()}, fx["inputs"], cfg, fx["ids_keep"], fx["ids_restore"])
    for k, ref in o_preds.items():
        assert rel_l2(preds[k], ref) < BF16_TOL, (k, rel_l2(preds[k], ref))
    assert max(rel_l2(plain[k], o_preds[k]) for k in o_preds) > 5 * BF16_TOL      # the factors do change the result
    for k, ref in o_losses.items():
        assert abs(float(losses[k]) - float(ref)) < BF16_TOL * abs(float(ref)), (k, float(losses[k]), float(ref))
    named = dict(model.named_parameters())
    used = [k for k in train if train[k].grad is not None]
    _check_grads({k: named[k].grad for k in used}, {k: train[k].grad for k in used})


@pytest.mark.parametrize("task", ["depth", "semseg"])
def test_fp32_adapter_tier_against_oracle(golden_dir, dev, monkeypatch, task):
    """An adapter in the fp32 tier (fp32_output_adapters) with a 2-block decoder_transformer under drop path 0.5, pinned
    factors: prediction, encoder-token gradient and the adapter's parameter gradients against the oracle's decode_task
    run on the same encoder tokens (FP32_TOL)."""
    fx, c, model = _cuda_small(golden_dir, dev, 0.5)
    table = _pattern_scales(model, c["B"], dev)
    _pin_by_prefix(monkeypatch, table)
    cfg, p, train = _oracle(c)
    prefix = "output_adapters.%s." % task
    keys = [k for k in train if k.startswith(prefix)]
    B, n_tok = c["B"], (c["image_size"] // 16) ** 2
    g = torch.Generator().manual_seed(5)
    enc = torch.randn(B, c["num_encoded"] + 1, c["dim"], generator=g) * 0.5
    enc_o = enc.clone().requires_grad_(True)
    counts = {d: n_tok for d in c["in_domains"]}
    hw = (c["image_size"], c["image_size"])
    cpu_table = {k: (a.cpu(), m.cpu()) for k, (a, m) in table.items()}
    with applied(cpu_table):
        ref = O.decode_task(enc_o, p, task, O.DOMAINS[task], cfg, counts, hw, fx["ids_keep"], fx["ids_restore"])
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    info = model.generate_input_info({d: torch.empty(B, n_tok, 0) for d in c["in_domains"]}, hw)
    model.grad_arena(dev).zero_()
    enc_d = enc.to(dev).requires_grad_(True)
    pred = model.output_adapters[task](enc_d, info, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev), fp32=True)
    (pred * w.to(dev)).sum().backward()
    torch.cuda.synchronize()
    named = dict(model.named_parameters())
    total = sum(float(train[k].grad.norm()) ** 2 for k in keys) ** 0.5
    numel = sum(train[k].numel() for k in keys)
    worst = (0.0, None)
    for k in keys:
        r, got = train[k].grad, named[k].grad.detach().float().cpu()
        fair = total * (r.numel() / numel) ** 0.5
        worst = max(worst, (float((got - r).norm()) / max(float(r.norm()), 0.05 * fair), k))
    print("fp32 tier %s with drop path: pred %.2e, d_enc %.2e, worst gradient %.2e (%s)" %
          (task, rel_l2(pred, ref), rel_l2(enc_d.grad, enc_o.grad), worst[0], worst[1]))
    assert rel_l2(pred, ref) < FP32_TOL
    assert rel_l2(enc_d.grad, enc_o.grad) < FP32_TOL
    assert worst[0] < FP32_TOL, worst


def test_multivit_finetuning_shape_against_oracle(dev, monkeypatch):
    """multivit_base, rgb + depth at 224, drop_path_rate 0.1, B = 2, training: encoder tokens (last layer and
    return_all_layers) and the gradients of a weighted sum of them against the oracle with the same factors."""
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    B, S = 2, 224
    ins = {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=S),
           "depth": PatchedInputAdapter(num_channels=1, stride_level=1, patch_size_full=16, image_size=S)}
    torch.manual_seed(0)
    model = multivit_base(ins, None, drop_path_rate=0.1)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for k, v in sd.items():
            if k.endswith(".bias"):
                v.add_(torch.randn(v.shape, generator=g) * 0.05)
    model.load_state_dict(sd)
    model = model.to(dev).train()
    table = {}
    for i, b in enumerate(model.encoder):
        p = Fn.drop_path_prob(b)
        if p > 0:
            inv = float(torch.tensor(1.0) / (1.0 - p))
            a = torch.tensor([inv, inv]); a[i % 2] = 0.0
            m = torch.tensor([inv, inv]); m[(i + 1) % 2] = 0.0
            table["encoder.%d" % i] = (a.to(dev), m.to(dev))
    assert len(table) == 11
    _pin_by_prefix(monkeypatch, table)
    cfg = O.make_config(in_domains=("rgb", "depth"), out_domains=[], extra_norm_pix=False)
    x = O.synthetic_inputs(cfg, B, S, seed=0)
    n_tok = 2 * (S // 16) ** 2
    ids = torch.arange(n_tok).unsqueeze(0).expand(B, -1).contiguous()
    p = {k: v.clone() for k, v in sd.items()}
    train = O.trainable(p)
    for v in train.values():
        v.requires_grad_(True)
    with applied({k: (a.cpu(), m.cpu()) for k, (a, m) in table.items()}):
        _, o_tokens = O.forward(p, x, cfg, ids, ids)
    w = torch.randn(o_tokens.shape, generator=g)
    (o_tokens * w).sum().backward()

    xd = {k: v.to(dev) for k, v in x.items()}
    got = model(xd)
    (got * w.to(dev)).sum().backward()
    torch.cuda.synchronize()
    assert rel_l2(got, o_tokens) < BF16_TOL, rel_l2(got, o_tokens)
    named = dict(model.named_parameters())
    used = [k for k in train if train[k].grad is not None]
    _check_grads({k: named[k].grad for k in used}, {k: train[k].grad for k in used})
    with torch.no_grad():
        layers = model(xd, return_all_layers=True)
    assert len(layers) == 12 and rel_l2(layers[-1], o_tokens) < BF16_TOL


def test_draws_on_device(dev):
    """Drawn factors are exactly 0 or 1/keep with the kept fraction within 4 sigma of keep; the same seed gives the same
    factors and the same outputs; eval() draws nothing and equals p = 0."""
    blocks, arena = _block_stack(dev, n=3)
    _set_drop_path(blocks, 0.5)
    torch.manual_seed(11)
    sc = Fn.drop_path_scales(list(blocks), 8192, dev)
    assert sc[0] is None
    for i in (1, 2):
        keep = 1.0 - Fn.drop_path_prob(blocks[i])
        inv = float(torch.tensor(1.0) / keep)
        for s in sc[i]:
            assert s.device == dev and s.dtype == torch.float32 and s.shape == (8192,)
            assert bool(((s == 0) | (s == inv)).all())
            frac = float((s > 0).float().mean())
            assert abs(frac - keep) < 4 * (keep * (1 - keep) / 8192) ** 0.5, (frac, keep)
    torch.manual_seed(11)
    again = Fn.drop_path_scales(list(blocks), 8192, dev)
    assert all(torch.equal(a, b) for i in (1, 2) for a, b in zip(sc[i], again[i]))

    B, N, D = 4, 37, 128
    g = torch.Generator(device=dev).manual_seed(12)
    x = torch.randn(B, N, D, device=dev, generator=g)
    dout = torch.randn(B, N, D, device=dev, generator=g)
    outs = []
    for _ in range(2):
        torch.manual_seed(13)
        outs.append(_run_stack(blocks, arena, x, dout))
    assert torch.equal(outs[0][0], outs[1][0]) or rel_l2(outs[0][0], outs[1][0]) < 1e-6
    assert rel_l2(outs[0][1], outs[1][1]) < 1e-6
    for k in outs[0][2]:
        assert rel_l2(outs[0][2][k], outs[1][2][k]) < 1e-6, k

    blocks.eval()
    state = torch.cuda.get_rng_state(dev)
    with torch.no_grad():
        y_eval = Fn.block_stack(blocks, x)
    assert torch.equal(torch.cuda.get_rng_state(dev), state)
    _set_drop_path(blocks, 0.0)
    with torch.no_grad():
        y_plain = Fn.block_stack(blocks, x)
    assert torch.equal(y_eval, y_plain)


def _train_step(golden_dir, dev, rate):
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep
    fx, c, model = _cuda_small(golden_dir, dev, rate)
    triple = ({k: v.to(dev) for k, v in fx["task_masks"].items()}, fx["ids_keep"].to(dev), fx["ids_restore"].to(dev))
    model.generate_random_masks = lambda *a, **k: triple
    opt = FlatAdamW(model, lr=1e-3)
    scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
    step = TrainStep(model, _loss_modules(), opt, scaler, num_encoded_tokens=12, loss_sources={"norm_rgb": "rgb"})
    return fx, c, model, opt, step


def test_cuda_graph_pinned_scales_match_eager(golden_dir, dev, monkeypatch):
    """TrainStep.capture with drop path 0.5 and pinned factors: 1 eager warm-up + 3 replays equal 4 eager steps."""
    def run(use_graph):
        fx, c, model, opt, step = _train_step(golden_dir, dev, 0.5)
        _pin_by_prefix(monkeypatch, _pattern_scales(model, c["B"], dev))
        x = {k: v.to(dev) for k, v in fx["inputs"].items()}
        if use_graph:
            step.capture(x, warmup=1)
            assert step.graph is not None
        else:
            step(x)
        losses = [float(step(x)[0]) for _ in range(3)]
        torch.cuda.synchronize()
        return losses, opt.flat_params.clone()

    l_eager, p_eager = run(False)
    l_graph, p_graph = run(True)
    assert all(abs(a - b) <= 2e-3 * abs(a) for a, b in zip(l_eager, l_graph)), (l_eager, l_graph)
    assert rel_l2(p_graph, p_eager) < 1e-3


def test_cuda_graph_live_draws(golden_dir, dev, monkeypatch):
    """Captured with live draws: every replay draws new factors (torch's generator advances inside the graph) and the
    losses stay finite."""
    drawn = []
    real = Fn.drop_path_scales

    def spy(blocks, batch, device):
        out = real(blocks, batch, device)
        drawn.append(out)
        return out
    monkeypatch.setattr(Fn, "drop_path_scales", spy)
    fx, c, model, opt, step = _train_step(golden_dir, dev, 0.5)
    x = {k: v.to(dev) for k, v in fx["inputs"].items()}
    step.capture(x, warmup=1)
    captured = [s for entry in drawn[-5:] for pair in entry if pair is not None for s in pair]   # encoder + 4 decoders
    assert len(captured) == 2 * (3 + 4)
    seen = []
    for _ in range(4):
        loss, _ = step(x)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss))
        seen.append(torch.cat([s.clone() for s in captured]))
    assert all(not torch.equal(seen[i], seen[i + 1]) for i in range(len(seen) - 1))
    inv = {float(torch.tensor(1.0) / (1.0 - Fn.drop_path_prob(b))) for _, blocks in _model_stacks(model) for b in blocks
           if Fn.drop_path_prob(b) > 0}
    assert set(torch.cat(seen).unique().tolist()) <= inv | {0.0}
