"""GPU: dropout inside the fused block and attention kernels (their dropout arguments and mmae_dropout_keep_mask).

The masks of a run are materialised from the seeds it drew (functional.dropout_seeds, spied on) by mmae_dropout_keep_mask,
which uses the kernels' own generator, and handed to the fp32 oracle with explicit masks (tests/dropout_oracle.py).
Nothing here reads the reference checkout."""
import math

import pytest
import torch

from dropout_oracle import block as oracle_block
from helpers import rel_l2
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from test_cuda_drop_path import BF16_TOL, GRAD_TOL

pytestmark = pytest.mark.gpu

SITES = {"attn": 0, "proj": 1, "mlp": 2}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def keep_mask(seed, site, rows, cols, p):
    """[rows, cols] bool keep mask of `site` for the 0-dim int64 device tensor `seed`."""
    out = torch.empty((rows, cols), dtype=torch.uint8, device=seed.device)
    L.check(L.lib().mmae_dropout_keep_mask(seed.data_ptr(), site, rows, cols, p, out.data_ptr(), L.current_stream()),
            "mmae_dropout_keep_mask")
    return out.bool()


def _spy_seeds(monkeypatch):
    drawn = []
    real = Fn.dropout_seeds

    def spy(blocks, device):
        out = real(blocks, device)
        drawn.append(out)
        return out
    monkeypatch.setattr(Fn, "dropout_seeds", spy)
    return drawn


def _blocks(dev, n, dim, heads, drop, attn_drop, seed=0):
    from multimae_b200.multimae_utils import Block
    torch.manual_seed(seed)
    blocks = torch.nn.Sequential(*[Block(dim, heads, qkv_bias=True, drop=drop, attn_drop=attn_drop) for _ in range(n)])
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


def _run(blocks, arena, x, dout):
    arena.zero_()
    xi = x.clone().requires_grad_(True)
    out = Fn.block_stack(blocks, xi)
    out.backward(dout)
    torch.cuda.synchronize()
    return out.detach().clone(), xi.grad.clone(), {k: v.clone() for k, v in arena.views.items()}


def _oracle_stack(blocks, seeds, x, dout):
    """fp32 CPU oracle of the stack with the masks of `seeds`; returns output, dx and the parameter gradients."""
    B, N, D = x.shape
    p = {k: v.detach().float().cpu().clone().requires_grad_(True) for k, v in blocks.named_parameters()}
    xo = x.cpu().clone().requires_grad_(True)
    h = xo
    for i, (b, s) in enumerate(zip(blocks, seeds)):
        H = b.num_heads
        rates = Fn.dropout_rates(b)
        sites = {}
        if s is not None:
            sites["attn"] = (keep_mask(s, 0, B * H * N, N, rates[0]).reshape(B, H, N, N).cpu(), rates[0])
            sites["proj"] = (keep_mask(s, 1, B * N, D, rates[1]).reshape(B, N, D).cpu(), rates[1])
            sites["mlp"] = (keep_mask(s, 2, B * N, D, rates[2]).reshape(B, N, D).cpu(), rates[2])
        h = oracle_block(h, p, "%d" % i, H, b.norm1.eps, sites)
    h.backward(dout.cpu())
    return h.detach(), xo.grad, {k: v.grad for k, v in p.items()}


@pytest.mark.parametrize("chain", [True, False])
@pytest.mark.parametrize("heads", [2, 4])                 # head_dim 64 and 32 at D = 128
@pytest.mark.parametrize("N", [197, 577])                 # fused attention backward (<= 256 keys) and dQ + dK/dV
def test_block_stack_against_oracle(dev, monkeypatch, chain, heads, N):
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", chain)
    drawn = _spy_seeds(monkeypatch)
    B, D = 2, 128
    blocks, arena = _blocks(dev, 3, D, heads, drop=0.2, attn_drop=0.3)
    blocks[1].mlp.drop.p = 0.5                                   # rates are per module and per site
    g = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(B, N, D, device=dev, generator=g)
    dout = torch.randn(B, N, D, device=dev, generator=g)
    out, dx, grads = _run(blocks, arena, x, dout)
    seeds = drawn[-1]
    assert all(s is not None for s in seeds)
    ref_out, ref_dx, ref_grads = _oracle_stack(blocks, seeds, x, dout)
    assert rel_l2(out, ref_out) < BF16_TOL, rel_l2(out, ref_out)
    assert rel_l2(dx, ref_dx) < GRAD_TOL, rel_l2(dx, ref_dx)
    for k, ref in ref_grads.items():
        assert rel_l2(grads[k], ref) < GRAD_TOL, (k, rel_l2(grads[k], ref))
    # the masks matter: the oracle without them is far off
    plain = x.cpu()
    p = {k: v.detach().float().cpu() for k, v in blocks.named_parameters()}
    for i, b in enumerate(blocks):
        plain = oracle_block(plain, p, "%d" % i, heads, b.norm1.eps)
    assert rel_l2(plain, ref_out) > 5 * BF16_TOL


def _attn_inputs(dev, B, H, N, dh, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    qkv = (torch.randn(B * N, 3 * H * dh, device=dev, generator=g)).bfloat16()
    d_o = torch.randn(B * N, H * dh, device=dev, generator=g).bfloat16()
    return qkv, d_o


def _attn_call(qkv, d_o, B, H, N, dh, p, seed):
    lib, D = L.lib(), H * dh
    dev = qkv.device
    o = torch.empty(B * N, D, dtype=torch.bfloat16, device=dev)
    lse = torch.empty(B, H, N, device=dev)
    delta = torch.empty(B, H, N, device=dev)
    dqkv = torch.empty_like(qkv)
    sc, st = dh ** -0.5, L.current_stream()
    q, k, v = qkv.data_ptr(), qkv[:, D:].data_ptr(), qkv[:, 2 * D:].data_ptr()
    L.check(lib.mmae_attention_forward(q, 3 * D, k, 3 * D, v, 3 * D, o.data_ptr(), D, lse.data_ptr(), B, H, N, N, dh, sc,
                                       p, L.ptr(seed), st), "mmae_attention_forward")
    L.check(lib.mmae_attention_backward(q, 3 * D, k, 3 * D, v, 3 * D, o.data_ptr(), D, d_o.data_ptr(), D, lse.data_ptr(),
                                        delta.data_ptr(), dqkv.data_ptr(), 3 * D, dqkv[:, D:].data_ptr(), 3 * D,
                                        dqkv[:, 2 * D:].data_ptr(), 3 * D, B, H, N, N, dh, sc, p, L.ptr(seed), st),
            "mmae_attention_backward")
    torch.cuda.synchronize()
    return o, dqkv


@pytest.mark.parametrize("N", [197, 577])
@pytest.mark.parametrize("dh", [32, 64])
def test_attention_dropout_against_oracle_and_tc_switch(dev, N, dh):
    """mmae_attention_forward / _backward with dropout against the fp32 attention with the keep mask; with the wgmma kernels selected
    (MMAE_ATTN_TC bits) the results are bit for bit those of the mma.sync kernels: dropout always runs on the latter."""
    B, H, p = 2, 2, 0.3
    qkv, d_o = _attn_inputs(dev, B, H, N, dh)
    seed = torch.tensor(123456789012345, dtype=torch.int64, device=dev)
    lib = L.lib()
    try:
        lib.mmae_attention_set_tc(0)
        o0, d0 = _attn_call(qkv, d_o, B, H, N, dh, p, seed)
        lib.mmae_attention_set_tc(1 | 2 | 4 | 8 | 32 | 64 | 128)
        o1, d1 = _attn_call(qkv, d_o, B, H, N, dh, p, seed)
    finally:
        lib.mmae_attention_set_tc(-1)
    assert torch.equal(o0, o1) and torch.equal(d0, d1)
    D = H * dh
    m = keep_mask(seed, SITES["attn"], B * H * N, N, p).reshape(B, H, N, N).cpu()
    x = qkv.float().cpu().reshape(B, N, 3 * D).requires_grad_(True)
    q, k, v = x.chunk(3, dim=-1)
    from oracle import multimae_oracle as O
    q, k, v = O._heads(q, H), O._heads(k, H), O._heads(v, H)
    w = torch.softmax((q @ k.transpose(-2, -1)) * dh ** -0.5, dim=-1) * m / (1 - p)
    ref = (w @ v).transpose(1, 2).reshape(B, N, D)
    ref.backward(d_o.float().cpu().reshape(B, N, D))
    assert rel_l2(o0.float().cpu(), ref.reshape(B * N, D)) < BF16_TOL
    assert rel_l2(d0.float().cpu(), x.grad.reshape(B * N, 3 * D)) < GRAD_TOL
    # p = 1: everything dropped - zero output and zero gradients
    o, d = _attn_call(qkv, d_o, B, H, N, dh, 1.0, seed)
    assert not o.float().abs().max() and not d.float().abs().max()


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_mask_statistics(dev, p):
    """Keep fraction within 5 sigma of 1 - p per site; distinct sites, seeds give different masks; a seed gives the same
    mask every time; the attention site's masks of the forward and backward match the ones the kernels applied."""
    rows, cols = 4096, 197
    seeds = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device=dev)
    masks = {}
    for j in range(2):
        for name, site in SITES.items():
            m = keep_mask(seeds[j], site, rows, cols, p)
            frac = float(m.float().mean())
            n = rows * cols
            assert abs(frac - (1 - p)) < 5 * math.sqrt(p * (1 - p) / n), (name, frac, p)
            masks[(j, site)] = m
            assert torch.equal(m, keep_mask(seeds[j], site, rows, cols, p))
    vals = list(masks.values())
    assert all(not torch.equal(a, b) for i, a in enumerate(vals) for b in vals[i + 1:])
    assert bool(keep_mask(seeds[0], 1, rows, cols, 0.0).all()) and not bool(keep_mask(seeds[0], 1, rows, cols, 1.0).any())


def test_rate_one_branches_give_zero(dev, monkeypatch):
    """proj and mlp rates 1: both residual branches are zero, so the block is the identity in forward and backward and
    the weights of the branches get zero gradients."""
    blocks, arena = _blocks(dev, 2, 128, 2, drop=1.0, attn_drop=0.0)
    g = torch.Generator(device=dev).manual_seed(4)
    x = torch.randn(2, 197, 128, device=dev, generator=g)
    dout = torch.randn(2, 197, 128, device=dev, generator=g)
    out, dx, grads = _run(blocks, arena, x, dout)
    assert torch.equal(out, x) and torch.equal(dx, dout)
    for k, v in grads.items():
        assert not v.abs().max(), k


def test_same_manual_seed_same_results(dev):
    blocks, arena = _blocks(dev, 3, 128, 2, drop=0.1, attn_drop=0.1)
    g = torch.Generator(device=dev).manual_seed(6)
    x = torch.randn(2, 197, 128, device=dev, generator=g)
    dout = torch.randn(2, 197, 128, device=dev, generator=g)
    runs = []
    for s in (7, 7, 8):
        torch.manual_seed(s)
        runs.append(_run(blocks, arena, x, dout))
    a, b, c = runs
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in a[2]:
        assert rel_l2(a[2][k], b[2][k]) < 1e-6, k                 # split-K reduce-add order of the weight gradients
    assert not torch.equal(a[0], c[0])


def _train_step(golden_dir, dev, rate):
    from test_cuda_drop_path import _train_step as dp_train_step
    fx, c, model, opt, step = dp_train_step(golden_dir, dev, 0.0)
    for b in model.encoder:
        b.attn.attn_drop.p = b.attn.proj_drop.p = b.mlp.drop.p = rate
    return fx, c, model, opt, step


def test_cuda_graph_pinned_seeds_match_eager(golden_dir, dev, monkeypatch):
    """TrainStep.capture with dropout 0.2 in the encoder and pinned seeds: 1 eager warm-up + 3 replays equal 4 eager steps."""
    def run(use_graph):
        fx, c, model, opt, step = _train_step(golden_dir, dev, 0.2)
        fixed = {}

        def pinned(blocks, device):         # made in the eager warm-up, reused (no host copy) while capturing
            out = []
            for b in blocks:
                if not any(p > 0 for p in Fn.dropout_rates(b)):
                    out.append(None)
                    continue
                if id(b) not in fixed:
                    fixed[id(b)] = torch.tensor(1000 + len(fixed), dtype=torch.int64, device=device)
                out.append(fixed[id(b)])
            return out
        monkeypatch.setattr(Fn, "dropout_seeds", pinned)
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
    """Captured with live draws: every replay draws new seeds inside the graph and the losses stay finite."""
    drawn = _spy_seeds(monkeypatch)
    fx, c, model, opt, step = _train_step(golden_dir, dev, 0.2)
    x = {k: v.to(dev) for k, v in fx["inputs"].items()}
    step.capture(x, warmup=1)
    captured = [s for entry in drawn for s in entry if s is not None][-len(model.encoder):]   # the capture's draw
    assert len(captured) == len(model.encoder)
    seen = []
    for _ in range(3):
        loss, _ = step(x)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss))
        seen.append(torch.stack([s.clone() for s in captured]))
    assert all(not torch.equal(seen[i], seen[i + 1]) for i in range(len(seen) - 1))


def test_finetune_cls_sequence_with_dropout(dev):
    """The run_finetuning_cls.py train_one_epoch sequence of test_cuda_cls_head with --drop 0.1 --attn_drop_rate 0.1:
    finite losses that fall on a fixed batch."""
    from multimae_b200 import multimae as mm
    from multimae_b200 import overlay
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from test_cls_head_host import _build
    from test_cuda_cls_head import _mixup, _param_groups
    from cls_head_oracle import soft_target_ce
    old = mm.AUTO_OWN_GRADIENTS
    mm.AUTO_OWN_GRADIENTS = True
    try:
        torch.manual_seed(0)
        C, B, update_freq = 37, 8, 2
        model = _build(num_classes=C, mean_pool=True, drop_path_rate=0.1, size=64)
        for blk in model.encoder:
            blk.attn.attn_drop.p, blk.attn.proj_drop.p, blk.mlp.drop.p = 0.1, 0.1, 0.1
        model = overlay._IdentityDDP(model.to(dev), device_ids=[0])
        optimizer = torch.optim.AdamW(_param_groups(model.module, 0.05, 0.65), lr=1e-3)
        loss_scaler = NativeScalerWithGradNormCount()
        g = torch.Generator().manual_seed(3)
        data = [({"rgb": torch.randn(B, 3, 64, 64, generator=g), "depth": torch.randn(B, 1, 64, 64, generator=g)},
                 torch.randint(0, C, (B,), generator=g)) for _ in range(update_freq)]
        model.train(True)
        optimizer.zero_grad()
        losses = []
        for it in range(10 * update_freq):
            samples, targets = data[it % update_freq]
            samples = {k: v.to(dev) for k, v in samples.items()}
            targets = targets.to(dev)
            mixed = {}
            for k, v in samples.items():
                mixed[k], soft = _mixup(v, targets, C, lam=0.7)
            with torch.cuda.amp.autocast():
                loss = soft_target_ce(model(mixed)["cls"], soft)
            losses.append(loss.item())
            assert math.isfinite(losses[-1])
            loss_scaler(loss / update_freq, optimizer, clip_grad=1.0, parameters=model.parameters(), create_graph=False,
                        update_grad=(it + 1) % update_freq == 0)
            if (it + 1) % update_freq == 0:
                optimizer.zero_grad()
        assert sum(losses[-update_freq:]) < 0.9 * sum(losses[:update_freq]), losses
    finally:
        mm.AUTO_OWN_GRADIENTS = old
