"""CPU: stochastic depth (drop path) without a GPU.

1. The oracle with stochastic depth (tests/drop_path_oracle.py), given the keep vectors recorded from the live reference
   (tests/golden/make_golden_drop_path.py), reproduces the reference's predictions, losses and parameter gradients.
2. The host layer against a stub of the C library: which entry points run and which scale pointers they receive."""
import pytest
import torch

from drop_path_oracle import applied
from helpers import load_fixture
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from oracle import multimae_oracle as O


def _cfg_from_fixture(fx):
    c = fx["config"]
    cfg = O.make_config(in_domains=tuple(c["in_domains"]), out_domains=c.get("out_domains"))
    cfg.dim, cfg.depth, cfg.heads = c["dim"], c["depth"], c["heads"]
    cfg.dec_dim, cfg.dec_depth, cfg.dec_heads = c["dec_dim"], c["dec_depth"], c["dec_heads"]
    cfg.posemb_grid = c["image_size"] // 16
    return cfg


def test_oracle_drop_path_against_reference(golden_dir):
    fx = load_fixture(golden_dir, "drop_path.pt")
    cfg = _cfg_from_fixture(fx)
    assert cfg.depth == 3 and cfg.dec_depth == 2
    p = {k: v.clone() for k, v in fx["state_dict"].items()}
    train = O.trainable(p)
    for v in train.values():
        v.requires_grad_(True)
    scales = {k: (a / (1 - fx["drop_prob"][k]), m / (1 - fx["drop_prob"][k])) for k, (a, m) in fx["keep"].items()}
    assert "encoder.0" not in scales and len(scales) == 2 + 4          # block 0 of every stack has p = 0
    original = O._block
    with applied(scales):
        losses, preds = O.step_losses(p, fx["inputs"], cfg, fx["task_masks"], fx["ids_keep"], fx["ids_restore"])
    assert O._block is original
    for k, ref in fx["preds"].items():
        torch.testing.assert_close(preds[k], ref, rtol=1e-4, atol=1e-5)
    for k, ref in fx["losses"].items():
        torch.testing.assert_close(losses[k], ref, rtol=1e-5, atol=1e-6)
    sum(losses.values()).backward()
    assert set(fx["grads"]) == {k for k, v in train.items() if v.grad is not None}
    for k, ref in fx["grads"].items():
        torch.testing.assert_close(train[k].grad, ref, rtol=2e-4, atol=2e-6, msg=lambda m, k=k: "%s: %s" % (k, m))
    # the fixture does exercise stochastic depth: without the recorded factors the predictions differ
    plain, _ = O.forward({k: v.detach() for k, v in p.items()}, fx["inputs"], cfg, fx["ids_keep"], fx["ids_restore"])
    assert any(not torch.allclose(plain[k], fx["preds"][k], rtol=1e-3, atol=1e-4) for k in plain)


class _Rec:
    """Stub library: records (name, args) of every call; x_mid lives 64 bytes into a block's saved buffer."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        res, argtypes = L.SIGNATURES[name]

        def fn(*args):
            assert len(args) == len(argtypes), name
            self.calls.append((name, args))
            if name.endswith("_bytes"):
                return 4096
            if name == "mmae_block_saved_x_mid":
                return args[0] + 64
            if name == "mmae_abi_version":
                return L.ABI_VERSION
            if name == "mmae_last_error":
                return b""
            return 0
        return fn

    def names(self):
        return [n for n, _ in self.calls]


@pytest.fixture()
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(L, "lib", lambda: r)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    return r


def _stack(n=4, dim=128, rate=0.3):
    from multimae_b200.multimae_utils import Block
    dpr = [v.item() for v in torch.linspace(0, rate, n)]
    blocks = torch.nn.Sequential(*[Block(dim, 2, qkv_bias=True, drop_path=dpr[i]) for i in range(n)])
    arena = Fn.GradArena(list(blocks.named_parameters()), torch.device("cpu"))
    for i, b in enumerate(blocks):
        b.bind(arena, "%d." % i)
    return blocks


def _pinned(monkeypatch, B):
    """Substitutes drop_path_scales: distinct recognisable [B] tensors per block (None where nothing drops)."""
    made = {}

    def fake(blocks, batch, device):
        assert batch == B
        out = []
        for b in blocks:
            if Fn.drop_path_prob(b) == 0.0:
                out.append(None)
                continue
            pair = (torch.full((batch,), 2.0), torch.full((batch,), 3.0))
            made[id(b)] = pair
            out.append(pair)
        return out
    monkeypatch.setattr(Fn, "drop_path_scales", fake)
    return made


@pytest.mark.parametrize("chain", [True, False])
def test_drop_path_scale_arguments(rec, monkeypatch, chain):
    """p > 0 in training: every block of the call carries its factors; block i gets its own (s_attn, s_mlp) and - chained -
    block i-1's s_mlp as the previous block's scale, forward and backward.  Block 0 (p = 0) has no own scales: unchained,
    all its scale arguments are None."""
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", chain)
    B = 3
    blocks = _stack().train()
    made = _pinned(monkeypatch, B)
    x = torch.randn(B, 5, 128, requires_grad=True)
    out = Fn.block_stack(blocks, x)
    out.sum().backward()
    fwd = [a for n, a in rec.calls if n == "mmae_block_forward"]
    bwd = [a for n, a in rec.calls if n == "mmae_block_backward"][::-1]      # issued for blocks 3..0
    assert len(made) == 3 and len(fwd) == len(bwd) == 4
    for i, b in enumerate(blocks):
        own = made.get(id(b))
        prev = made.get(id(blocks[i - 1])) if (chain and i > 0) else None
        want = (None, None) if own is None else (own[0].data_ptr(), own[1].data_ptr())
        want_prev = None if prev is None else prev[1].data_ptr()
        # forward args: ..., eps (10), s_attn (11), s_mlp (12), s_prev (13); backward: ..., hidden (10), 11, 12, 13
        assert fwd[i][11:14] == want + (want_prev,), i
        assert bwd[i][11:14] == want + (want_prev,), i
        if own is not None:
            assert own[0].numel() == own[1].numel() == B and own[0].dtype == torch.float32
    if chain:
        assert fwd[0][1] is None and all(f[1] is not None for f in fwd[1:])    # x_add: chained hand-off
    else:
        assert all(f[1] is None and f[4] is None for f in fwd[1:])              # each block adds its own MLP branch


def test_eval_and_zero_rate_pass_no_scales(rec, monkeypatch):
    """eval() or drop_path = 0: the same call sequence as a stack without DropPath modules; nothing is drawn."""
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", True)
    x = torch.randn(2, 5, 128)
    stacks = (_stack(rate=0.0).train(), _stack(rate=0.3).eval())
    state = torch.get_rng_state()
    seqs, chained, scale_args = [], [], []
    block_calls = ("mmae_block_forward", "mmae_block_backward")
    for blocks in stacks:
        rec.calls.clear()
        xi = x.clone().requires_grad_(True)
        Fn.block_stack(blocks, xi).sum().backward()
        seqs.append(rec.names())
        chained.append(any(a[1] is not None for n, a in rec.calls if n == "mmae_block_forward"))     # x_add handed over
        scale_args += [a[11:14] for n, a in rec.calls if n in block_calls]
    assert seqs[0] == seqs[1] and all(chained)
    assert torch.equal(torch.get_rng_state(), state)
    from multimae_b200.multimae_utils import Block
    rec.calls.clear()
    b = Block(128, 2, qkv_bias=True, drop_path=0.2).eval()
    b(x.clone().requires_grad_(True)).sum().backward()
    assert rec.names().count("mmae_block_forward") == 1 and rec.names().count("mmae_block_backward") == 1
    scale_args += [a[11:14] for n, a in rec.calls if n in block_calls]
    assert len(scale_args) == 2 * 2 * 4 + 2 and all(s == (None, None, None) for s in scale_args)


def test_stand_alone_block_with_drop_path_trains(rec):
    """A stand-alone Block with drop_path > 0 in training no longer raises; it draws its two [B] factors itself."""
    from multimae_b200.multimae_utils import Block, DropPath
    b = Block(128, 2, qkv_bias=True, drop_path=0.25).train()
    assert repr(b.drop_path) == "DropPath(p=0.25)" and not list(b.drop_path.state_dict())
    x = torch.randn(4, 5, 128, requires_grad=True)
    b(x).sum().backward()
    (f,) = [a for n, a in rec.calls if n == "mmae_block_forward"]
    (g,) = [a for n, a in rec.calls if n == "mmae_block_backward"]
    assert f[11] is not None and f[12] is not None and f[13] is None and f[11:14] == g[11:14]
    with pytest.raises(NotImplementedError, match="inside Block"):
        DropPath(0.25).train()(x)
    assert DropPath(0.25).eval()(x) is x


def test_drop_path_scales_values():
    """drop_path_scales on CPU tensors (the draw itself is plain torch): exactly 0 or 1/keep, attention and MLP pairs for
    the blocks with p > 0 only, from one generator sequence."""
    blocks = _stack(n=3, rate=0.5).train()
    torch.manual_seed(3)
    sc = Fn.drop_path_scales(list(blocks), 4096, torch.device("cpu"))
    assert sc[0] is None
    for i, keep in ((1, 0.75), (2, 0.5)):
        for s in sc[i]:
            vals = set(s.unique().tolist())
            assert vals <= {0.0, float(torch.tensor(1.0) / keep)} and len(vals) == 2      # fp32 1/keep
            frac = float((s > 0).float().mean())
            assert abs(frac - keep) < 4 * (keep * (1 - keep) / 4096) ** 0.5
    torch.manual_seed(3)
    again = Fn.drop_path_scales(list(blocks), 4096, torch.device("cpu"))
    assert all(torch.equal(a, b) for i in (1, 2) for a, b in zip(sc[i], again[i]))
    assert all(s is None for s in Fn.drop_path_scales(list(blocks.eval()), 4, torch.device("cpu")))


def test_model_paths_pass_drop_path_scales(rec, monkeypatch):
    """MultiMAE (encoder + every decoder_transformer, one adapter in the fp32 tier) and MultiViT with return_all_layers run
    stochastic depth through the block calls' scale arguments when drop_path > 0 in training."""
    from multimae_b200.multimae_utils import DropPath
    from test_host_api import _build
    model = _build(depth=3, dec_depth=2).train()
    for blocks in [model.encoder] + [ad.decoder_transformer for ad in model.output_adapters.values()]:
        for i, b in enumerate(blocks):
            if i > 0:
                b.drop_path = DropPath(0.1 * i)
    x = {"rgb": torch.randn(2, 3, 64, 64), "depth": torch.randn(2, 1, 64, 64),
         "semseg": torch.randint(0, 133, (2, 16, 16))}
    preds, masks = model(x, num_encoded_tokens=12, fp32_output_adapters=["depth"])
    sum(v.float().sum() for v in preds.values()).backward()
    # bf16 tier: the 3 encoder blocks and the 3 two-block decoder transformers; every block with p > 0 (2 + 3 * 1) carries
    # its own factors, and the encoder's block 2 also block 1's
    for name in ("mmae_block_forward", "mmae_block_backward"):
        scales = [a[11:14] for n, a in rec.calls if n == name]
        assert len(scales) == 3 + 3 * 2, name
        assert sum(s[0] is not None and s[1] is not None for s in scales) == 2 + 3 * 1, name
        assert sum(s[0] is None and s[1] is None for s in scales) == 1 + 3 * 1, name
        assert sum(s[2] is not None for s in scales) == 1, name
    # the fp32 tier runs block by block: block 0 (p = 0) without factors, block 1 with them
    for name in ("mmae_block_f32_forward", "mmae_block_f32_backward"):
        scales = sorted((a[8:10] for n, a in rec.calls if n == name), key=lambda s: s[0] is None)
        assert len(scales) == 2 and None not in scales[0] and scales[1] == (None, None), name
