"""CPU: dropout (drop_rate, attn_drop_rate) without a GPU.

1. The oracle with explicit dropout masks (tests/dropout_oracle.py), given the masks recorded from the live reference
   (tests/golden/make_golden_dropout.py), reproduces the reference's encoder tokens and every parameter gradient.
2. The host layer against a stub of the C library: which dropout struct each block call gets, with which rates and seed
   pointers."""
import ctypes

import pytest
import torch

from dropout_oracle import applied
from helpers import load_fixture
from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from oracle import multimae_oracle as O
from test_drop_path_host import _Rec

BLOCK_CALLS = ("mmae_block_forward", "mmae_block_backward")


def _multivit_oracle(c):
    cfg = O.make_config(in_domains=tuple(c["in_domains"]), out_domains=[], extra_norm_pix=False)
    cfg.dim, cfg.depth, cfg.heads = c["dim"], c["depth"], c["heads"]
    cfg.posemb_grid = c["size"] // 16
    return cfg


def test_oracle_dropout_against_reference(golden_dir):
    fx = load_fixture(golden_dir, "dropout.pt")
    c = fx["config"]
    cfg = _multivit_oracle(c)
    p = {k: v.clone() for k, v in fx["state_dict"].items()}
    train = O.trainable(p)
    for v in train.values():
        v.requires_grad_(True)
    table = {prefix: {site: (m, rate) for site, (m, rate) in sites.items()} for prefix, sites in fx["masks"].items()}
    assert all(rate == c["attn_drop_rate"] for _, rate in (s["attn"] for s in table.values()))
    assert all(rate == c["drop_rate"] for s in table.values() for _, rate in (s["proj"], s["mlp"]))
    n_tok = len(c["in_domains"]) * (c["size"] // 16) ** 2
    ids = torch.arange(n_tok).unsqueeze(0).expand(c["B"], -1).contiguous()
    original = O._block
    with applied(table):
        _, tokens = O.forward(p, fx["inputs"], cfg, ids, ids)
    assert O._block is original
    torch.testing.assert_close(tokens, fx["tokens"], rtol=1e-4, atol=1e-5)
    (tokens * fx["weight"]).sum().backward()
    assert set(fx["grads"]) == {k for k, v in train.items() if v.grad is not None}
    for k, ref in fx["grads"].items():
        err = float((train[k].grad - ref).norm())
        assert err <= 1e-4 * float(ref.norm()) + 1e-6, (k, err, float(ref.norm()))     # fp32 summation order
    # the fixture does exercise dropout: without the masks the tokens differ
    _, plain = O.forward({k: v.detach() for k, v in p.items()}, fx["inputs"], cfg, ids, ids)
    assert not torch.allclose(plain, fx["tokens"], rtol=1e-3, atol=1e-4)


# ------------------------------------------------------------------------------------------------- host layer (stub)
@pytest.fixture()
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(L, "lib", lambda: r)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    return r


def _stack(n=3, dim=128, drop=0.0, attn_drop=0.0):
    from multimae_b200.multimae_utils import Block
    blocks = torch.nn.Sequential(*[Block(dim, 2, qkv_bias=True, drop=drop, attn_drop=attn_drop) for _ in range(n)])
    arena = Fn.GradArena(list(blocks.named_parameters()), torch.device("cpu"))
    for i, b in enumerate(blocks):
        b.bind(arena, "%d." % i)
    return blocks


def _pinned_seeds(monkeypatch):
    """Substitutes dropout_seeds: a distinct recognisable 0-dim int64 tensor per block that drops something."""
    made = {}

    def fake(blocks, device):
        out = []
        for b in blocks:
            if not any(p > 0 for p in Fn.dropout_rates(b)):
                out.append(None)
                continue
            made[id(b)] = torch.tensor(1000 + len(made), dtype=torch.int64)
            out.append(made[id(b)])
        return out
    monkeypatch.setattr(Fn, "dropout_seeds", fake)
    return made


def _drop_struct(args):
    d = args[14]._obj
    assert isinstance(d, L.BlockDropout)
    return (d.attn_p, d.proj_p, d.mlp_p, d.seed, d.prev_mlp_p, d.prev_seed)


@pytest.mark.parametrize("chain", [True, False])
def test_block_calls_carry_dropout_rates_and_seeds(rec, monkeypatch, chain):
    """Rates > 0 in training: every block call carries a dropout struct with its modules' rates and its seed, forward and
    backward with the same seed pointer; chained, block i+1 also gets block i's mlp rate and seed as prev_*."""
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", chain)
    blocks = _stack(drop=0.25, attn_drop=0.4).train()
    blocks[1].attn.proj_drop.p = 0.125                       # the three rates are read per module
    seeds = _pinned_seeds(monkeypatch)
    x = torch.randn(2, 5, 128, requires_grad=True)
    Fn.block_stack(blocks, x).sum().backward()
    assert all(a[14] is not None for n, a in rec.calls if n in BLOCK_CALLS)
    fwd = [_drop_struct(a) for n, a in rec.calls if n == "mmae_block_forward"]
    bwd = [_drop_struct(a) for n, a in rec.calls if n == "mmae_block_backward"][::-1]     # issued for blocks 2..0
    assert len(fwd) == len(bwd) == 3 and len(seeds) == 3
    for i, b in enumerate(blocks):
        own = seeds[id(b)].data_ptr()
        prev = (0.25, seeds[id(blocks[i - 1])].data_ptr()) if chain and i > 0 else (0.0, None)
        want = (0.4, 0.125 if i == 1 else 0.25, 0.25, own) + prev
        assert fwd[i] == pytest.approx(want) and bwd[i] == fwd[i], (i, fwd[i], bwd[i], want)
    # the scale arguments and the rest of each call are those of a call without dropout
    for n, a in rec.calls:
        if n in BLOCK_CALLS:
            assert a[11:14] == (None, None, None)


def test_prev_only_block_gets_dropout_struct(rec, monkeypatch):
    """A block without dropout of its own after one with mlp dropout still gets a dropout struct (chained): it applies the
    previous block's MLP mask to the branch it adds in front of its first LayerNorm."""
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", True)
    blocks = _stack(n=2).train()
    blocks[0].mlp.drop.p = 0.5
    seeds = _pinned_seeds(monkeypatch)
    Fn.block_stack(blocks, torch.randn(2, 5, 128, requires_grad=True)).sum().backward()
    fwd = [_drop_struct(a) for n, a in rec.calls if n == "mmae_block_forward"]
    assert len(fwd) == 2 and list(seeds) == [id(blocks[0])]
    assert fwd[0] == (0.0, 0.0, 0.5, seeds[id(blocks[0])].data_ptr(), 0.0, None)
    assert fwd[1] == (0.0, 0.0, 0.0, None, 0.5, seeds[id(blocks[0])].data_ptr())


def test_eval_no_grad_and_zero_rates_make_todays_calls(rec, monkeypatch):
    """eval() (with or without no_grad) or all rates 0: the block calls get a NULL dropout struct and the same arguments as
    a stack built without dropout; nothing is drawn."""
    monkeypatch.setattr(Fn, "BLOCK_CHAIN", True)
    x = torch.randn(2, 5, 128)

    def calls(blocks, grad):
        rec.calls.clear()
        xi = x.clone().requires_grad_(grad)
        state = torch.get_rng_state()
        if grad:
            Fn.block_stack(blocks, xi).sum().backward()
        else:
            with torch.no_grad():
                Fn.block_stack(blocks, xi)
        assert torch.equal(torch.get_rng_state(), state)
        assert all(a[14] is None for n, a in rec.calls if n in BLOCK_CALLS)
        return [(n, tuple(a[6:14])) for n, a in rec.calls]

    ref_grad, ref_nograd = calls(_stack().train(), True), calls(_stack().eval(), False)
    assert calls(_stack(drop=0.3, attn_drop=0.3).eval(), True) == ref_grad
    assert calls(_stack(drop=0.3, attn_drop=0.3).eval(), False) == ref_nograd
    assert calls(_stack(drop=0.0, attn_drop=0.0).train(), True) == ref_grad
    from multimae_b200.multimae_utils import Block
    rec.calls.clear()
    Block(128, 2, qkv_bias=True, drop=0.2, attn_drop=0.2).eval()(x.clone().requires_grad_(True)).sum().backward()
    assert rec.names().count("mmae_block_forward") == 1 and rec.names().count("mmae_block_backward") == 1
    assert all(a[14] is None for n, a in rec.calls if n in BLOCK_CALLS)


def test_stand_alone_block_draws_its_dropout_seed(rec):
    """A stand-alone Block with dropout in training draws one seed and gives the same pointer to forward and backward."""
    from multimae_b200.multimae_utils import Block
    b = Block(128, 2, qkv_bias=True, drop=0.1, attn_drop=0.2).train()
    b(torch.randn(3, 5, 128, requires_grad=True)).sum().backward()
    (f,) = [_drop_struct(a) for n, a in rec.calls if n == "mmae_block_forward"]
    (g,) = [_drop_struct(a) for n, a in rec.calls if n == "mmae_block_backward"]
    assert f == g and f[:3] == pytest.approx((0.2, 0.1, 0.1)) and f[3] is not None and f[4:] == (0.0, None)


def test_dropout_seeds_one_draw_per_stack(monkeypatch):
    """dropout_seeds: one torch.randint per call, [live blocks] int64 on the device, None for blocks that drop nothing."""
    blocks = _stack(n=4).train()
    blocks[1].attn.attn_drop.p = 0.1
    blocks[3].mlp.drop.p = 0.2
    draws = []
    real = torch.randint

    def counting(*a, **k):
        draws.append((a, k))
        return real(*a, **k)
    monkeypatch.setattr(torch, "randint", counting)
    torch.manual_seed(5)
    seeds = Fn.dropout_seeds(list(blocks), torch.device("cpu"))
    assert len(draws) == 1 and draws[0][1]["dtype"] == torch.int64 and draws[0][0][-1] == (2,)
    assert seeds[0] is None and seeds[2] is None
    assert seeds[1].dtype == torch.int64 and seeds[1].dim() == 0 and seeds[1].data_ptr() != seeds[3].data_ptr()
    assert int(seeds[1]) != int(seeds[3])
    torch.manual_seed(5)
    again = Fn.dropout_seeds(list(blocks), torch.device("cpu"))
    assert int(again[1]) == int(seeds[1]) and int(again[3]) == int(seeds[3])
    draws.clear()
    assert Fn.dropout_seeds(list(blocks.eval()), torch.device("cpu")) == [None] * 4 and not draws


def test_fp32_tier_training_with_dropout_raises(rec):
    blocks = _stack(n=2, drop=0.1).train()
    x = torch.randn(2, 5, 128, requires_grad=True)
    with pytest.raises(NotImplementedError, match="fp32 tier"):
        Fn.block_stack(blocks, x, fp32=True)
    assert not rec.calls
    Fn.block_stack(blocks.eval(), x, fp32=True).sum().backward()
    assert rec.names().count("mmae_block_f32_forward") == 2 and rec.names().count("mmae_block_f32_backward") == 2


def test_modules_accept_dropout_with_reference_state_dict(golden_dir):
    """multivit_base(drop_rate, attn_drop_rate) builds; the nn.Dropout modules carry the rates and add no state; a small
    MultiViT with dropout has exactly the reference's state_dict keys (the fixture's); CrossAttention still refuses."""
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import MultiViT, multivit_base
    from multimae_b200.multimae_utils import CrossAttention

    def ins(size):
        return {"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=size),
                "depth": PatchedInputAdapter(num_channels=1, stride_level=1, patch_size_full=16, image_size=size)}
    m = multivit_base(ins(224), None, drop_rate=0.1, attn_drop_rate=0.1)
    plain = multivit_base(ins(224), None)
    assert list(m.state_dict()) == list(plain.state_dict())
    blk = m.encoder[3]
    assert (blk.attn.attn_drop.p, blk.attn.proj_drop.p, blk.mlp.drop.p) == (0.1, 0.1, 0.1)
    assert repr(blk.mlp.drop) == "Dropout(p=0.1, inplace=False)"
    c = load_fixture(golden_dir, "dropout.pt")["config"]
    small = MultiViT(input_adapters=ins(c["size"]), output_adapters=None, num_global_tokens=1, dim_tokens=c["dim"],
                     depth=c["depth"], num_heads=c["heads"], drop_rate=c["drop_rate"], attn_drop_rate=c["attn_drop_rate"])
    assert list(small.state_dict()) == list(load_fixture(golden_dir, "dropout.pt")["state_dict"])
    with pytest.raises(AssertionError, match="no dropout"):
        CrossAttention(256, 8, qkv_bias=True, attn_drop=0.1)


def test_block_dropout_struct_matches_header(tmp_path):
    """mmae_block_dropout (declared with a separate struct tag) against its ctypes twin: sizeof and every field offset."""
    import os
    import shutil
    import subprocess
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    header = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "multimae_b200.h")
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "%s"' % header, "int main(void) {",
             '  printf("sizeof %zu\\n", sizeof(mmae_block_dropout));']
    for f, _ in L.BlockDropout._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(mmae_block_dropout, %s));' % (f, f))
    lines += ["  return 0;", "}"]
    (tmp_path / "d.c").write_text("\n".join(lines))
    subprocess.run([gcc, "-std=c99", "-o", str(tmp_path / "d"), str(tmp_path / "d.c")], check=True, capture_output=True)
    out = subprocess.run([str(tmp_path / "d")], check=True, capture_output=True, text=True).stdout.split("\n")
    for line in filter(None, out):
        k, v = line.split()
        mine = ctypes.sizeof(L.BlockDropout) if k == "sizeof" else getattr(L.BlockDropout, k).offset
        assert mine == int(v), (k, mine, v)
