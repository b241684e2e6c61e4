"""CPU: the float64 block reference of tests/test_cuda_block.py against torch autograd of the fp32 oracle's block, and its
rounding and deliberately wrong variants against the plain one."""
import pytest
import torch

import block_oracle as BO
import drop_path_oracle as DP

B, N, D, H, HID, EPS = 3, 5, 64, 2, 128, 1e-6


def _inputs(seed=0):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    prm = {"norm1_w": 1 + 0.1 * r(D), "norm1_b": 0.1 * r(D), "norm2_w": 1 + 0.1 * r(D), "norm2_b": 0.1 * r(D),
           "qkv_w": r(3 * D, D) / D ** 0.5, "qkv_b": 0.1 * r(3 * D), "proj_w": r(D, D) / D ** 0.5, "proj_b": 0.1 * r(D),
           "fc1_w": r(HID, D) / D ** 0.5, "fc1_b": 0.1 * r(HID), "fc2_w": r(D, HID) / HID ** 0.5, "fc2_b": 0.1 * r(D)}
    s_attn = torch.tensor([0.0, 1.0, 2.5], dtype=torch.float64)
    s_mlp = torch.tensor([0.0, 1 / 0.9, 1.0], dtype=torch.float64)
    return prm, r(B, N, D), r(B, N, D), (s_attn, s_mlp)


ORACLE_NAMES = {"norm1_w": "b.norm1.weight", "norm1_b": "b.norm1.bias", "qkv_w": "b.attn.qkv.weight",
                "qkv_b": "b.attn.qkv.bias", "proj_w": "b.attn.proj.weight", "proj_b": "b.attn.proj.bias",
                "norm2_w": "b.norm2.weight", "norm2_b": "b.norm2.bias", "fc1_w": "b.mlp.fc1.weight",
                "fc1_b": "b.mlp.fc1.bias", "fc2_w": "b.mlp.fc2.weight", "fc2_b": "b.mlp.fc2.bias"}


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def test_plain_reference_matches_oracle_autograd():
    prm, x, dout, sc = _inputs()
    ref = BO.block_reference(x, prm, H, EPS, dout, round=False, s_attn=sc[0], s_mlp=sc[1])
    p = {ORACLE_NAMES[k]: v.clone().requires_grad_(True) for k, v in prm.items()}
    xl = x.clone().requires_grad_(True)
    out = DP.block(xl, p, "b", H, EPS, sc)
    out.backward(dout)
    assert _rel(ref["x_out"], out.detach()) < 1e-12
    assert _rel(ref["dx_in"], xl.grad) < 1e-12
    for k in BO.PARAMS:
        assert _rel(ref[k], p[ORACLE_NAMES[k]].grad) < 1e-12, k
    # a sample with both factors 0 passes its input and its gradient through unchanged
    assert torch.equal(ref["x_out"][0], x[0]) and torch.equal(ref["dx_in"][0], dout[0])


@pytest.mark.parametrize("fuse", [0, 1])
def test_rounding_reference_differs_by_order_u(fuse):
    prm, x, dout, sc = _inputs()
    plain = BO.block_reference(x, prm, H, EPS, dout, round=False, s_attn=sc[0], s_mlp=sc[1])
    rnd = BO.block_reference(x, prm, H, EPS, dout, fuse_gelu=bool(fuse), s_attn=sc[0], s_mlp=sc[1])
    u = 2.0 ** -8
    # fc2_b is the column sum of s_mlp dx_out taken before any rounding: exact in both
    assert torch.equal(rnd["fc2_b"], plain["fc2_b"])
    for k in ["attn", "mlp", "dx_in"] + [k for k in BO.PARAMS if k != "fc2_b"]:
        ref = plain[k] if k != "dx_in" else plain[k] - dout
        got = rnd[k] if k != "dx_in" else rnd[k] - dout
        e = _rel(got, ref)
        assert u / 64 < e < 16 * u, (k, e)


def test_gelu_modes_differ():
    prm, x, dout, sc = _inputs()
    a = BO.block_reference(x, prm, H, EPS, dout, fuse_gelu=False)
    b = BO.block_reference(x, prm, H, EPS, dout, fuse_gelu=True)
    assert not torch.equal(a["mlp"], b["mlp"]) and not torch.equal(a["fc1_b"], b["fc1_b"])


@pytest.mark.parametrize("mutate", BO.MUTATIONS)
def test_mutations_differ(mutate):
    prm, x, dout, sc = _inputs()
    good = BO.block_reference(x, prm, H, EPS, dout, s_attn=sc[0], s_mlp=sc[1])
    bad = BO.block_reference(x, prm, H, EPS, dout, s_attn=sc[0], s_mlp=sc[1], mutate=mutate)
    assert _rel(bad["x_out"] - x, good["x_out"] - x) > 0.05, mutate


def test_chain_matches_single_blocks_and_handoff_mutations_differ():
    """The chained reference equals block_reference applied block by block (forward values, then the gradient handed
    down from block to block); the two hand-off variants change only the fc2 bias gradient of the blocks below the top."""
    prms = [_inputs(s)[0] for s in range(3)]
    _, x, dout, sc = _inputs()
    scales = [sc, (sc[1], sc[0]), None]
    chain = BO.chain_reference(x, prms, H, EPS, dout, scales=scales)
    xin = x
    for i in range(3):
        s = scales[i] or (None, None)
        one = BO.block_reference(xin, prms[i], H, EPS, chain[i]["dx_in"] * 0, s_attn=s[0], s_mlp=s[1])
        assert _rel(one["x_out"], chain[i]["x_out"]) < 1e-15
        xin = one["x_out"]
    for i in reversed(range(3)):
        s = scales[i] or (None, None)
        d = dout if i == 2 else chain[i + 1]["dx_in"]
        one = BO.block_reference(chain[i]["x"], prms[i], H, EPS, d, s_attn=s[0], s_mlp=s[1])
        for k in ["dx_in"] + BO.PARAMS:
            assert _rel(one[k], chain[i][k]) < 1e-12, (i, k)
    for m in ("handoff_twice", "handoff_missing"):
        bad = BO.chain_reference(x, prms, H, EPS, dout, scales=scales, mutate=m)
        for i in range(3):
            for k in ["x_out", "dx_in"] + BO.PARAMS:
                same = torch.equal(bad[i][k], chain[i][k])
                assert same == (k != "fc2_b" or i == 2), (m, i, k)
