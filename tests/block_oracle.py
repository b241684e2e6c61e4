"""Float64 reference of the transformer block entry points (tests/test_cuda_block.py), store by store.

bf16 tier (mmae_block_forward / mmae_block_backward, modules.cu): float64 with a bf16 rounding wherever the kernels store
a bf16 tensor.  Forward: h1, qkv, o, the attention branch y, h2, z, a (two GELU modes, as dechead_reference) and the MLP
branch y2; the residual sums x_mid = x + s_attn y and x_out = x_mid + s_mlp y2 stay unrounded (fp32 in the kernels).
Backward: every bf16 gradient operand - g = bf16(s_mlp dx_out), dz, dh (fc1's dgrad), g2 = bf16(s_attn dx_mid), d_o,
dqkv, dh (qkv's dgrad) and the hand-off bf16(s_prev dx_in) - and the column sums the bias gradients are formed from:
  * fc2_b, proj_b and the hand-off column sum: of the fp32 scaled gradient BEFORE its bf16 rounding
    (cast_colsum_f32_scaled, layernorm_backward_ex_scaled sum the fp32 value they then pack);
  * fc1_b, qkv_b: of the stored bf16 dz / dqkv (mmae_dgelu_colsum_bf16 / mmae_colsum_bf16 sum what is stored).
round=False: plain float64 with plain attention (the fp32 tier, mmae_block_f32_*).

The block input is x_in + s_prev * x_add (x_add: the previous block's bf16 MLP branch in a chain, or None).  Per-sample
factors are [B] tensors or None (factor 1).  `mutate` names a deliberately wrong variant for the sensitivity checks:
  "neighbour_keys"    every sample attends to the previous sample's keys;
  "head_shift"        q of head h against k / v of head h+1;
  "neighbour_scales"  every sample gets the previous sample's drop-path factors."""
import math

import torch

from pretrain_io_oracle import Attention, _ln, bf16, gelu, rb, rf  # noqa: F401  (bf16 / Attention re-exported)
from pretrain_io_oracle import attention, roundings

PARAMS = ["norm1_w", "norm1_b", "qkv_w", "qkv_b", "proj_w", "proj_b", "norm2_w", "norm2_b", "fc1_w", "fc1_b", "fc2_w",
          "fc2_b"]
MUTATIONS = ("neighbour_keys", "head_shift", "neighbour_scales")


def _per_sample(s, mutate):
    if s is None:
        return 1.0
    if mutate == "neighbour_scales":
        s = torch.roll(s, 1, 0)
    return s.reshape(-1, 1, 1)


def block_forward(x_in, prm, H, eps, fuse_gelu=False, round=True, s_attn=None, s_mlp=None, x_add=None, s_prev=None,
                  mutate=None):
    """One block: returns (x, x_mid, y2, qkv) with x the block input (x_in + s_prev x_add), x_out = x_mid + s_mlp * y2.
    prm: float64 tensors named as PARAMS (leaves with requires_grad for a backward)."""
    rf_, rb_ = roundings(round)
    B, N, D = x_in.shape
    dh = D // H
    x = x_in if x_add is None else x_in + _per_sample(s_prev, mutate) * x_add
    h1 = rb_(rf_(_ln(x, prm["norm1_w"], prm["norm1_b"], eps)))
    qkv = rb_(rf_(h1 @ rf_(prm["qkv_w"]).t() + prm["qkv_b"]))
    q, k, v = (t.reshape(B, N, H, dh).transpose(1, 2) for t in qkv.split(D, -1))
    if mutate == "neighbour_keys":
        k = torch.roll(k, 1, 0)
    elif mutate == "head_shift":
        k, v = torch.roll(k, -1, 1), torch.roll(v, -1, 1)
    o = rb_(rf_(attention(q, k, v, 1.0 / math.sqrt(dh), round).transpose(1, 2).reshape(B, N, D)))
    y = rf_(rb_(o @ rf_(prm["proj_w"]).t()) + prm["proj_b"])
    x_mid = x + _per_sample(s_attn, mutate) * y
    h2 = rb_(rf_(_ln(x_mid, prm["norm2_w"], prm["norm2_b"], eps)))
    zp = h2 @ rf_(prm["fc1_w"]).t() + prm["fc1_b"]
    z = rb_(rf_(zp))
    if fuse_gelu and round:
        # GELU in the fc1 epilogue on the fp32 pre-activation; fc2's dgrad applies GELU'(bf16 z) before its one bf16 store
        gz = gelu(z)
        a = rf(gelu(zp).detach() + gz - gz.detach())
    else:
        # a streaming kernel applies GELU to the stored bf16 z; fc2's dgrad is stored bf16 before GELU' is applied
        a = rb_(rf_(gelu(z)))
    y2 = rf_(rb_(a @ rf_(prm["fc2_w"]).t()) + prm["fc2_b"])
    return x, x_mid, y2, qkv


def block_reference(x_in, prm, H, eps, dout, fuse_gelu=False, round=True, s_attn=None, s_mlp=None, x_add=None,
                    s_prev=None, mutate=None):
    """Forward and backward of one block for the float64 values x_in (and x_add).  Returns a dict: the forward values
    x_mid, x_out, the branch outputs attn = x_mid - x and mlp = x_out - x_mid, the input gradient dx_in (of x_in) and,
    with x_add, dx_add (of x_add, i.e. s_prev dx_in: what the hand-off rounds and sums), every parameter gradient under
    its PARAMS name, and dk_abs: the column sums of |dk|, the terms of the key part of qkv_b's gradient."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in prm.items()}
    xi = x_in.detach().clone().requires_grad_(True)
    xa = None if x_add is None else x_add.detach().clone().requires_grad_(True)
    x, x_mid, y2, qkv = block_forward(xi, leaves, H, eps, fuse_gelu, round, s_attn, s_mlp, xa, s_prev, mutate)
    x_out = x_mid + _per_sample(s_mlp, mutate) * y2
    x_mid.retain_grad()
    qkv.retain_grad()
    x_out.backward(dout)
    out = {"x": x.detach(), "x_mid": x_mid.detach(), "x_out": x_out.detach(), "attn": (x_mid - x).detach(),
           "mlp": (x_out - x_mid).detach(), "dx_in": xi.grad, "dx_mid": x_mid.grad, "dk_abs": _dk_abs(qkv)}
    if xa is not None:
        out["dx_add"] = xa.grad
    for k in PARAMS:
        out[k] = leaves[k].grad
    return out


def _dk_abs(qkv):
    """column sums of |dk|.  The key bias's gradient colsum(dk) is 0 in exact arithmetic (a shift of every key's score
    by the same amount leaves the softmax unchanged): what is left is rounding noise on the scale of these terms."""
    D = qkv.shape[-1] // 3
    return qkv.grad[..., D:2 * D].abs().sum((0, 1))


def chain_reference(x_in, prms, H, eps, dout, fuse_gelu=False, scales=None, mutate=None):
    """n blocks chained as BlockFunction chains them (functional.py): block i+1's input is block i's x_mid plus
    s_mlp(i) times its bf16 MLP branch.  scales: one (s_attn, s_mlp) or None per block.  Returns one dict per block as
    block_reference's (x: the block's input, x_out: its output), from ONE backward through the whole stack.

    mutate: the variants of block_forward apply to every block; "handoff_twice" / "handoff_missing" give every block but
    the last an fc2 bias gradient with the column sum handed down by the next block counted twice / left out (in the
    chain that column sum is the whole of it)."""
    n = len(prms)
    scales = scales or [None] * n
    fwd_mut = mutate if mutate in MUTATIONS else None
    leaves = [{k: v.detach().clone().requires_grad_(True) for k, v in p.items()} for p in prms]
    xi = x_in.detach().clone().requires_grad_(True)
    outs, xs, mids, qkvs, x_add, s_prev = [], [], [], [], None, None
    x = xi
    for i in range(n):
        s_attn, s_mlp = scales[i] if scales[i] is not None else (None, None)
        xb, x_mid, y2, qkv = block_forward(x, leaves[i], H, eps, fuse_gelu, True, s_attn, s_mlp, x_add, s_prev, fwd_mut)
        xb.retain_grad()
        x_mid.retain_grad()
        qkv.retain_grad()
        qkvs.append(qkv)
        xs.append(xb)
        mids.append(x_mid)
        x, x_add, s_prev = x_mid, y2, s_mlp
    x_out = x + _per_sample(s_prev, fwd_mut) * x_add
    x_out.backward(dout)
    for i in range(n):
        nxt = xs[i + 1] if i + 1 < n else x_out
        r = {"x": xs[i].detach(), "x_mid": mids[i].detach(), "x_out": nxt.detach(), "attn": (mids[i] - xs[i]).detach(),
             "mlp": (nxt - mids[i]).detach(), "dx_in": xs[i].grad, "dx_mid": mids[i].grad, "dk_abs": _dk_abs(qkvs[i])}
        for k in PARAMS:
            r[k] = leaves[i][k].grad
        if i + 1 < n and mutate in ("handoff_twice", "handoff_missing"):
            r["fc2_b"] = 2 * r["fc2_b"] if mutate == "handoff_twice" else torch.zeros_like(r["fc2_b"])
        outs.append(r)
    return outs
