"""Transformer building blocks with the reference's module / parameter names (multimae/multimae_utils.py), executing on
the sm_90a kernels.  `Block` is the unit of execution (one fused forward / backward sequence, stochastic depth included); `Attention`, `Mlp` and
`CrossAttention` are parameter containers with the reference constructor signatures so that `state_dict()` keys match
(SURVEY.md §A.1)."""
import math
import warnings

import torch
import torch.nn as nn

from . import functional as Fn


def pair(t):
    return t if isinstance(t, tuple) else (t, t)


def build_2d_sincos_posemb(h, w, embed_dim=1024, temperature=10000.0):
    """Fixed 2D sin-cos table [1, embed_dim, h, w] with the reference's axis convention
    (multimae/multimae_utils.py:29-45: grid built as meshgrid(w, h) then read back as '(h w)')."""
    assert embed_dim % 4 == 0, "Embed dimension must be divisible by 4 for 2D sin-cos position embedding"
    quarter = embed_dim // 4
    freq = (1.0 / (temperature ** (torch.arange(quarter, dtype=torch.float32) / quarter)))
    a = torch.arange(w, dtype=torch.float32).repeat_interleave(h)      # first meshgrid axis, flattened 'ij'
    b = torch.arange(h, dtype=torch.float32).repeat(w)                 # second meshgrid axis
    pa, pb = a[:, None] * freq[None, :], b[:, None] * freq[None, :]
    table = torch.cat([pa.sin(), pa.cos(), pb.sin(), pb.cos()], dim=1)  # [(w*h), D]
    return table.reshape(h, w, embed_dim).permute(2, 0, 1).unsqueeze(0).contiguous()


def trunc_normal_(tensor, mean=0.0, std=1.0, a=-2.0, b=2.0):
    """Truncated normal init with absolute cut-offs a, b (multimae/multimae_utils.py:84-102)."""
    if (mean < a - 2 * std) or (mean > b + 2 * std):
        warnings.warn("mean is more than 2 std from [a, b] in trunc_normal_", stacklevel=2)
    return nn.init.trunc_normal_(tensor, mean=mean, std=std, a=a, b=b)


class DropPath(nn.Module):
    """Stochastic depth (multimae/multimae_utils.py:105-132): holds `drop_prob` for its Block, which applies it per sample
    inside the fused block kernels (residual adds and branch-gradient casts, functional.drop_path_scales).  No parameters;
    repr and state_dict as the reference's."""

    def __init__(self, drop_prob=None):
        super().__init__()
        self.drop_prob = drop_prob

    def forward(self, x):
        if not self.drop_prob or not self.training:
            return x
        raise NotImplementedError("multimae_b200: drop path is applied inside Block (the fused block kernels); "
                                  "a stand-alone DropPath in training mode is not supported")

    def extra_repr(self):
        return "p={}".format(self.drop_prob)


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.0):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        assert act_layer is nn.GELU, "multimae_b200: exact-erf GELU only"
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)
        self.drop = nn.Dropout(drop)


class Attention(nn.Module):
    def __init__(self, dim, num_heads=8, qkv_bias=False, attn_drop=0.0, proj_drop=0.0):
        super().__init__()
        assert qkv_bias, "multimae_b200: qkv_bias=True only"
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)


class CrossAttention(nn.Module):
    def __init__(self, dim, num_heads=8, qkv_bias=False, attn_drop=0.0, proj_drop=0.0):
        super().__init__()
        assert qkv_bias and attn_drop == 0.0 and proj_drop == 0.0, "multimae_b200: qkv_bias=True, no dropout"
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.q = nn.Linear(dim, dim, bias=qkv_bias)
        self.kv = nn.Linear(dim, dim * 2, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)


def _ln_eps(norm_layer, dim):
    probe = norm_layer(dim)
    assert isinstance(probe, nn.LayerNorm), "multimae_b200: norm_layer must build nn.LayerNorm"
    return probe


class Block(nn.Module):
    """Pre-LN transformer layer; forward = one BlockFunction (multimae/multimae_utils.py:217-232)."""

    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=False, drop=0.0, attn_drop=0.0, drop_path=0.0,
                 act_layer=nn.GELU, norm_layer=nn.LayerNorm):
        super().__init__()
        self.norm1 = _ln_eps(norm_layer, dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, attn_drop=attn_drop, proj_drop=drop)
        self.drop_path = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.norm2 = _ln_eps(norm_layer, dim)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop)
        self.dim, self.num_heads, self.hidden = dim, num_heads, int(dim * mlp_ratio)
        assert dim // num_heads in (32, 64), "multimae_b200: head_dim must be 32 or 64"
        self._meta = None

    def bind(self, arena, prefix, on_grads_ready=None):
        """Attach the model's gradient arena; `prefix` is this block's state_dict prefix (with trailing dot)."""
        self._own_arena = False
        self._meta = dict(heads=self.num_heads, hidden=self.hidden, eps=self.norm1.eps, arena=arena, prefix=prefix,
                          on_grads_ready=on_grads_ready)

    def _params(self):
        return (self.norm1.weight, self.norm1.bias, self.attn.qkv.weight, self.attn.qkv.bias, self.attn.proj.weight,
                self.attn.proj.bias, self.norm2.weight, self.norm2.bias, self.mlp.fc1.weight, self.mlp.fc1.bias,
                self.mlp.fc2.weight, self.mlp.fc2.bias)

    def forward(self, x, fp32=False):
        """`fp32`: run this block in the fp32 tier (a decoder block of an adapter listed in fp32_output_adapters).  In
        training mode with drop_path > 0 each call draws the per-sample factors of both residual branches, and with a
        dropout rate > 0 the seed of its dropout masks."""
        return self.run(x, fp32=fp32, scales=Fn.drop_path_scales([self], x.shape[0], x.device)[0],
                        drops=Fn.block_dropouts([self], x.device, fp32)[0])

    def run(self, x, fp32=False, scales=None, drops=None):
        """One BlockFunction; `scales`: this block's entry of functional.drop_path_scales (None: no stochastic depth);
        `drops`: its entry of functional.block_dropouts (None: no dropout)."""
        if self._meta is None or self._meta["arena"].flat.device != x.device:
            # stand-alone use (outside MultiMAE): private gradient arena, zeroed on every forward
            self.bind(Fn.GradArena(list(self.named_parameters()), x.device), "")
            self._own_arena = True
        if getattr(self, "_own_arena", False) and torch.is_grad_enabled():
            self._meta["arena"].zero_()
        meta = dict(self._meta, fp32=True) if fp32 else self._meta
        return Fn.BlockFunction.apply(x, [meta], [scales], [drops], *self._params())
