"""Dropout for the fp32 oracle (test infrastructure).

oracle/multimae_oracle.py restates Block without dropout.  `applied(masks)` runs the oracle's forward / step_losses with
explicit dropout masks instead:

    with applied({"encoder.1": dict(attn=(m_attn, 0.1), proj=(m_proj, 0.1), mlp=(m_mlp, 0.1))}):
        _, tokens = O.forward(...)

Keys are block prefixes as in state_dict.  Each site is (keep mask, p): the attention site's mask is [B, H, N, N] over the
softmax probabilities (Attention.attn_drop, multimae/multimae_utils.py:177), the proj and mlp sites' masks are [B, N, D]
over the branch outputs (Attention.proj_drop :181, Mlp.drop after fc2 :154).  A kept element is scaled by 1/(1-p), as
nn.Dropout does; p = 1 zeroes the site.  A site may be missing (no dropout there).  Per-sample stochastic-depth factors
(tests/drop_path_oracle.py) may be given as "scales": (s_attn, s_mlp).  Blocks not listed run unchanged."""
import contextlib

import torch

from oracle import multimae_oracle as O


def _apply(t, site):
    if site is None:
        return t
    mask, p = site
    return t * mask.to(t.dtype) * (1.0 / (1.0 - p)) if p < 1.0 else t * 0.0


def attention(x, p, prefix, heads, attn_site=None, proj_site=None):   # multimae/multimae_utils.py:170-182
    q, k, v = O._lin(x, p, prefix + ".qkv").chunk(3, dim=-1)
    q, k, v = O._heads(q, heads), O._heads(k, heads), O._heads(v, heads)
    w = torch.softmax((q @ k.transpose(-2, -1)) * q.shape[-1] ** -0.5, dim=-1)
    o = _apply(w, attn_site) @ v
    o = o.transpose(1, 2).reshape(o.shape[0], o.shape[2], -1)
    return _apply(O._lin(o, p, prefix + ".proj"), proj_site)


def block(x, p, prefix, heads, eps, sites=None):                      # multimae/multimae_utils.py:229-232
    """Pre-LN transformer block with the dropout sites (and optional stochastic-depth factors) of `sites`."""
    sites = sites or {}
    s_attn, s_mlp = sites.get("scales", (None, None))
    a = attention(O._ln(x, p, prefix + ".norm1", eps), p, prefix + ".attn", heads, sites.get("attn"), sites.get("proj"))
    x = x + (a if s_attn is None else a * s_attn.reshape(-1, 1, 1))
    m = _apply(O._mlp(O._ln(x, p, prefix + ".norm2", eps), p, prefix + ".mlp"), sites.get("mlp"))
    return x + (m if s_mlp is None else m * s_mlp.reshape(-1, 1, 1))


@contextlib.contextmanager
def applied(table):
    """Inside the context every oracle block whose prefix is a key of `table` applies those sites."""
    original = O._block

    def dispatch(x, p, prefix, heads, eps):
        return block(x, p, prefix, heads, eps, table.get(prefix))

    O._block = dispatch
    try:
        yield
    finally:
        O._block = original
