"""Stochastic depth for the fp32 oracle (test infrastructure).

oracle/multimae_oracle.py restates Block with drop_path = 0.  `applied(factors)` runs the oracle's forward /
decode_task / step_losses with per-sample stochastic-depth factors instead:

    with applied({"encoder.3": (s_attn, s_mlp), "output_adapters.rgb.decoder_transformer.1": (s_attn, s_mlp)}):
        losses, preds = O.step_losses(...)

Keys are block prefixes as in state_dict; each factor is a [B] tensor, 0 for a dropped sample and 1/keep for a kept one
(multimae/multimae_utils.py:105-132: the branch output times floor(keep + u) / keep).  Blocks not listed run unchanged.
The oracle's functions look `_block` up at call time, so the context swaps in `block` below for its duration; autograd
keeps what it recorded, so backward may run after the context has closed."""
import contextlib

from oracle import multimae_oracle as O


def block(x, p, prefix, heads, eps, scales=None):                       # multimae/multimae_utils.py:229-232
    """Pre-LN transformer block with optional per-sample factors (s_attn, s_mlp) on its two residual branches."""
    s_attn, s_mlp = (None, None) if scales is None else (scales[0].reshape(-1, 1, 1), scales[1].reshape(-1, 1, 1))
    a = O._self_attention(O._ln(x, p, prefix + ".norm1", eps), p, prefix + ".attn", heads)
    x = x + (a if s_attn is None else a * s_attn)
    m = O._mlp(O._ln(x, p, prefix + ".norm2", eps), p, prefix + ".mlp")
    return x + (m if s_mlp is None else m * s_mlp)


@contextlib.contextmanager
def applied(factors):
    """Inside the context every oracle block whose prefix is a key of `factors` applies those factors."""
    original = O._block

    def dispatch(x, p, prefix, heads, eps):
        return block(x, p, prefix, heads, eps, factors.get(prefix))

    O._block = dispatch
    try:
        yield
    finally:
        O._block = original
