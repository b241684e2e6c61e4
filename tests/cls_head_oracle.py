"""fp32 restatement of the fine-tuning classification model for the tests: MultiViT's encoder through the oracle
(oracle/multimae_oracle.py, every token kept) and LinearOutputAdapter.forward (multimae/output_adapters.py:345-356)."""
import torch
import torch.nn.functional as F

from oracle import multimae_oracle as O
from pretrain_io_oracle import _ln, roundings


def vit_config(in_domains, dim, depth, heads, image_size):
    cfg = O.make_config(in_domains=tuple(in_domains), out_domains=[], extra_norm_pix=False)
    cfg.dim, cfg.depth, cfg.heads = dim, depth, heads
    cfg.posemb_grid = image_size // 16
    return cfg


def encoder_tokens(p, x, cfg):
    """MultiViT.process_input + encoder (multimae/multimae.py:439-486): all tokens of every modality, global token last."""
    B = next(iter(x.values())).shape[0]
    total = sum((v.shape[-1] // 16) * (v.shape[-2] // 16) for v in x.values())
    ids = torch.arange(total).unsqueeze(0).expand(B, -1).contiguous()
    _, enc = O.forward(p, x, cfg, ids, ids)
    return enc


def head(enc, norm_w, norm_b, head_w=None, head_b=None, mean_pool=True, eps=1e-6, round=False, mutate=None):
    """mmae_clshead_*: pool -> LayerNorm -> Linear (no Linear when head_w is None: num_classes = 0, nn.Identity).
    round=True: float64 with the kernels' bf16 stores (tests/test_cuda_heads.py) - the LayerNorm output and the weight as
    the head GEMM's operands (rf) and the logit gradient as its backward operand (rb), the bias gradient a column sum of
    the fp32 logit gradient; the pool and the LayerNorm are fp32.  mutate="mean_short": the mean over the first N - 1
    tokens (the sensitivity checks)."""
    rf_, rb_ = roundings(round)
    if mean_pool:
        x = enc[:, :-1].mean(1) if mutate == "mean_short" else enc.mean(1)
    else:
        x = enc[:, -1]
    x = _ln(x, norm_w, norm_b, eps)
    if head_w is None:
        return x
    return rb_(rf_(x) @ rf_(head_w).t()) + head_b


def cls_head(enc, p, mean_pool=True, eps=1e-6, prefix="output_adapters.cls."):
    """pool -> LayerNorm -> Linear (no Linear when the state has no head weight: num_classes = 0, nn.Identity)."""
    return head(enc, p[prefix + "norm.weight"], p[prefix + "norm.bias"], p.get(prefix + "head.weight"),
                p.get(prefix + "head.bias"), mean_pool, eps)


def soft_target_ce(logits, target):
    """SoftTargetCrossEntropy (the criterion of run_finetuning_cls.py with mixup)."""
    return torch.sum(-target * F.log_softmax(logits, dim=-1), dim=-1).mean()
