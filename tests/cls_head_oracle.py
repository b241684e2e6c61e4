"""fp32 restatement of the fine-tuning classification model for the tests: MultiViT's encoder through the oracle
(oracle/multimae_oracle.py, every token kept) and LinearOutputAdapter.forward (multimae/output_adapters.py:345-356)."""
import torch
import torch.nn.functional as F

from oracle import multimae_oracle as O


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


def cls_head(enc, p, mean_pool=True, eps=1e-6, prefix="output_adapters.cls."):
    """pool -> LayerNorm -> Linear (no Linear when the state has no head weight: num_classes = 0, nn.Identity)."""
    x = enc.mean(1) if mean_pool else enc[:, -1]
    x = F.layer_norm(x, (x.shape[-1],), p[prefix + "norm.weight"], p[prefix + "norm.bias"], eps)
    if prefix + "head.weight" in p:
        x = x @ p[prefix + "head.weight"].t() + p[prefix + "head.bias"]
    return x


def soft_target_ce(logits, target):
    """SoftTargetCrossEntropy (the criterion of run_finetuning_cls.py with mixup)."""
    return torch.sum(-target * F.log_softmax(logits, dim=-1), dim=-1).mean()
