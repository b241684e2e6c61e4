"""Masked reconstruction losses with the reference's constructor / call contract (multimae/criterion.py), each executed
as one fused forward kernel + one fused backward kernel with no host synchronisation."""
import torch.nn as nn

from . import functional as Fn
from .lazy_meters import DeferredScalar


class _MaskedLoss(nn.Module):
    """Common shape of the three criteria: per-pixel loss -> mean over channels -> patch mask upsampled by
    `scale_factor = patch_size // stride` -> per-sample mean over masked pixels -> nanmean over the batch
    (multimae/criterion.py:37-57, 84-114, 141-171); `mask=None` is the plain mean (loss_on_unmasked)."""

    kind = None                     # kernel selector of mmae_masked_loss_*: 0 MSE, 1 L1, 2 cross-entropy

    def _configure(self, patch_size, stride, norm_pix=False, label_smoothing=0.0):
        self.patch_size = patch_size
        self.stride = stride
        self.scale_factor = patch_size // stride
        self.norm_pix = norm_pix
        self.label_smoothing = label_smoothing

    def forward(self, input, target, mask=None):
        Fn.sync_deterministic()
        loss = Fn.MaskedLossFunction.apply(input, target, mask, self.kind, bool(self.norm_pix), self.scale_factor,
                                           float(self.label_smoothing))
        return DeferredScalar.wrap(loss)       # plain tensor unless the overlay's lazy meters are on (lazy_meters.py)


class MaskedCrossEntropyLoss(_MaskedLoss):
    """Cross-entropy loss with masking (multimae/criterion.py:23-57)."""

    kind = 2

    def __init__(self, patch_size: int = 16, stride: int = 1, label_smoothing: float = 0.0):
        super().__init__()
        self._configure(patch_size, stride, label_smoothing=label_smoothing)


class MaskedMSELoss(_MaskedLoss):
    """MSE loss with masking and optional per-patch target normalisation (multimae/criterion.py:60-114)."""

    kind = 0

    def __init__(self, patch_size: int = 16, stride: int = 1, norm_pix=False):
        super().__init__()
        self._configure(patch_size, stride, norm_pix=norm_pix)


class MaskedL1Loss(_MaskedLoss):
    """L1 loss with masking and optional per-patch target normalisation (multimae/criterion.py:117-171)."""

    kind = 1

    def __init__(self, patch_size: int = 16, stride: int = 1, norm_pix=False):
        super().__init__()
        self._configure(patch_size, stride, norm_pix=norm_pix)
