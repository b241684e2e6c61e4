"""GPU: the float64 checks of the pre-training input side, run again in deterministic mode at their own tolerances.

test_embed_bit_exact (tests/test_cuda_pretrain_io.py) holds mmae_embed_backward to float64: the global-token (G = 1 and 2)
and per-task bias gradients bit-exact, the semseg class-embedding gradient per table row, at shapes with hundreds of
blocks per reduction.  In deterministic mode these sums are the per-block partials added in block order
(embed_assemble_bwd_kernel, semseg_emb_bwd_det_kernel and colred_finalize) instead of atomics."""
import pytest
import torch

from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from test_cuda_pretrain_io import dev, test_embed_bit_exact  # noqa: F401  (fixture, test run again here)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def deterministic_mode():
    """torch's flag on (warn_only) and the library's switch with it; both restored afterwards."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    Fn.sync_deterministic()
    assert Fn._deterministic
    L.lib()
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
        Fn.sync_deterministic()
