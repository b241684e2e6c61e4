"""GPU: oracle checks of tests/test_cuda_parity.py run again in deterministic mode, at their own tolerances.

  - test_model_against_golden_and_oracle: a pre-training step (semseg input, a global token) against the float64 oracle,
    every gradient tensor on its own (embedding biases, global tokens, class-embedding table included), the losses and
    the reference fixture's per-tensor digests;
  - test_losses_against_oracle: the masked MSE / L1 / cross-entropy losses and gradients, whose per-sample sums are the
    [patch rows, B] partials added in row order;
  - test_flat_adamw_matches_torch: mmae_grad_unscale_norm over ~100 blocks, whose sum is the per-block partials added in
    block order."""
import pytest

from test_cuda_deterministic_io import deterministic_mode  # noqa: F401  (autouse fixture)
from test_cuda_parity import dev  # noqa: F401  (fixture)
from test_cuda_parity import test_flat_adamw_matches_torch, test_losses_against_oracle  # noqa: F401
from test_cuda_parity import test_model_against_golden_and_oracle  # noqa: F401

pytestmark = pytest.mark.gpu
