"""Stand-in for the optimizer factory of the reference's `utils` package (EPFL-VILAB/MultiMAE, utils/optim_factory.py),
restated so that the tests run without a reference checkout: the same parameter groups (per-layer lr_scale, weight decay
or none), the same `create_optimizer` arguments, and the same module global `optim` through which it builds the
optimizer - which is what the overlay's MMAE_FLAT_ADAMW switch rebinds.

Only the tests import it, with this directory put on sys.path; nothing else here is named `utils`."""
from . import optim_factory  # noqa: F401
