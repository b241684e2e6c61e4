"""Stand-in for the part of the reference's `utils` package (EPFL-VILAB/MultiMAE, utils/) that run_finetuning_cls.py
uses around --model_ema, restated so that the tests run without a reference checkout.  Same module layout
(utils.model_ema, utils.model, utils.checkpoint) and same behaviour - printed messages included - of ModelEma,
unwrap_model / get_state_dict and the torch.amp branch of save_model / auto_load_model.

Only the tests import it, with this directory put on sys.path; nothing else here is named `utils`."""
from .checkpoint import _load_checkpoint_for_ema, auto_load_model, save_model  # noqa: F401
from .model import get_state_dict, unwrap_model  # noqa: F401
from .model_ema import ModelEma  # noqa: F401
