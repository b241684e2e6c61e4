"""utils/model.py:17-25 restated: unwrap_model tests `isinstance(model, ModelEma)` against this module's global, which is
why the overlay also rebinds utils.model.ModelEma."""
from .model_ema import ModelEma


def unwrap_model(model):
    if isinstance(model, ModelEma):
        return unwrap_model(model.ema)
    return model.module if hasattr(model, 'module') else model


def get_state_dict(model, unwrap_fn=unwrap_model):
    return unwrap_fn(model).state_dict()
