"""utils/model_ema.py:18-84 restated: ModelEma as the reference defines it (the class the overlay replaces)."""
from collections import OrderedDict
from copy import deepcopy

import torch


class ModelEma:
    def __init__(self, model, decay=0.9999, device='', resume=''):
        self.ema = deepcopy(model)
        self.ema.eval()
        self.decay = decay
        self.device = device
        if device:
            self.ema.to(device=device)
        self.ema_has_module = hasattr(self.ema, 'module')
        if resume:
            self._load_checkpoint(resume)
        for p in self.ema.parameters():
            p.requires_grad_(False)

    def _load_checkpoint(self, checkpoint_path):
        checkpoint = torch.load(checkpoint_path, map_location='cpu')
        assert isinstance(checkpoint, dict)
        if 'state_dict_ema' not in checkpoint:
            print("Failed to find state_dict_ema, starting from loaded model weights")
            return
        renamed = OrderedDict()
        for k, v in checkpoint['state_dict_ema'].items():
            renamed[('module.' + k if not k.startswith('module') else k) if self.ema_has_module else k] = v
        self.ema.load_state_dict(renamed)
        print("Loaded state_dict_ema")

    def update(self, model):
        # the prefix is added whenever the live model has `.module` and the EMA copy has not
        prefix = 'module.' if hasattr(model, 'module') and not self.ema_has_module else ''
        with torch.no_grad():
            msd = model.state_dict()
            for k, ema_v in self.ema.state_dict().items():
                model_v = msd[prefix + k].detach()
                if self.device:
                    model_v = model_v.to(device=self.device)
                ema_v.copy_(ema_v * self.decay + (1. - self.decay) * model_v)
