"""ModelEma with the reference's contract (utils/model_ema.py:18-84): an exponential moving average of everything in the
model's state_dict, kept in a deep copy of the model (`ema`), for run_finetuning_cls.py --model_ema.

On CUDA, `update(model)` is ONE mmae_ema_update call on the current stream for all state_dict entries, instead of four
torch kernels per entry, and computes bitwise what the reference's `ema_v * decay + (1. - decay) * model_v` computes.
The frozen position tables are averaged too, as the reference does.

Differences from the reference, none of which changes a value:
  - `update` unwraps `.module` (DistributedDataParallel, or the overlay's stand-in for it) on both sides and pairs entries
    by name: the reference adds a 'module.' prefix that the stand-in's forwarded state_dict() does not have;
  - the copy shares nothing with the live model's training machinery (gradient arena, data-parallel reducer, bound
    arena views, cached position tables), even when the model has already trained.

`device='cpu'` (--model_ema_force_cpu) keeps the reference's per-tensor torch loop on the host; as the reference notes,
an EMA kept there cannot be evaluated on the GPU path.

Resume keeps the reference's behaviour, quirk included: the script's auto_load_model hands `_load_checkpoint_for_ema` the
bare state_dict stored under 'model_ema' (utils/checkpoint.py:131-132), which has no 'state_dict_ema' key, so a resumed
run prints "Failed to find state_dict_ema, starting from loaded model weights" and the EMA keeps the weights it was built
from.  `_load_checkpoint({'state_dict_ema': ...})` does load them."""
import ctypes
import weakref
from collections import OrderedDict
from copy import deepcopy

import torch
from torch.autograd.graph import increment_version

from . import _lib as L
from . import functional as Fn

# per-module attributes of the training machinery (multimae.py, multimae_utils.py, input_adapters.py, output_adapters.py,
# overlay.py) that the EMA copy must not inherit: those in _FRESH get the value a freshly built module has, those in _DROP
# are removed (a fresh module does not have them)
_FRESH = {"_arena": None, "_grad_callback": None, "_meta": None, "_bound": None, "_own_arena": False,
          "_dec_streams": None, "_alphas_dev": None}
_DROP = ("_pos_cache", "_mmae_reducer")


def _unwrap(model):
    return model.module if hasattr(model, "module") else model


def _detached_copy(model):
    """deepcopy(model) without the objects listed in _FRESH / _DROP: they are neither copied nor shared."""
    memo = {}
    root = _unwrap(model)
    for m in root.modules():
        for name in list(_FRESH) + list(_DROP):
            v = m.__dict__.get(name)
            if v is not None and not isinstance(v, bool):
                memo[id(v)] = None
    ema = deepcopy(model, memo)
    for m in _unwrap(ema).modules():
        for name, fresh in _FRESH.items():
            if name in m.__dict__:
                m.__dict__[name] = fresh
        for name in _DROP:
            m.__dict__.pop(name, None)
    return ema


def _slots(module):
    """{state_dict key: (the `_parameters` or `_buffers` dict holding its tensor, name)}."""
    slots = {}
    for k, t in module.state_dict(keep_vars=True).items():
        owner, _, name = k.rpartition(".")
        sub = module.get_submodule(owner)
        if sub._parameters.get(name) is t:
            slots[k] = (sub._parameters, name)
        elif sub._buffers.get(name) is t:
            slots[k] = (sub._buffers, name)
        else:
            raise NotImplementedError("ModelEma: state_dict entry %r is not a parameter or buffer of %r" % (k, owner))
    return slots


class ModelEma:
    """Model Exponential Moving Average (reference utils/model_ema.py:18-84, same constructor, attributes and methods)."""

    def __init__(self, model, decay=0.9999, device='', resume=''):
        self.ema = _detached_copy(model)
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
        self._slots = None         # (weakref to the live model, where each pair's tensors live): see _pairs
        self._args = None          # (pointers, ctypes arrays) of the last update: reused while the pointers hold

    def _load_checkpoint(self, checkpoint_path):
        checkpoint = torch.load(checkpoint_path, map_location='cpu')
        assert isinstance(checkpoint, dict)
        if 'state_dict_ema' in checkpoint:
            new_state_dict = OrderedDict()
            for k, v in checkpoint['state_dict_ema'].items():
                # the EMA model may have been wrapped by DataParallel and need the module prefix
                if self.ema_has_module:
                    name = 'module.' + k if not k.startswith('module') else k
                else:
                    name = k
                new_state_dict[name] = v
            self.ema.load_state_dict(new_state_dict)
            print("Loaded state_dict_ema")
        else:
            print("Failed to find state_dict_ema, starting from loaded model weights")

    def update(self, model):
        model = _unwrap(model)
        with torch.no_grad():
            if self.device:
                msd = model.state_dict()
                for k, ema_v in _unwrap(self.ema).state_dict().items():
                    model_v = msd[k].detach().to(device=self.device)
                    ema_v.copy_(ema_v * self.decay + (1. - self.decay) * model_v)
                return
            self._update_cuda(model)

    def _pairs(self, model):
        """(EMA tensor, model tensor) of every state_dict entry of the EMA, in its order, paired by name.  The slots the
        tensors live in are found once per model; reading the tensors from them at every update sees replaced parameters
        and `.data` swaps at a fraction of the cost of two state_dict() calls."""
        if self._slots is None or self._slots[0]() is not model:
            ema_slots, live_slots = _slots(_unwrap(self.ema)), _slots(model)
            self._slots = (weakref.ref(model), [(ema_slots[k], live_slots[k]) for k in ema_slots])
        return [(ed[en], md[mn]) for (ed, en), (md, mn) in self._slots[1]]

    def _update_cuda(self, model):
        pairs = self._pairs(model)
        key = [t.data_ptr() for pair in pairs for t in pair]
        if self._args is None or self._args[0] != key:
            for e, v in pairs:
                if e.dtype != torch.float32 or v.dtype != torch.float32:
                    raise TypeError("ModelEma.update: the CUDA path averages fp32 tensors only, got %s / %s"
                                    % (e.dtype, v.dtype))
                Fn._require_cuda(e, "ModelEma.update (device='cpu' keeps the EMA on the host)")
                if e.device != v.device:
                    raise ValueError("ModelEma.update: EMA on %s, model on %s" % (e.device, v.device))
                if e.shape != v.shape or not (e.is_contiguous() and v.is_contiguous()):
                    raise ValueError("ModelEma.update: EMA and model entries must be contiguous tensors of one shape")
            n = len(pairs)
            self._args = (key, (ctypes.c_void_p * n)(*key[0::2]), (ctypes.c_void_p * n)(*key[1::2]),
                          (ctypes.c_int64 * n)(*[e.numel() for e, _ in pairs]))
        _, dst, src, sizes = self._args
        L.check(L.lib().mmae_ema_update(dst, src, sizes, len(pairs), float(self.decay), float(1.0 - self.decay),
                                        L.current_stream()), "mmae_ema_update")
        increment_version([e for e, _ in pairs])     # what copy_ does: caches keyed on the version see the new values
