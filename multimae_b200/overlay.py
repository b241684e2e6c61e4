"""Drop-in overlay: make `import multimae...` / `from utils import NativeScalerWithGradNormCount` resolve to this package
so the reference's UNCHANGED run_pretraining_multimae.py drives the sm_90a path.

    python -m multimae_b200.overlay /path/to/MultiMAE/run_pretraining_multimae.py -c cfg.yaml [script args...]

What is replaced (north_star "Subsystems replaced"): multimae.multimae, multimae.multimae_utils, multimae.input_adapters,
multimae.output_adapters (SpatialOutputAdapter, LinearOutputAdapter, ConvNeXtAdapter), multimae.criterion,
utils.native_scaler.NativeScalerWithGradNormCount, utils.ModelEma (also as utils.model_ema.ModelEma and
utils.model.ModelEma, the name unwrap_model tests), with MMAE_FLAT_ADAMW=1 the AdamW that utils.optim_factory builds
(GroupedFlatAdamW) and — because the model owns its bucketed gradient all-reduce —
torch.nn.parallel.DistributedDataParallel is substituted by an identity wrapper.  Everything else (argument parsing, data pipeline, optimizer factory, logging, checkpoints)
stays the reference's own code from `reference_root`."""
import importlib
import math
import os
import runpy
import sys
import types


class _IdentityDDP:
    """Stands in for DistributedDataParallel (run_pretraining_multimae.py:380-383) around a MultiMAE: gradients are reduced
    in place by multimae_b200.parallel.FlatGradReducer, so no wrapper logic is needed.  Exposes `.module` like DDP does.
    Any OTHER module the script wraps (the task balancer, run_pretraining_multimae.py:384-386) keeps the real
    DistributedDataParallel: its few parameters are outside the flat arena and must still be averaged across ranks."""

    _real = None          # torch's own class, saved by install() before the substitution

    def __new__(cls, module, *args, **kwargs):
        import torch
        from .multimae import MultiMAE
        from .parallel import attach_data_parallel, broadcast_parameters
        if isinstance(module, MultiMAE):
            if torch.distributed.is_initialized():
                broadcast_parameters(module)
                module._mmae_reducer = attach_data_parallel(module)
            return _Wrapped(module)
        trainable = any(p.requires_grad for p in module.parameters())
        if cls._real is not None and trainable and torch.distributed.is_initialized():
            if not any(p.is_cuda for p in module.parameters()):
                kwargs.pop("device_ids", None)
            return cls._real(module, *args, **kwargs)
        return _Wrapped(module)


class _Wrapped:
    def __init__(self, module):
        self.__dict__["module"] = module

    def __call__(self, *a, **k):
        return self.module(*a, **k)

    def __getattr__(self, name):
        return getattr(self.__dict__["module"], name)


class _FactoryOptim:
    """MMAE_FLAT_ADAMW=1: what utils.optim_factory sees as `optim` (torch.optim).  `AdamW` builds the one-kernel
    multimae_b200.optim.GroupedFlatAdamW - or torch's AdamW, with one printed line, when a trainable parameter is not on
    CUDA or not a parameter of the MultiMAE / MultiViT; every other name (SGD, Adam) is torch's."""

    def __init__(self, stock):
        self._stock = stock

    def __getattr__(self, name):
        return getattr(self._stock, name)

    @staticmethod
    def AdamW(params, *args, **kwargs):
        from .optim import adamw_or_stock
        return adamw_or_stock(params, *args, **kwargs)


def _legacy_checkpoint_load():
    """torch >= 2.6 made `torch.load` default to weights_only=True; the reference (pinned to torch 1.10) re-loads its OWN
    checkpoints - model / optimizer / scaler state plus the argparse Namespace and numpy schedule scalars - with a bare
    `torch.load(path, map_location='cpu')` (utils/checkpoint.py:124).  Restore the default the script was written against
    for calls that do not say otherwise.  Like the `torch._six` stub this is a torch-version shim, not a change of the script."""
    import functools
    import torch
    if getattr(torch.load, "_mmae_legacy_default", False):
        return
    original = torch.load

    @functools.wraps(original)
    def load(*args, **kwargs):
        kwargs.setdefault("weights_only", False)
        return original(*args, **kwargs)

    load._mmae_legacy_default = True
    torch.load = load


def _deterministic_from_env():
    """MMAE_DETERMINISTIC=1 (or `warn`): torch.use_deterministic_algorithms(True) (warn_only=True for `warn`) before the
    script runs, which also puts the CUDA path into its deterministic mode (functional.sync_deterministic).  cuBLAS needs
    CUBLAS_WORKSPACE_CONFIG for deterministic results in the script's own torch ops; :4096:8 is set unless it is given."""
    mode = os.environ.get("MMAE_DETERMINISTIC", "0").strip().lower()
    if mode in ("", "0"):
        return
    if mode not in ("1", "warn"):
        raise ValueError("MMAE_DETERMINISTIC=%r: expected 0, 1 or warn" % mode)
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    import torch
    torch.use_deterministic_algorithms(True, warn_only=mode == "warn")


def install(reference_root=None, replace_ddp=True, legacy_checkpoint_load=True):
    """Install the overlay into sys.modules.  `reference_root`: checkout of EPFL-VILAB/MultiMAE (for its `utils` package)."""
    if "torch._six" not in sys.modules:            # utils/native_scaler.py:11 imports a module removed in torch >= 2
        six = types.ModuleType("torch._six")
        six.inf = math.inf
        sys.modules["torch._six"] = six
    if legacy_checkpoint_load:
        _legacy_checkpoint_load()
    _deterministic_from_env()
    if reference_root is not None and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    pkg = types.ModuleType("multimae")
    pkg.__path__ = []                              # namespace-like: submodules are injected below
    sys.modules["multimae"] = pkg
    for sub in ("multimae_utils", "input_adapters", "output_adapters", "criterion", "multimae"):
        mod = importlib.import_module("multimae_b200." + sub)
        sys.modules["multimae." + sub] = mod
        setattr(pkg, sub, mod)
    from . import multimae as mm
    mm.AUTO_OWN_GRADIENTS = True                   # p.grad = views of the flat gradient arena (see multimae.py)
    # register the factories in the reference's registry if it only became importable now
    try:
        from utils.registry import _model_entrypoints, register_model  # type: ignore
        for name in mm.__all__:
            if name not in _model_entrypoints:
                register_model(getattr(mm, name))
    except Exception:  # noqa: BLE001
        pass
    try:
        import utils  # type: ignore
        from .native_scaler import NativeScalerWithGradNormCount, get_grad_norm_
        utils.NativeScalerWithGradNormCount = NativeScalerWithGradNormCount
        utils.native_scaler.NativeScalerWithGradNormCount = NativeScalerWithGradNormCount
        utils.native_scaler.get_grad_norm_ = get_grad_norm_
    except Exception:  # noqa: BLE001
        pass
    try:
        import utils  # type: ignore
        from .model_ema import ModelEma
        utils.ModelEma = ModelEma
        utils.model_ema.ModelEma = ModelEma
        utils.model.ModelEma = ModelEma            # unwrap_model's isinstance test: save_model stores the EMA's state_dict
    except Exception:  # noqa: BLE001
        pass
    if os.environ.get("MMAE_FLAT_ADAMW", "0") == "1":
        try:
            import utils.optim_factory as factory  # type: ignore
            if not isinstance(factory.optim, _FactoryOptim):
                factory.optim = _FactoryOptim(factory.optim)   # create_optimizer calls optim.AdamW through this global
        except Exception:  # noqa: BLE001
            pass
    from . import lazy_meters
    lazy_meters.install()                          # MMAE_LAZY_METERS=1: the script's ~10 .item() per step answer one step late
    from . import data
    data.install()                                 # MMAE_DEVICE_FEED=1 / MMAE_SYNTHETIC_DATA=N: see data.py
    if replace_ddp:
        import torch
        if torch.nn.parallel.DistributedDataParallel is not _IdentityDDP:
            _IdentityDDP._real = torch.nn.parallel.DistributedDataParallel
        torch.nn.parallel.DistributedDataParallel = _IdentityDDP
    return pkg


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit(__doc__)
    script = os.path.abspath(argv[0])
    install(reference_root=os.path.dirname(script))
    sys.argv = [script] + argv[1:]
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
