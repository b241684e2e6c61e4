"""NativeScalerWithGradNormCount with the reference's call contract (utils/native_scaler.py:14-46):
scaled backward -> unscale -> global grad-norm (-> clip / skip) -> optimizer step -> scale update.

When the parameters are backed by a model GradArena (multimae_b200.MultiMAE), unscale + non-finite check + L2 norm are
ONE pass over the flat gradient buffer (mmae_grad_unscale_norm) instead of ~344 per-tensor launches, and an optimizer
that exposes `fused_step(found_inf=...)` (multimae_b200.optim.FlatAdamW) is skipped on the device without a host sync.
The loss scale lives on the device; state_dict() has GradScaler's keys so checkpoints interoperate."""
import torch

from . import functional as Fn
from .lazy_meters import METERS, DeferredScalar

inf = float("inf")


def get_grad_norm_(parameters, norm_type: float = 2.0) -> torch.Tensor:
    """Generic per-tensor path (reference utils/native_scaler.py:49-62) for parameters that are not arena-backed."""
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    parameters = [p for p in parameters if p.grad is not None]
    norm_type = float(norm_type)
    if len(parameters) == 0:
        return torch.tensor(0.0)
    device = parameters[0].grad.device
    if norm_type == inf:
        return max(p.grad.detach().abs().max().to(device) for p in parameters)
    return torch.norm(torch.stack([torch.norm(p.grad.detach(), norm_type).to(device) for p in parameters]), norm_type)


def _find_arena(optimizer, parameters):
    """The flat gradient buffer behind the parameters: published by the optimizer (FlatAdamW), or - after backward - the
    arena all p.grad alias (data-parallel models own their gradients: parallel.attach_data_parallel)."""
    arena = getattr(optimizer, "mmae_arena", None)
    if arena is not None:
        return arena
    if parameters is not None:
        return Fn.find_arena_for(parameters)
    return None


class _LazyScalerState(dict):
    """state_dict() under lazy meters: `["scale"]` - what train_one_epoch reads every step
    (run_pretraining_multimae.py:538) - answers one step late without a host sync; every other use (iteration, pickling by
    utils.save_model, load_state_dict) sees the exact, synchronously read state."""

    def __init__(self, scaler):
        super().__init__()
        self._scaler = scaler

    def _exact(self):
        s = self._scaler
        return {"scale": float(s._scale), "growth_factor": s._growth_factor, "backoff_factor": s._backoff_factor,
                "growth_interval": s._growth_interval, "_growth_tracker": int(s._growth_tracker)}

    def __getitem__(self, key):
        if key == "scale":
            return METERS.read(self._scaler._scale, "loss_scale")
        return self._exact()[key]

    def get(self, key, default=None):
        return self._exact().get(key, default)

    def keys(self):
        return self._exact().keys()

    def values(self):
        return self._exact().values()

    def items(self):
        return self._exact().items()

    def __iter__(self):
        return iter(self._exact())

    def __len__(self):
        return 5

    def __contains__(self, key):
        return key in self._exact()

    def __bool__(self):
        return True

    def __reduce__(self):
        return (dict, (self._exact(),))


class NativeScalerWithGradNormCount:
    state_dict_key = "amp_scaler"

    def __init__(self, enabled=True, init_scale=2.0 ** 16, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000):
        self._enabled = enabled
        self._init_scale = float(init_scale)
        self._growth_factor, self._backoff_factor, self._growth_interval = growth_factor, backoff_factor, growth_interval
        self._scale = None           # device tensors, created lazily on the loss's device
        self._growth_tracker = None
        self._init_tracker = 0       # growth tracker restored by load_state_dict before the first step
        self._arena = None
        self._reducer = None

    def attach_reducer(self, reducer):
        """Data-parallel: join the bucketed all-reduce after backward and fold 1/world into the unscale pass."""
        self._reducer = reducer
        return self

    def attach_arena(self, arena):
        """Tell the scaler which flat gradient buffer backs the parameters (MultiMAE.grad_arena())."""
        self._arena = arena
        return self

    def _lazy_init(self, device):
        if self._scale is None:
            self._scale = torch.full((), self._init_scale if self._enabled else 1.0, dtype=torch.float32, device=device)
            self._growth_tracker = torch.full((), int(self._init_tracker), dtype=torch.int32, device=device)

    def __call__(self, loss, optimizer, clip_grad=None, skip_grad=None, parameters=None, create_graph=False,
                 update_grad=True):
        Fn.sync_deterministic()
        self._lazy_init(loss.device)
        if parameters is not None and not isinstance(parameters, (list, tuple)):
            parameters = list(parameters)            # the script passes the generator model.parameters()
        (loss * self._scale if self._enabled else loss).backward(create_graph=create_graph)
        arena = self._arena or _find_arena(optimizer, parameters)
        if not update_grad:
            # gradient accumulation (utils/native_scaler.py:25,39): keep what is in the flat buffer across the next forward
            if arena is not None:
                arena.accumulating = True
            return None
        # the bucketed all-reduces started during backward are joined here; a reducer that was attached to the model
        # behind the script's back (overlay: DistributedDataParallel -> identity wrapper) is found through its arena
        reducer = self._reducer if self._reducer is not None else getattr(arena, "reducer", None)
        post = reducer.finish() if reducer is not None else 1.0
        if arena is not None:
            inv = (1.0 / self._scale) if self._enabled else None
            norm, out2 = Fn.grad_unscale_norm(arena.flat, inv_scale=1.0, post_scale=post, inv_scale_tensor=inv)
            found_inf = out2[1:2]
            if not arena.owned and parameters is not None:
                # autograd may have copied instead of aliasing the arena views: make p.grad the (unscaled) views
                for (n, v), p in zip(arena.views.items(), [p for p in parameters if p.requires_grad]):
                    if p.grad is not None and p.grad.data_ptr() != v.data_ptr():
                        p.grad = v
        else:
            params = [p for p in (parameters or []) if p.grad is not None]
            inv = (1.0 / self._scale) if self._enabled else None
            if inv is not None:
                for p in params:
                    p.grad.mul_(inv)
            norm = get_grad_norm_(params)
            found_inf = (~torch.isfinite(norm)).float().reshape(1)
        # GradScaler.unscale_(optimizer) (utils/native_scaler.py:34) covers EVERY parameter the optimizer holds, not only
        # `parameters`: e.g. the uncertainty task balancer's log_vars sit in the optimizer but not in model.parameters().
        # Unscale them too and fold their non-finite check into found_inf (they are not part of the returned norm, as in
        # the reference, whose norm runs over `parameters` only).
        if self._enabled:
            found_inf = self._unscale_outside(optimizer, arena, None if arena is not None else params, inv, found_inf)
        if clip_grad is not None:
            assert parameters is not None or arena is not None
            coef = torch.clamp(clip_grad / (norm + 1e-6), max=1.0)
            if arena is not None:
                arena.flat.mul_(coef)
            else:
                for p in params:
                    p.grad.mul_(coef)
        elif skip_grad is not None:
            if norm >= skip_grad:        # host sync, as in the reference (utils/native_scaler.py:30)
                self._update(found_inf)
                return norm
        if hasattr(optimizer, "fused_step"):
            optimizer.fused_step(found_inf=found_inf)
        elif float(found_inf) == 0.0:    # host sync, as GradScaler.step does for stock optimizers
            optimizer.step()
        self._update(found_inf)
        if arena is not None:
            arena.accumulating = False
        return DeferredScalar.wrap(norm)

    def _unscale_outside(self, optimizer, arena, handled, inv, found_inf):
        key = (id(optimizer), id(arena), sum(len(g["params"]) for g in getattr(optimizer, "param_groups", [])))
        cached = getattr(self, "_outside_cache", None)
        if arena is not None and arena.owned and cached is not None and cached[0] == key:
            outside = cached[1]                            # owned arena: which gradients alias it never changes
        else:
            lo = hi = None
            if arena is not None:
                lo = arena.flat.data_ptr()
                hi = lo + arena.flat.numel() * arena.flat.element_size()
            seen = {id(p) for p in (handled or [])}
            outside = []
            for group in getattr(optimizer, "param_groups", []):
                for p in group["params"]:
                    g = p.grad
                    if id(p) in seen or (g is None and not (arena is not None and arena.owned)):
                        continue
                    if g is not None and lo is not None and g.device == arena.flat.device and lo <= g.data_ptr() < hi:
                        continue                           # lives in the flat buffer: already unscaled and checked
                    seen.add(id(p))
                    outside.append(p)
            if arena is not None and arena.owned:
                self._outside_cache = (key, outside)
        bad = None
        a_lo = arena.flat.data_ptr() if arena is not None else 0
        a_hi = a_lo + (arena.flat.numel() * arena.flat.element_size() if arena is not None else 0)
        for p in outside:
            g = p.grad
            if g is None or a_lo <= g.data_ptr() < a_hi:
                continue
            g.mul_(inv.to(g.device))
            flag = (~torch.isfinite(g).all()).float().reshape(1)
            bad = flag if bad is None else torch.maximum(bad, flag.to(bad.device))
        if bad is None:
            return found_inf
        return torch.maximum(found_inf, bad.to(found_inf.device))

    def _update(self, found_inf):
        if not self._enabled:
            return
        bad = found_inf.reshape(()) > 0
        grown = self._growth_tracker + 1
        hit = grown >= self._growth_interval
        self._scale = torch.where(bad, self._scale * self._backoff_factor,
                                  torch.where(hit, self._scale * self._growth_factor, self._scale))
        self._growth_tracker = torch.where(bad | hit, torch.zeros_like(grown), grown)

    def state_dict(self):
        if not self._enabled:
            return {"scale": 1.0}
        if METERS.enabled and self._scale is not None and self._scale.is_cuda:
            return _LazyScalerState(self)
        scale = float(self._scale) if self._scale is not None else self._init_scale
        tracker = int(self._growth_tracker) if self._growth_tracker is not None else 0
        return {"scale": scale, "growth_factor": self._growth_factor, "backoff_factor": self._backoff_factor,
                "growth_interval": self._growth_interval, "_growth_tracker": tracker}

    def load_state_dict(self, state_dict):
        if not self._enabled or not state_dict:
            return
        self._init_scale = float(state_dict["scale"])
        self._growth_factor = state_dict.get("growth_factor", self._growth_factor)
        self._backoff_factor = state_dict.get("backoff_factor", self._backoff_factor)
        self._growth_interval = state_dict.get("growth_interval", self._growth_interval)
        self._init_tracker = int(state_dict.get("_growth_tracker", 0))   # resume order: loaded before the first step
        if self._scale is not None:
            self._scale.fill_(self._init_scale)
            self._growth_tracker.fill_(self._init_tracker)
