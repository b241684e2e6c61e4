"""Flat-buffer AdamW (SURVEY.md §8f n1): parameters live as views of one fp32 buffer, gradients in the model's
GradArena, so the update of all ~98 M parameters is ONE kernel (mmae_adamw_step) instead of per-tensor loops, and a
non-finite step is skipped on the device.  Same update rule / hyper-parameter semantics as torch.optim.AdamW as the
reference builds it (utils/optim_factory.py:155-174; betas (0.9, 0.95), weight_decay 0.05 on every parameter).

GroupedFlatAdamW is the same layout behind torch.optim.AdamW's constructor: parameter groups with their own lr and
weight decay (the layer-decay groups utils/optim_factory.py:get_parameter_groups builds for the fine-tuning scripts),
stepped by ONE mmae_adamw_step_groups launch.

Checkpoints: `state_dict()` / `load_state_dict()` use torch.optim.AdamW's per-parameter layout ({step, exp_avg,
exp_avg_sq} per parameter index, sliced out of / copied into the flat moment buffers), so utils.save_model /
auto_load_model (utils/checkpoint.py:85,124-133) resume this optimizer - and a checkpoint written by the stock AdamW over
the same parameter order loads here, and vice versa."""
import ctypes

import torch

from . import _lib as L
from . import functional as Fn


class _FlatParams:
    """Parameters re-homed into one flat fp32 buffer laid out exactly like the model's gradient arena, with a bf16 twin
    that the GEMMs read their weight operands from (no per-step casts of ~117 tensors).  The update kernel keeps the twin
    current; ensure_mirror_fresh() catches every other modification through torch."""

    def _rehome(self, named, arena):
        dev = arena.flat.device
        self.flat_params = torch.zeros_like(arena.flat)
        with torch.no_grad():
            for n, p in named:
                o, numel, shape = arena.offsets[n]
                view = self.flat_params[o:o + numel].view(shape)
                view.copy_(p.data.to(dev))
                p.data = view
        self.flat_bf16 = None
        self._mirror_version = None
        self._invalidations = 0
        self._flat_views = [p for _, p in named]
        self._named = named
        if dev.type == "cuda":
            self.flat_bf16 = torch.empty(self.flat_params.numel(), dtype=torch.bfloat16, device=dev)
            L.check(L.lib().mmae_weight_mirror_register(self.flat_params.data_ptr(), self.flat_bf16.data_ptr(),
                                                        self.flat_params.numel()), "mmae_weight_mirror_register")
            Fn.register_mirror(self)

    def _params_version(self):
        # in-place torch ops on a Parameter (copy_, load_state_dict, init) bump its counter; our kernels do not
        return self._invalidations + sum(p._version for p in self._flat_views)

    def invalidate_mirror(self):
        """Call after modifying parameters in a way autograd's version counters do not see (writes through `.data`)."""
        self._invalidations += 1

    def ensure_mirror_fresh(self):
        """Re-cast the whole flat buffer (one kernel) if the parameters were modified through torch since the twin was
        last written.  The update kernel itself writes the twin and does not touch the version counters.  Called by the
        model at the start of every forward."""
        if self.flat_bf16 is None:
            return
        ver = self._params_version()
        if self._mirror_version == ver:
            return
        L.check(L.lib().mmae_cast_f32_to_bf16(self.flat_params.data_ptr(), self.flat_bf16.data_ptr(),
                                              self.flat_params.numel(), L.current_stream()), "mmae_cast_f32_to_bf16")
        self._mirror_version = ver

    def release_mirror(self):
        if getattr(self, "flat_bf16", None) is not None:
            try:
                L.lib().mmae_weight_mirror_register(self.flat_params.data_ptr(), None, 0)
            except Exception:  # noqa: BLE001  (interpreter shutdown)
                pass
            self.flat_bf16 = None

    def __del__(self):
        self.release_mirror()


class FlatAdamW(_FlatParams, torch.optim.Optimizer):
    def __init__(self, model, lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.05):
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        params = [p for _, p in named]
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, lr_scale=1.0))
        arena = model.own_gradients(True)
        self.mmae_arena = arena
        dev = arena.flat.device
        self._rehome(named, arena)
        self.exp_avg = torch.zeros_like(self.flat_params)
        self.exp_avg_sq = torch.zeros_like(self.flat_params)
        # {learning rate, step count} on the device: the update kernel reads them there, so a captured CUDA graph replays
        # with the current schedule value and an advancing bias correction
        self._dyn = torch.zeros(2, dtype=torch.float32, device=dev)
        self._lr_host = torch.zeros(1, dtype=torch.float32).pin_memory() if dev.type == "cuda" else torch.zeros(1)
        self._lr_synced = None
        self._bind_state()
        self.sync_hyperparams()

    # ------------------------------------------------------------------------------------------------------------
    # optimizer state in torch.optim.AdamW's layout, as views of the flat buffers (checkpoint / resume contract)
    # ------------------------------------------------------------------------------------------------------------
    def _bind_state(self):
        arena = self.mmae_arena
        step = self._dyn[1]                      # 0-dim view of the device-side step counter, shared by every entry
        for n, p in self._named:
            o, numel, shape = arena.offsets[n]
            self.state[p] = {"step": step, "exp_avg": self.exp_avg[o:o + numel].view(shape),
                             "exp_avg_sq": self.exp_avg_sq[o:o + numel].view(shape)}

    def load_state_dict(self, state_dict):
        """torch.optim.AdamW-layout state -> flat moment buffers + device step counter; hyper-parameters as usual."""
        super().load_state_dict(state_dict)      # validates sizes, restores param_groups, materialises per-parameter state
        loaded_step = None
        with torch.no_grad():
            for n, p in self._named:
                st = self.state.get(p)
                if not st:
                    continue
                o, numel, shape = self.mmae_arena.offsets[n]
                if "exp_avg" in st:
                    self.exp_avg[o:o + numel].view(shape).copy_(st["exp_avg"])
                if "exp_avg_sq" in st:
                    self.exp_avg_sq[o:o + numel].view(shape).copy_(st["exp_avg_sq"])
                if "step" in st and loaded_step is None:
                    loaded_step = float(st["step"])
            if loaded_step is not None:
                self._dyn[1].fill_(loaded_step)
        self._bind_state()
        self._lr_synced = None
        self.sync_hyperparams()
        self.invalidate_mirror()

    def sync_hyperparams(self):
        """Push the current param_group learning rate to the device scalar (call before a graph replay)."""
        g = self.param_groups[0]
        lr = g["lr"] * g.get("lr_scale", 1.0)
        if lr == self._lr_synced:
            return                                  # nothing to copy: keeps a replayed step free of H2D traffic
        self._lr_host[0] = lr
        self._dyn[0:1].copy_(self._lr_host, non_blocking=True)
        self._lr_synced = lr

    @torch.no_grad()
    def fused_step(self, found_inf=None):
        """One kernel over the flat buffers.  The step counter lives on the device and is advanced by the call itself,
        only when the step is taken (found_inf == 0): a skipped step leaves moments, parameters AND the bias correction
        untouched, like GradScaler.step."""
        Fn.sync_deterministic()
        g = self.param_groups[0]
        if not (self._dyn.is_cuda and torch.cuda.is_current_stream_capturing()):
            self.sync_hyperparams()
        Fn.adamw_step(self.flat_params, self.mmae_arena.flat, self.exp_avg, self.exp_avg_sq, g["lr"] * g.get("lr_scale", 1.0),
                      g["betas"], g["eps"], g["weight_decay"], 1, found_inf, dyn=self._dyn)

    @torch.no_grad()
    def step(self, closure=None):
        self.fused_step(None)

    def zero_grad(self, set_to_none=True):
        """Gradients alias the model's arena, which the model zeroes (one memset) at the start of the next training
        forward - unless an accumulation is in progress (NativeScalerWithGradNormCount(update_grad=False)); after a step the
        accumulation is over."""
        self.mmae_arena.accumulating = False
        return None


# ---------------------------------------------------------------------------------------------------------------------
# torch.optim.AdamW with parameter groups over the flat buffers
# ---------------------------------------------------------------------------------------------------------------------
def _flatten_params(params):
    """Every tensor of a torch.optim-style `params` argument (tensors, or dicts with a "params" entry)."""
    out = []
    for item in params:
        if isinstance(item, dict):
            ps = item["params"]
            out += [ps] if isinstance(ps, torch.Tensor) else list(ps)
        else:
            out.append(item)
    return out


def _on_device(p):
    return p.device.type == "cuda"


def owning_model(params):
    """The live MultiMAE / MultiViT whose trainable parameters include every tensor of `params` (a flat list of trainable
    tensors), with its
    {id(parameter): name} map; (None, reason) when there is none."""
    from . import multimae as mm
    if not params:
        return None, "no parameters"
    off = [p for p in params if not _on_device(p)]
    if off:
        return None, "%d parameter(s) not on CUDA" % len(off)
    ids = {id(p) for p in params}
    if len(ids) != len(params):
        return None, "a parameter appears more than once"
    for model in mm.live_models():
        names = {id(p): n for n, p in model.named_parameters() if p.requires_grad}
        if ids <= names.keys():
            return model, names
    return None, "a parameter is not a trainable parameter of one MultiMAE / MultiViT model"


class GroupedFlatAdamW(_FlatParams, torch.optim.Optimizer):
    """torch.optim.AdamW (decoupled weight decay, torch's defaults) whose parameter groups - each with its own lr and
    weight_decay, read from `param_groups` at every step - are stepped by one kernel over flat buffers laid out like the
    model's gradient arena.  The parameters must all be trainable parameters of one live MultiMAE / MultiViT on CUDA.

    `fused_step(found_inf)` is the GradScaler-style entry: a non-zero found_inf[0] skips the step on the device (step count
    included) without a host sync.  `betas` and `eps` are shared by all groups."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, *, maximize=False,
                 foreach=None, capturable=False, differentiable=False, fused=None):
        unsupported = [k for k, v in (("amsgrad", amsgrad), ("maximize", maximize), ("capturable", capturable),
                                      ("differentiable", differentiable)) if v]
        unsupported += [k for k, v in (("foreach", foreach), ("fused", fused)) if v is not None]
        if unsupported:
            raise NotImplementedError("GroupedFlatAdamW: %s not supported" % ", ".join(unsupported))
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: %s" % lr)
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: %s" % eps)
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError("Invalid beta parameters: %s" % (betas,))
        if not 0.0 <= weight_decay:
            raise ValueError("Invalid weight_decay value: %s" % weight_decay)
        # the keys torch.optim.AdamW writes into every param group: a checkpoint of either optimizer steps in the other
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False, foreach=None,
                        capturable=False, differentiable=False, fused=None, decoupled_weight_decay=True)
        self._layout_fixed = False
        super().__init__(params, defaults)
        self._layout_fixed = True
        # frozen tensors (requires_grad=False, e.g. a fixed position table in model.parameters()) are never stepped, as in
        # torch, where they have no gradient
        flat = [p for g in self.param_groups for p in g["params"] if p.requires_grad]
        model, names = owning_model(flat)
        if model is None:
            raise ValueError("GroupedFlatAdamW: %s" % names)
        Fn._require_cuda(flat[0], "GroupedFlatAdamW")
        arena = model.own_gradients(True)
        self.mmae_arena = arena
        self._rehome([(names[id(p)], p) for p in flat], arena)
        self.exp_avg = torch.zeros_like(self.flat_params)
        self.exp_avg_sq = torch.zeros_like(self.flat_params)
        self._step = torch.zeros(1, dtype=torch.float32, device=arena.flat.device)   # advanced by the kernel launch
        self._build_segments()
        self._bind_state()

    def add_param_group(self, param_group):
        if getattr(self, "_layout_fixed", False):
            raise NotImplementedError("GroupedFlatAdamW: the flat layout is fixed at construction; no groups can be added")
        super().add_param_group(param_group)

    def _build_segments(self):
        """(arena offset, length, group) per segment: every parameter's 8-element-padded slot, adjacent slots of one group
        merged into one segment (slot padding is zero in every buffer, and stays zero under the update)."""
        offsets = self.mmae_arena.offsets
        name_of = {id(p): n for n, p in self._named}
        slots = []
        for k, g in enumerate(self.param_groups):
            for p in g["params"]:
                if id(p) not in name_of:
                    continue                     # frozen
                o, numel, _ = offsets[name_of[id(p)]]
                slots.append((o, (numel + 7) // 8 * 8, k))
        slots.sort()
        segs = []
        for o, n, k in slots:
            if segs and segs[-1][2] == k and segs[-1][0] + segs[-1][1] == o:
                segs[-1] = (segs[-1][0], segs[-1][1] + n, k)
            else:
                segs.append((o, n, k))
        self.segments = segs
        fb, tw = self.flat_params.data_ptr(), (self.flat_bf16.data_ptr() if self.flat_bf16 is not None else None)
        g_ptr, m_ptr, v_ptr = self.mmae_arena.flat.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr()
        table = (L.AdamwSegment * max(len(segs), 1))()
        for i, (o, n, k) in enumerate(segs):
            table[i] = L.AdamwSegment(fb + 4 * o, g_ptr + 4 * o, m_ptr + 4 * o, v_ptr + 4 * o,
                                      None if tw is None else tw + 2 * o, n, k, 0)
        self._table = table
        self._lrs = (ctypes.c_double * len(self.param_groups))()
        self._wds = (ctypes.c_double * len(self.param_groups))()

    def _bind_state(self):
        offsets = self.mmae_arena.offsets
        step = self._step[0]                     # 0-dim view of the device-side step counter
        for n, p in self._named:
            o, numel, shape = offsets[n]
            self.state[p] = {"step": step, "exp_avg": self.exp_avg[o:o + numel].view(shape),
                             "exp_avg_sq": self.exp_avg_sq[o:o + numel].view(shape)}

    def state_dict(self):
        """torch.optim.AdamW's layout; each parameter gets its own host `step` tensor, as torch keeps them (reads the
        device step count: a host sync, at checkpoint time only)."""
        sd = super().state_dict()
        step = float(self._step[0])
        sd["state"] = {k: dict(v, step=torch.tensor(step, dtype=torch.float32)) for k, v in sd["state"].items()}
        return sd

    def load_state_dict(self, state_dict):
        """torch.optim.AdamW-layout state -> flat moment buffers + device step counter; param_groups as torch restores
        them (their lr / weight_decay apply from the next step)."""
        super().load_state_dict(state_dict)      # validates sizes, restores param_groups, materialises per-parameter state
        loaded_step = 0.0
        offsets = self.mmae_arena.offsets
        with torch.no_grad():
            for n, p in self._named:
                o, numel, shape = offsets[n]
                st = self.state.get(p) or {}
                for key, buf in (("exp_avg", self.exp_avg), ("exp_avg_sq", self.exp_avg_sq)):
                    if key in st:
                        buf[o:o + numel].view(shape).copy_(st[key])
                    else:
                        buf[o:o + numel].zero_()
                if "step" in st:
                    loaded_step = max(loaded_step, float(st["step"]))
            self._step.fill_(loaded_step)
        self._bind_state()
        self.invalidate_mirror()

    def _shared(self):
        g0 = self.param_groups[0]
        for g in self.param_groups[1:]:
            if tuple(g["betas"]) != tuple(g0["betas"]) or g["eps"] != g0["eps"]:
                raise ValueError("GroupedFlatAdamW: every parameter group must have the same betas and eps")
        return g0["betas"], g0["eps"]

    @torch.no_grad()
    def fused_step(self, found_inf=None):
        """One launch over every group (more for a table longer than one launch holds).  The step count lives on the
        device and advances only when the step is taken (found_inf[0] == 0): a skipped step leaves parameters, moments, the
        bf16 twin and the bias correction untouched, like GradScaler.step, and needs no host sync."""
        Fn.sync_deterministic()
        betas, eps = self._shared()
        for k, g in enumerate(self.param_groups):
            self._lrs[k] = float(g["lr"])
            self._wds[k] = float(g["weight_decay"])
        Fn.adamw_step_groups(self._table, len(self.segments), self._lrs, self._wds, betas, eps, self._step, found_inf)

    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.fused_step(None)
        return loss

    def zero_grad(self, set_to_none=True):
        """As FlatAdamW.zero_grad: the gradients alias the model's arena, which the next training forward zeroes."""
        self.mmae_arena.accumulating = False
        return None


def adamw_or_stock(params, *args, **kwargs):
    """GroupedFlatAdamW over `params` when one live MultiMAE / MultiViT on CUDA owns them all; torch.optim.AdamW (with
    one printed line saying why) otherwise - e.g. the uncertainty task balancer's log_vars in pre-training."""
    params = [dict(g, params=list(g["params"]) if not isinstance(g["params"], torch.Tensor) else [g["params"]])
              if isinstance(g, dict) else g for g in params]
    model, why = owning_model([p for p in _flatten_params(params) if p.requires_grad])
    if model is None:
        print("MMAE_FLAT_ADAMW: %s; using torch.optim.AdamW" % why)
        return torch.optim.AdamW(params, *args, **kwargs)
    return GroupedFlatAdamW(params, *args, **kwargs)
